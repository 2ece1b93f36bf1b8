#include "abi_common.h"

namespace ara {

std::string& last_error_ref() {
    static thread_local std::string err;
    return err;
}

int set_error(const char* fmt, ...) {
    char buf[1024];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof(buf), fmt, ap);
    va_end(ap);
    last_error_ref() = buf;
    return -1;
}

static thread_local int g_pdl_suspended = 0;
PdlSuspend::PdlSuspend(bool on) : on_(on) {
    if (on_) ++g_pdl_suspended;
}
PdlSuspend::~PdlSuspend() {
    if (on_) --g_pdl_suspended;
}

bool pdl_enabled() { return g_pdl_suspended == 0; }

}  // namespace ara

extern "C" const char* ara_last_error(void) { return ara::last_error_ref().c_str(); }
