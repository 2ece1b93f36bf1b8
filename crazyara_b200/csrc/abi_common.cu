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

// ------------------------------------------------------------------ DeviceRanges
namespace {
struct VmmCalls {
    decltype(&cuMemGetAllocationGranularity) granularity = nullptr;
    decltype(&cuMemAddressReserve) reserve = nullptr;
    decltype(&cuMemAddressFree) free = nullptr;
    decltype(&cuMemCreate) create = nullptr;
    decltype(&cuMemRelease) release = nullptr;
    decltype(&cuMemMap) map = nullptr;
    decltype(&cuMemUnmap) unmap = nullptr;
    decltype(&cuMemSetAccess) set_access = nullptr;
    bool ok = false;
};
template <typename F>
bool entry_point(const char* name, F* fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint(name, &p, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess) return false;
    *fn = reinterpret_cast<F>(p);
    return true;
}
const VmmCalls& vmm() {
    static const VmmCalls c = [] {
        VmmCalls v;
        v.ok = entry_point("cuMemGetAllocationGranularity", &v.granularity) && entry_point("cuMemAddressReserve", &v.reserve) &&
               entry_point("cuMemAddressFree", &v.free) && entry_point("cuMemCreate", &v.create) &&
               entry_point("cuMemRelease", &v.release) && entry_point("cuMemMap", &v.map) && entry_point("cuMemUnmap", &v.unmap) &&
               entry_point("cuMemSetAccess", &v.set_access);
        return v;
    }();
    return c;
}
CUmemAllocationProp pinned_on(int device) {
    CUmemAllocationProp prop = {};
    prop.type = CU_MEM_ALLOCATION_TYPE_PINNED;
    prop.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
    prop.location.id = device;
    return prop;
}
}  // namespace

DeviceRanges::~DeviceRanges() {
    if (!vmm().ok) return;
    for (const Piece& p : pieces_) {
        vmm().unmap(p.at, p.bytes);
        vmm().release(p.h);
    }
    for (const Piece& r : reserved_) vmm().free(r.at, r.bytes);
}

int DeviceRanges::init(int device) {
    if (!vmm().ok) return set_error("the CUDA virtual memory management entry points are not available");
    device_ = device;
    const CUmemAllocationProp prop = pinned_on(device);
    const CUresult r = vmm().granularity(&gran_, &prop, CU_MEM_ALLOC_GRANULARITY_MINIMUM);
    if (r != CUDA_SUCCESS) return set_error("cuMemGetAllocationGranularity failed: %d", static_cast<int>(r));
    return 0;
}

int DeviceRanges::reserve(size_t bytes, CUdeviceptr* base) {
    bytes = (bytes + gran_ - 1) / gran_ * gran_;
    const CUresult r = vmm().reserve(base, bytes, gran_, 0, 0);
    if (r != CUDA_SUCCESS) return set_error("cuMemAddressReserve(%zu bytes) failed: %d", bytes, static_cast<int>(r));
    reserved_.push_back(Piece{*base, bytes, 0});
    return 0;
}

int DeviceRanges::map(CUdeviceptr at, size_t bytes, cudaStream_t zero_on) {
    const CUmemAllocationProp prop = pinned_on(device_);
    CUmemGenericAllocationHandle h;
    CUresult r = vmm().create(&h, bytes, &prop, 0);
    if (r == CUDA_ERROR_OUT_OF_MEMORY) return 1;
    if (r != CUDA_SUCCESS) return set_error("cuMemCreate(%zu bytes) failed: %d", bytes, static_cast<int>(r));
    r = vmm().map(at, bytes, 0, h, 0);
    if (r != CUDA_SUCCESS) {
        vmm().release(h);
        return set_error("cuMemMap(%zu bytes) failed: %d", bytes, static_cast<int>(r));
    }
    pieces_.push_back(Piece{at, bytes, h});
    CUmemAccessDesc access = {};
    access.location = prop.location;
    access.flags = CU_MEM_ACCESS_FLAGS_PROT_READWRITE;
    r = vmm().set_access(at, bytes, &access, 1);
    if (r != CUDA_SUCCESS) return set_error("cuMemSetAccess(%zu bytes) failed: %d", bytes, static_cast<int>(r));
    ARA_CUDA_OK(cudaMemsetAsync(reinterpret_cast<void*>(at), 0, bytes, zero_on));
    return 0;
}

void DeviceRanges::unmap(CUdeviceptr lo, CUdeviceptr hi) {
    size_t k = 0;
    for (const Piece& p : pieces_) {
        if (p.at >= lo && p.at + p.bytes <= hi) {
            vmm().unmap(p.at, p.bytes);
            vmm().release(p.h);
        } else {
            pieces_[k++] = p;
        }
    }
    pieces_.resize(k);
}

}  // namespace ara

extern "C" const char* ara_last_error(void) { return ara::last_error_ref().c_str(); }
