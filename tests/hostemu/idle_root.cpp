// Test scaffolding: the host emulation (hostemu.cpp) plus the root phase of a go that leaves the tree out
// (ara_search_set_active): root_kernel's idle path, search_dev.cuh idle_root, for both thread views.  Compiled on its
// own by tests/test_idle_tree_hostemu.py; the HeSearch it works on comes from the same source, so the layouts agree.
#include "hostemu.cpp"

extern "C" void he_search_idle_root(HeSearch* s) {
    for (HeBatch& bt : s->batch) idle_root(bt.t);
}
