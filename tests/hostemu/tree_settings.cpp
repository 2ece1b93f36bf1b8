// Test scaffolding: the host emulation (hostemu.cpp) plus the root phase of a go in which the tree has its own Q-value
// weight and Dirichlet epsilon (ara_search_set_tree_settings): root_kernel applies them once the root has been created or
// taken over (search_dev.cuh apply_tree_settings).  Compiled on its own by tests/test_tree_settings_hostemu.py.
#include "hostemu.cpp"

extern "C" int he_search_set_root_with_settings(HeSearch* s, const HeState* root, float q_value_weight, float dirichlet_epsilon) {
    const int n = he_search_set_root(s, root);
    apply_tree_settings(s->st, q_value_weight, dirichlet_epsilon);
    return n;
}
