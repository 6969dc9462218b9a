// progress_emul.cu -- TEST HARNESS ONLY: the product's update between two chained corrections (rmcl_b200/csrc/icp_loop.cuh: micp_progress,
// icp_adaptive_max_dist) compiled for the CPU, so that it can be compared with the C restatement in a container without a GPU.
// Included into the emulator library (tests/emul/emul.cu).

extern "C" {
__attribute__((visibility("default"))) double emul_micp_progress(const b2_transform* Tom, const b2_transform* T_onew_oold, uint32_t n_meas, uint32_t valid, int adaptive)
{
    return micp_progress(*Tom, *T_onew_oold, n_meas, valid, adaptive != 0);
}
__attribute__((visibility("default"))) float emul_adaptive_max_dist(float max_dist, float max_dist_min, double cp) { return icp_adaptive_max_dist(max_dist, max_dist_min, cp); }
}
