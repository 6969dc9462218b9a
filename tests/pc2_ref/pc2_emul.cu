// pc2_emul.cu -- TEST HARNESS ONLY: the product's per-ray function of b2_rcc_set_cloud_o1dn (rmcl_b200/csrc/kernels.cuh: o1dn_cloud_entry, with
// cloud_coord, o1dn_from_point and dataset_entry inlined) compiled for the CPU, one call per output ray as the kernel's threads make them.
// Built by tests/pc2_ref.py with the flags of tests/chain_ref (host code with -ffp-contract=off: plain float ops rounded like __fmul_rn etc.).
#include "../../rmcl_b200/csrc/kernels.cuh"

extern "C" __attribute__((visibility("default"))) void emul_o1dn_from_cloud(const uint8_t* cloud, uint32_t w_out, uint32_t h_out, uint64_t row_step,
                                                                           uint32_t point_step, const uint32_t* off, uint32_t f64, const uint32_t* h_skip_inc,
                                                                           const uint32_t* w_skip_inc, float range_min, float range_max,
                                                                           float* dirs, float* ranges, float* pts, uint8_t* mask)
{
    CloudO1Dn c;
    c.w_out = w_out; c.h_out = h_out; c.row_step = row_step; c.point_step = point_step;
    for (int k = 0; k < 3; k++) c.off[k] = off[k];
    c.f64 = f64; c.h_begin = h_skip_inc[0]; c.h_inc = h_skip_inc[1]; c.w_begin = w_skip_inc[0]; c.w_inc = w_skip_inc[1];
    c.range_min = range_min; c.range_max = range_max;
    for (uint32_t k = 0; k < w_out * h_out; k++) o1dn_cloud_entry(cloud, c, k, dirs, ranges, pts, mask);
}
