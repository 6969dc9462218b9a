// cloud_emul.cu -- TEST HARNESS ONLY: the product's per-sample function of b2_pf_sample_cloud (rmcl_b200/csrc/kernels.cuh: pf_sample_beam,
// with philox4x32_10 and cloud_coord inlined) compiled for the CPU, run for samples 0 .. n_samples-1 as k_pf_sample_cloud runs them: each
// writes its valid flag and its beam (all zero when invalid).  Built by tests/pf_cloud_ref.py with the flags of tests/chain_ref (host code
// with -ffp-contract=off: plain ops rounded like __fmul_rn etc.).
#include "../../rmcl_b200/csrc/kernels.cuh"

extern "C" __attribute__((visibility("default"))) void emul_pf_samples(const uint8_t* cloud, uint32_t width, uint32_t height, uint64_t row_step,
                                                                      uint32_t point_step, const uint32_t* off, uint32_t f64, uint64_t seed, uint32_t step,
                                                                      uint32_t n_samples, uint32_t* valid, b2_range_meas* out)
{
    CloudBeams c;
    c.width = width; c.n_points = (uint32_t)((uint64_t)width * height); c.row_step = row_step; c.point_step = point_step;
    for (int k = 0; k < 3; k++) c.off[k] = off[k];
    c.f64 = f64; c.seed = seed; c.step = step;
    for (uint32_t k = 0; k < n_samples; k++) {
        PfBeamSample s = {};
        s.valid = pf_sample_beam(cloud, c, k, &s.m) ? 1u : 0u;
        valid[k] = s.valid;
        out[k] = s.m;
    }
}
