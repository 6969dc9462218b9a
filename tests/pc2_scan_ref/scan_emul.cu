// scan_emul.cu -- TEST HARNESS ONLY: the product's per-point and per-cell functions of b2_rcc_set_cloud_spherical (rmcl_b200/csrc/kernels.cuh:
// scan_cloud_key and scan_cell_entry, with scan_point_key, scan_bin and dataset_entry inlined) compiled for the CPU.  Points are visited in
// the caller's order and each cell keeps the larger key, as k_scan_bin_cloud's atomicMax does; then one scan_cell_entry per cell.
// Built by tests/pc2_scan_ref.py with the flags of tests/chain_ref (host code with -ffp-contract=off: plain ops rounded like __fmul_rn etc.).
#include <algorithm>
#include <vector>

#include "../../rmcl_b200/csrc/kernels.cuh"

extern "C" __attribute__((visibility("default"))) void emul_scan_from_cloud(const uint8_t* cloud, uint32_t width, uint32_t height, uint64_t row_step,
                                                                           uint32_t point_step, const uint32_t* off, uint32_t f64, const b2_transform* T,
                                                                           const b2_spherical_model* m, const uint32_t* order, const float* dirs,
                                                                           float* ranges, float* pts, uint8_t* mask)
{
    CloudScan c;
    c.width = width; c.n_points = width * height; c.row_step = row_step; c.point_step = point_step;
    for (int k = 0; k < 3; k++) c.off[k] = off[k];
    c.f64 = f64; c.T = tf_from_pod(*T);
    c.phi_min = m->phi_min; c.phi_inc = m->phi_inc; c.theta_min = m->theta_min; c.theta_inc = m->theta_inc; c.phi_n = m->phi_size; c.theta_n = m->theta_size;
    c.range_min = m->range_min; c.range_max = m->range_max; c.fill = (float)((double)m->range_max + 1.0);
    const uint32_t n = m->phi_size * m->theta_size;
    std::vector<unsigned long long> keys(n, 0ull);
    for (uint32_t j = 0; j < c.n_points; j++) {
        const uint32_t i = order ? order[j] : j;
        uint32_t cell = 0;
        const unsigned long long key = scan_cloud_key(cloud, c, i, cell);
        if (key) keys[cell] = std::max(keys[cell], key);
    }
    const float orig[3] = {0.f, 0.f, 0.f};
    for (uint32_t k = 0; k < n; k++) scan_cell_entry(k, keys.data(), c, dirs, orig, ranges, pts, mask);
}
