// search_emul.cu -- TEST HARNESS ONLY: the product's functions of b2_pf_global_search (rmcl_b200/csrc/kernels.cuh: search_pose,
// search_cell + search_candidate, pf_surface_pose, search_is_peak, search_key, search_keep) compiled for the CPU, so that they can be compared
// with the C restatement (pf_search_ref.c) in a container without a GPU.  The yaw table is made as b2_pf_global_search makes it.
// It is the emulator library (tests/emul/emul.cu: the scene handle and the host BVH build) plus the functions below, built into a library
// of its own by tests/pf_search_ref.py.
#include "../emul/emul.cu"

static std::vector<float> emul_search_yaw(uint32_t K)
{
    std::vector<float> yaw(2 * (size_t)K);
    for (uint32_t k = 0; k < K; k++) { const double half = 0.5 * search_psi(k, K); yaw[2 * k] = (float)std::sin(half); yaw[2 * k + 1] = (float)std::cos(half); }
    return yaw;
}

// candidates [0, n) of the grid: surface 0 -> search_pose; 1 -> the per-cell probe plus placement (search_cell, search_candidate); 2 ->
// pf_surface_pose on every candidate.  valid[c] = 0 where the rule finds no ground (poses then unchanged from search_pose).
EMUL_API void emul_search_candidates(void* sc, float x0, float y0, float z0, float step, uint32_t nx, uint32_t ny, uint32_t K, int surface,
                                     const b2_surface_config* cfg, b2_transform* out, uint8_t* valid)
{
    const std::vector<float> yaw = emul_search_yaw(K);
    const SearchGrid g{x0, y0, z0, step, nx, ny, K, yaw.data()};
    const uint32_t n = nx * ny * K, n_cells = nx * ny;
    b2_surface_config c{};
    float cos_max = 0.0f, tfar = 0.0f;
    if (cfg) { c = *cfg; cos_max = (float)std::cos((double)c.max_slope); tfar = c.probe_above + c.probe_below; }
    std::vector<SearchCell> cells(surface == 1 ? n_cells : 0);
    if (surface == 1) {
        const BvhView bvh = view_of(sc);
        #pragma omp parallel for schedule(dynamic, 64)
        for (int64_t q = 0; q < (int64_t)n_cells; q++) cells[q] = search_cell(bvh, g, (uint32_t)q, c, cos_max, tfar);
    }
    #pragma omp parallel for schedule(dynamic, 256)
    for (int64_t q = 0; q < (int64_t)n; q++) {
        Tf T = search_pose(g, (uint32_t)q);
        bool ok = true;
        if (surface == 1) ok = search_candidate(g, cells.data(), c, (uint32_t)q, T);
        else if (surface == 2) { const BvhView bvh = view_of(sc); Tf U = T; ok = pf_surface_pose(bvh, U, c, cos_max, tfar); if (ok) T = U; }
        if (!ok) T = search_pose(g, (uint32_t)q);
        memset(out + q, 0, sizeof(b2_transform));
        tf_store(out + q, T);
        valid[q] = ok ? 1 : 0;
    }
}
// the peak rule at every candidate -> flags; and the rank keys of the listed candidates
EMUL_API void emul_search_peaks(const float* s, uint32_t nx, uint32_t ny, uint32_t K, uint8_t* peak)
{
    const uint32_t n = nx * ny * K;
    #pragma omp parallel for schedule(static)
    for (int64_t c = 0; c < (int64_t)n; c++) peak[c] = search_is_peak(s, nx, ny, K, (uint32_t)c) ? 1 : 0;
}
// the ranking (the keys in ascending order, as the radix sort orders them) and the separation pass, as b2_pf_global_search runs them
EMUL_API uint32_t emul_search_records(const float* s, const uint32_t* list, uint64_t m, float x0, float y0, float step, uint32_t nx, uint32_t ny, uint32_t K,
                                      uint32_t max_records, float sep_xy, float sep_yaw, uint32_t* kept)
{
    std::vector<unsigned long long> keys(m);
    for (uint64_t q = 0; q < m; q++) keys[q] = search_key(s[list[q]], list[q]);
    std::sort(keys.begin(), keys.end());
    const SearchGrid g{x0, y0, 0.0f, step, nx, ny, K, nullptr};
    uint32_t n_kept = 0;
    for (uint64_t q = 0; q < m && n_kept < max_records; q++) {
        const uint32_t c = (uint32_t)keys[q];
        if (search_keep(g, c, kept, n_kept, (double)sep_xy, (double)sep_yaw)) kept[n_kept++] = c;
    }
    return n_kept;
}
