// bnb_emul.cu -- TEST HARNESS ONLY: the product's functions of b2_pf_global_search_bnb (rmcl_b200/csrc/kernels.cuh: pyr_levels, pyr_fine2,
// pyr_fine4, pyr_brick, pyr_up, search_bnb_constants, bnb_node, bnb_beam_bound, bnb_candidate) compiled for the CPU, so that the pyramid and
// the bound can be checked in a container without a GPU.  It is the emulator library (tests/emul/emul.cu) plus the functions below, built
// into a library of its own by tests/pf_search_bnb_ref.py.
#include "../emul/emul.cu"

static std::vector<float> bnb_yaw(uint32_t K)
{
    std::vector<float> yaw(2 * (size_t)K);
    for (uint32_t k = 0; k < K; k++) { const double half = 0.5 * search_psi(k, K); yaw[2 * k] = (float)std::sin(half); yaw[2 * k + 1] = (float)std::cos(half); }
    return yaw;
}

// the pyramid as the kernels build it: fine2 (n_slots x 64), fine4 (n_slots x 8), the dense levels (off[L], returns their count)
EMUL_API uint32_t emul_bnb_pyramid(const float* lo, const float* hi, float h, float trunc, const uint32_t* index, const float* bricks, uint64_t n_slots,
                                   float* fine2, float* fine4, float* dense, uint64_t* off)
{
    const DfieldView f = field_of(lo, hi, h, trunc, index, bricks);
    SearchPyr P{};
    pyr_levels(f, P);
    for (uint64_t t = 0; t < n_slots * 64u; t++) fine2[t] = pyr_fine2(f, (uint32_t)(t / 64u), (uint32_t)(t % 64u));
    for (uint64_t t = 0; t < n_slots * 8u; t++) fine4[t] = pyr_fine4(fine2, (uint32_t)(t / 8u), (uint32_t)(t % 8u));
    for (uint64_t t = 0; t < (uint64_t)f.bx * f.by * f.bz; t++) dense[t] = pyr_brick(f, fine4, t);
    for (uint32_t L = 1; L < P.n_dense; L++) {
        const uint32_t dx = pyr_dim(f.bx, L), dy = pyr_dim(f.by, L), dz = pyr_dim(f.bz, L);
        for (uint64_t t = 0; t < (uint64_t)dx * dy * dz; t++)
            dense[P.off[L] + t] = pyr_up(dense + P.off[L - 1], pyr_dim(f.bx, L - 1), pyr_dim(f.by, L - 1), pyr_dim(f.bz, L - 1), dx, dy, t);
    }
    for (uint32_t L = 0; L < P.n_dense; L++) off[L] = P.off[L];
    return P.n_dense;
}

// bounds of the nodes of tree level `level` ((bi, bj, k) -> out[(k * nby + bj) * nbx + bi]) when level >= 1, or the scores of every candidate
// (c order, -1 off surface) when level is 0; scene: the map for the surface rule (nullable without surface)
EMUL_API void emul_bnb_eval(void* scene, const float* lo, const float* hi, float h, float trunc, const uint32_t* index, const float* bricks,
                            uint64_t n_slots, const b2_transform* Tsb_val, const b2_range_meas* beams, uint32_t n_beams, const b2_pf_params* prm,
                            const b2_search_config* cfg, const b2_surface_config* surface, uint32_t level, float* out)
{
    const DfieldView f = field_of(lo, hi, h, trunc, index, bricks);
    SearchPyr P{};
    const uint64_t n_dense = pyr_levels(f, P);
    std::vector<float> fine2(std::max<uint64_t>(1, n_slots * 64u)), fine4(std::max<uint64_t>(1, n_slots * 8u)), dense(n_dense);
    std::vector<uint64_t> off(B2_BNB_MAX_DENSE);
    emul_bnb_pyramid(lo, hi, h, trunc, index, bricks, n_slots, fine2.data(), fine4.data(), dense.data(), off.data());
    P.fine2 = fine2.data(); P.fine4 = fine4.data(); P.dense = dense.data();
    const b2_search_config c = *cfg;
    const std::vector<float> yaw = bnb_yaw(c.n_yaw);
    const SearchGrid g{c.x0, c.y0, c.z0, c.step, c.nx, c.ny, c.n_yaw, yaw.data()};
    float cos_max = 0.0f, tfar = 0.0f;
    if (surface) { cos_max = (float)std::cos((double)surface->max_slope); tfar = surface->probe_above + surface->probe_below; }
    const SearchBnb sb = search_bnb_constants(c, *Tsb_val, surface, cos_max, tfar);
    std::vector<PfBeam> pb(n_beams);
    for (uint32_t b = 0; b < n_beams; b++) {
        const b2_range_meas& m = beams[b];
        pb[b] = PfBeam{m.orig.x, m.orig.y, m.orig.z, m.dir.x, m.dir.y, m.dir.z, m.range, b};
    }
    float sigma_quad; double denom; pf_constants(*prm, sigma_quad, denom);
    const Tf Tsb = tf_from_pod(*Tsb_val);
    const uint64_t nbx = ((uint64_t)c.nx + (1ull << level) - 1) >> level, nby = ((uint64_t)c.ny + (1ull << level) - 1) >> level;
    const int64_t n = (int64_t)(nbx * nby * c.n_yaw);
    #pragma omp parallel for schedule(dynamic, 16)
    for (int64_t q = 0; q < n; q++) {
        const uint32_t bi = (uint32_t)(q % nbx), bj = (uint32_t)(q / nbx % nby), k = (uint32_t)(q / nbx / nby);
        std::vector<float> e(n_beams);
        bool ok = true;
        if (level > 0) {
            float ext[4];
            const Tf Tsm = tf_mul(bnb_node(g, sb, level, bnb_key(bi, bj, k), ext), Tsb);
            for (uint32_t b = 0; b < n_beams; b++)
                e[b] = bnb_beam_bound(f, P, sb, Tsm, (double)ext[1] - (double)ext[0], (double)ext[3] - (double)ext[2], bnb_tmax(sb, ext), pb[b], sigma_quad, denom);
        } else {
            const BvhView bvh = surface ? view_of(scene) : BvhView{};
            Tf T;
            ok = bnb_candidate(surface ? &bvh : nullptr, g, surface ? *surface : b2_surface_config{}, cos_max, tfar, bi, bj, k, T);
            const Tf Tsm = tf_mul(T, Tsb);
            if (ok) for (uint32_t b = 0; b < n_beams; b++) e[b] = pf_eval_field(f, Tsm, pb[b], sigma_quad, denom);
        }
        b2_gaussian1d lk; lk.mean = 0.0f; lk.sigma = 0.0f; lk.n_meas = 0u;
        pf_merge(lk, e.data(), n_beams);
        out[q] = ok ? lk.mean : -1.0f;
    }
}

// one pass's selection over L (its candidates Lc sorted ascending, scores Ls): the peak rule over L (search_peak_rule with bnb_find, a
// missing neighbour behind), the peaks ranked by a stable sort on search_rank over the c-ascending list (cub's stable radix sort), and the
// separation pass (search_keep over 64-bit c) until max_records are kept.  -> n_kept; kept_c / kept_s in rank order, *n_peaks
EMUL_API uint32_t emul_bnb_select(const uint64_t* Lc, const float* Ls, uint64_t n, const b2_search_config* cfg, uint64_t* kept_c, float* kept_s, uint64_t* n_peaks)
{
    const b2_search_config c = *cfg;
    std::vector<uint64_t> pk;
    for (uint64_t e = 0; e < n; e++)
        if (search_peak_rule<uint64_t>(Lc[e], Ls[e], c.nx, c.ny, c.n_yaw, [&](uint64_t q) { return bnb_find(Lc, Ls, n, q); })) pk.push_back(e);
    *n_peaks = pk.size();
    std::stable_sort(pk.begin(), pk.end(), [&](uint64_t a, uint64_t b) { return search_rank(Ls[a]) < search_rank(Ls[b]); });
    const SearchGrid g{c.x0, c.y0, c.z0, c.step, c.nx, c.ny, c.n_yaw, nullptr};
    uint32_t n_kept = 0;
    for (uint64_t e = 0; e < pk.size() && n_kept < c.max_records; e++)
        if (search_keep<uint64_t>(g, Lc[pk[e]], kept_c, n_kept, (double)c.min_separation_xy, (double)c.min_separation_yaw)) {
            kept_c[n_kept] = Lc[pk[e]]; kept_s[n_kept] = Ls[pk[e]]; n_kept++;
        }
    return n_kept;
}

// pyr_query over the cells lo .. hi (per axis) of the field's pyramid
EMUL_API float emul_bnb_query(const float* lo, const float* hi, float h, float trunc, const uint32_t* index, const float* bricks, uint64_t n_slots,
                              const uint32_t* clo, const uint32_t* chi)
{
    const DfieldView f = field_of(lo, hi, h, trunc, index, bricks);
    SearchPyr P{};
    const uint64_t n_dense = pyr_levels(f, P);
    std::vector<float> fine2(std::max<uint64_t>(1, n_slots * 64u)), fine4(std::max<uint64_t>(1, n_slots * 8u)), dense(n_dense);
    std::vector<uint64_t> off(B2_BNB_MAX_DENSE);
    emul_bnb_pyramid(lo, hi, h, trunc, index, bricks, n_slots, fine2.data(), fine4.data(), dense.data(), off.data());
    P.fine2 = fine2.data(); P.fine4 = fine4.data(); P.dense = dense.data();
    return pyr_query(P, f, clo, chi);
}
