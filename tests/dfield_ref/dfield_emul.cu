// dfield_emul.cu -- TEST HARNESS ONLY: the product's distance-field functions (rmcl_b200/csrc/kernels.cuh: df_grid, df_limits,
// df_brick_alloc, df_node_value, df_brick_node, df_lookup, pf_eval_field, pf_merge; trace.cuh: closest_point) compiled for the CPU over the
// product's host-built BVH.  The build runs the three device steps as host loops: every brick classified, slots handed out in brick order
// (the exclusive scan), every node of every allocated brick filled.  Included into the emulator library (tests/emul/emul.cu).

// grid of the box: dims_out[0..2] nodes, dims_out[3..5] bricks, origin / inv_h; returns 0, or 1 when df_grid refuses (reason in why)
EMUL_API int emul_df_grid(const float* lo, const float* hi, float h, float trunc, uint32_t* dims_out, float* inv_h, uint64_t* n_bricks, char* why, int why_cap)
{
    DfieldView f;
    const char* r = df_grid(lo, hi, h, trunc, &f, n_bricks);
    if (r) { snprintf(why, (size_t)why_cap, "%s", r); return 1; }
    dims_out[0] = f.dx; dims_out[1] = f.dy; dims_out[2] = f.dz; dims_out[3] = f.bx; dims_out[4] = f.by; dims_out[5] = f.bz; *inv_h = f.inv_h;
    return 0;
}

// the build: index (n_bricks words), bricks (capacity cap_bricks x 729 floats); returns the number of allocated bricks, or -1 if cap is short
EMUL_API int64_t emul_df_build(void* p, const float* lo, const float* hi, float h, float trunc, uint32_t* index, float* bricks, uint64_t cap_bricks)
{
    const BvhView bvh = view_of(p);
    DfieldView f; uint64_t nb = 0;
    if (df_grid(lo, hi, h, trunc, &f, &nb)) return -1;
    float ta, ta2, trunc2; df_limits(f, ta, ta2, trunc2);
    #pragma omp parallel for schedule(dynamic, 64)
    for (int64_t id = 0; id < (int64_t)nb; id++)
        index[id] = df_brick_alloc(bvh, f, (uint32_t)(id % f.bx), (uint32_t)(id / f.bx % f.by), (uint32_t)(id / f.bx / f.by), ta, ta2) ? 1u : 0u;
    std::vector<uint32_t> list;
    for (uint64_t id = 0; id < nb; id++) {
        if (index[id]) { index[id] = (uint32_t)list.size(); list.push_back((uint32_t)id); }
        else index[id] = B2_NOBRICK;
    }
    if (list.size() > cap_bricks) return -1;
    const int64_t n_nodes = (int64_t)list.size() * B2_DF_NODES;
    #pragma omp parallel for schedule(dynamic, 729)
    for (int64_t t = 0; t < n_nodes; t++) {
        uint32_t i, j, k;
        df_brick_node(f, list[t / B2_DF_NODES], (uint32_t)(t % B2_DF_NODES), i, j, k);
        bricks[t] = df_node_value(bvh, f, i, j, k, trunc2);
    }
    return (int64_t)list.size();
}

EMUL_API void emul_df_lookup(const float* lo, const float* hi, float h, float trunc, const uint32_t* index, const float* bricks, const float* pts, uint32_t n, float* out)
{
    const DfieldView f = field_of(lo, hi, h, trunc, index, bricks);
    #pragma omp parallel for schedule(static)
    for (int64_t i = 0; i < (int64_t)n; i++) out[i] = df_lookup(f, mk3(pts[3 * i], pts[3 * i + 1], pts[3 * i + 2]));
}

// closest point at n points, bounded (trunc2 = fl(trunc^2)) or not: d2 and face per point
EMUL_API void emul_df_closest(void* p, const float* pts, uint32_t n, int bounded, float trunc2, float* d2, uint32_t* face)
{
    const BvhView bvh = view_of(p);
    #pragma omp parallel for schedule(dynamic, 256)
    for (int64_t i = 0; i < (int64_t)n; i++) {
        CpBest best; uint32_t nn = 0, nt = 0;
        const V3 q = mk3(pts[3 * i], pts[3 * i + 1], pts[3 * i + 2]);
        if (bounded) closest_point<false, true>(bvh, q, best, nn, nt, trunc2);
        else closest_point<false>(bvh, q, best, nn, nt);
        d2[i] = best.d2; face[i] = best.face;
    }
}

// the sensor update from the field of k_pf_update_field, per particle: evaluations in beam order, merged with pf_merge
EMUL_API void emul_df_pf_update(const float* lo, const float* hi, float h, float trunc, const uint32_t* index, const float* bricks, const b2_transform* poses,
                                b2_particle_attr* attrs, uint32_t n, const b2_transform* Tsb_val, const b2_range_meas* beams, uint32_t n_beams, const b2_pf_params* prm)
{
    const DfieldView f = field_of(lo, hi, h, trunc, index, bricks);
    float sigma_quad; double denom; pf_constants(*prm, sigma_quad, denom);
    const Tf Tsb = tf_from_pod(*Tsb_val);
    #pragma omp parallel for schedule(dynamic, 64)
    for (int64_t i = 0; i < (int64_t)n; i++) {
        std::vector<float> e(n_beams);
        const Tf Tsm = tf_mul(tf_load(poses + i), Tsb);
        for (uint32_t b = 0; b < n_beams; b++) {
            const b2_range_meas& m = beams[b];
            const PfBeam pb{m.orig.x, m.orig.y, m.orig.z, m.dir.x, m.dir.y, m.dir.z, m.range, b};
            e[b] = pf_eval_field(f, Tsm, pb, sigma_quad, denom);
        }
        b2_gaussian1d lk = attrs[i].likelihood;
        pf_merge(lk, e.data(), n_beams);
        attrs[i].likelihood = lk;
    }
}
