// recovery_emul.cu -- TEST HARNESS ONLY: the product's per-particle function of b2_pf_recovery_inject (rmcl_b200/csrc/kernels.cuh:
// pf_recovery_one, with pf_box_pose, pf_surface_pose and the tracer inlined) compiled for the CPU over the product's host-built BVH, run for
// every particle of a slice as k_pf_recovery_inject runs it, and the record's update pf_recovery_filter.  The surface constants are computed
// as b2_pf_recovery_inject computes them.  Included into the emulator library (tests/emul/emul.cu).

// cfg == nullptr: no surface.  counts[0] += replaced, counts[1] += failed
EMUL_API void emul_pf_recovery(void* p, const b2_surface_config* cfg, uint32_t first, uint32_t n, double p_inject, const float* lo, const float* hi,
                               uint32_t max_tries, uint64_t seed, uint32_t step, b2_transform* poses, b2_particle_attr* attrs, uint64_t* counts)
{
    const BvhView v = view_of(p);
    const b2_surface_config c = cfg ? *cfg : b2_surface_config{};
    const float cos_max = cfg ? (float)std::cos((double)c.max_slope) : 0.0f, tfar = cfg ? c.probe_above + c.probe_below : 0.0f;
    PfInitBox box;
    for (int k = 0; k < 6; k++) { box.lo[k] = lo[k]; box.hi[k] = hi[k]; }
    uint64_t n_rep = 0, n_fail = 0;
    #pragma omp parallel for schedule(dynamic, 256) reduction(+ : n_rep, n_fail)
    for (int64_t i = 0; i < (int64_t)n; i++) {
        const uint32_t w = pf_recovery_one(cfg ? &v : nullptr, poses + i, attrs + i, first + (uint32_t)i, p_inject, box, c, cos_max, tfar, max_tries, seed, step);
        n_rep += w == B2_RECOVERY_REPLACED; n_fail += w == B2_RECOVERY_FAILED;
    }
    counts[0] += n_rep; counts[1] += n_fail;
}
EMUL_API void emul_recovery_filter(double S, uint32_t n, double alpha_slow, double alpha_fast, b2_recovery_state* st)
{
    pf_recovery_filter(S, n, alpha_slow, alpha_fast, st);
}
