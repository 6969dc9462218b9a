// surface_emul.cu -- TEST HARNESS ONLY: the product's per-particle function of b2_pf_project_to_surface (rmcl_b200/csrc/kernels.cuh:
// pf_surface_one, with trace_closest, tri_ng and the quaternion helpers inlined) compiled for the CPU over the product's host-built BVH, and
// run for every particle as k_pf_surface runs it.  The two constants are computed as b2_pf_project_to_surface computes them.
// Included into the emulator library (tests/emul/emul.cu).

EMUL_API void emul_pf_surface(void* p, b2_transform* poses, b2_particle_attr* attrs, uint32_t n, const b2_surface_config* cfg)
{
    const BvhView v = view_of(p);
    const float cos_max = (float)std::cos((double)cfg->max_slope), tfar = cfg->probe_above + cfg->probe_below;
    #pragma omp parallel for schedule(dynamic, 256)
    for (int64_t i = 0; i < (int64_t)n; i++) pf_surface_one(v, poses + i, attrs + i, *cfg, cos_max, tfar);
}
