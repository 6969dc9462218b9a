// surface_emul.cu -- TEST HARNESS ONLY: the product's per-particle function of b2_pf_project_to_surface (rmcl_b200/csrc/kernels.cuh:
// pf_surface_one, with trace_closest, tri_ng and the quaternion helpers inlined) compiled for the CPU over the product's host-built BVH, and
// run for every particle as k_pf_surface runs it.  The two constants are computed as b2_pf_project_to_surface computes them.  Built by
// tests/pf_surface_ref.py with the flags of tests/chain_ref (host code with -ffp-contract=off: plain ops rounded like __fmul_rn etc.).
#include "../../rmcl_b200/csrc/kernels.cuh"

#include <cmath>

#define EMUL_API extern "C" __attribute__((visibility("default")))

EMUL_API void* emul_surface_scene(const float* verts, uint32_t nv, const uint32_t* faces, uint32_t nf)
{
    B2BvhHost* b = new B2BvhHost();
    const char* err = "";
    if (b2_build_bvh8_host(verts, nv, faces, nf, b, &err) != 0) { delete b; return nullptr; }
    return b;
}
EMUL_API void emul_surface_scene_free(void* p)
{
    if (p) { b2_free_bvh8_host((B2BvhHost*)p); delete (B2BvhHost*)p; }
}
EMUL_API void emul_pf_surface(void* p, b2_transform* poses, b2_particle_attr* attrs, uint32_t n, const b2_surface_config* cfg)
{
    const B2BvhHost* b = (const B2BvhHost*)p;
    BvhView v; v.nodes = (const float4*)b->nodes; v.tris = (const float4*)b->tris;
    v.bx = b->abs_max[0]; v.by = b->abs_max[1]; v.bz = b->abs_max[2];
    const float cos_max = (float)std::cos((double)cfg->max_slope), tfar = cfg->probe_above + cfg->probe_below;
    #pragma omp parallel for schedule(dynamic, 256)
    for (int64_t i = 0; i < (int64_t)n; i++) pf_surface_one(v, poses + i, attrs + i, *cfg, cos_max, tfar);
}
