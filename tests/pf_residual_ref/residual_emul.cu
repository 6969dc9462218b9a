// residual_emul.cu -- TEST HARNESS ONLY: the product's per-element functions of residual resampling (rmcl_b200/csrc/kernels.cuh:
// residual_parent, residual_count, residual_normals, residual_copy) compiled for the CPU, so that they can be compared with the C
// restatement in a container without a GPU.  Built by tests/pf_residual_ref.py with the flags of tests/chain_ref (host code with
// -ffp-contract=off: plain float ops rounded like __fmul_rn / __fadd_rn).
#include "../../rmcl_b200/csrc/kernels.cuh"

#define EMUL_API extern "C" __attribute__((visibility("default")))

EMUL_API void emul_residual_parents(uint64_t seed, uint32_t step, uint64_t d0, uint64_t count, uint32_t n, uint32_t* out)
{
    for (uint64_t i = 0; i < count; i++) out[i] = residual_parent(seed, step, d0 + i, n);
}
// the counts of draws whose parents' likelihoods are L[0 .. count-1]
EMUL_API void emul_residual_counts(const float* L, uint64_t count, double S, uint64_t M, uint64_t* out)
{
    for (uint64_t i = 0; i < count; i++) out[i] = residual_count(L[i], S, M);
}
EMUL_API void emul_residual_normals(uint64_t seed, uint32_t step, uint32_t first, uint32_t count, float* out)
{
    for (uint32_t i = 0; i < count; i++) residual_normals(seed, step, first + i, out + 6 * (size_t)i);
}
// copy i of parent parents[i] with normals N[6 i .. 6 i + 5]
EMUL_API void emul_residual_copies(const b2_transform* poses, const b2_particle_attr* attrs, const uint32_t* parents, const float* N, uint32_t count, double L_max,
                                   const b2_gladiator_config* cfg, b2_transform* out_p, b2_particle_attr* out_a)
{
    for (uint32_t i = 0; i < count; i++) residual_copy(poses[parents[i]], attrs[parents[i]], L_max, N + 6 * (size_t)i, *cfg, out_p + i, out_a + i);
}
