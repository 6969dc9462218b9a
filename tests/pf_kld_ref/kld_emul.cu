// kld_emul.cu -- TEST HARNESS ONLY: the product's per-element functions of KLD-sampling (rmcl_b200/csrc/kernels.cuh: kld_weight,
// kld_parent, kld_key, kld_bound, kld_stop) compiled for the CPU, so that they can be compared with the C restatement in a container without
// a GPU.  Included into the emulator library (tests/emul/emul.cu).

// the inclusive prefix of the integer weights of L[0 .. n-1]
EMUL_API void emul_kld_prefix(const float* L, uint32_t n, double L_max, unsigned long long* W)
{
    unsigned long long s = 0;
    for (uint32_t i = 0; i < n; i++) { s += kld_weight(L[i], L_max); W[i] = s; }
}
EMUL_API void emul_kld_parents(uint64_t seed, uint32_t step, uint64_t d0, uint64_t count, const unsigned long long* W, uint32_t n, uint32_t* out)
{
    for (uint64_t i = 0; i < count; i++) out[i] = kld_parent(seed, step, d0 + i, W, n);
}
EMUL_API void emul_kld_keys(const b2_transform* poses, uint64_t count, float res_xy, float res_z, const float* cs, uint32_t K, uint64_t* out)
{
    const KldBins b{res_xy, res_z, K, cs};
    for (uint64_t i = 0; i < count; i++) out[i] = kld_key(poses[i], b);
}
EMUL_API void emul_kld_bounds(const uint64_t* k, uint64_t count, double epsilon, double z, uint32_t n_min, uint64_t* out)
{
    for (uint64_t i = 0; i < count; i++) out[i] = kld_bound(k[i], epsilon, z, n_min);
}
// the stop rule at draw j[i] with k[i] bins
EMUL_API void emul_kld_stop(const uint64_t* j, const uint64_t* k, uint64_t count, double epsilon, double z, uint32_t n_min, uint64_t n_max, uint8_t* out)
{
    for (uint64_t i = 0; i < count; i++) out[i] = kld_stop(j[i], k[i], epsilon, z, n_min, n_max) ? 1 : 0;
}
