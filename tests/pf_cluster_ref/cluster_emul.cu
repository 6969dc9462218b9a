// cluster_emul.cu -- TEST HARNESS ONLY: the product's bin-neighbour functions of b2_pf_cluster_stats (rmcl_b200/csrc/kernels.cuh:
// kld_key_neighbour, kld_key_offset) compiled for the CPU, so that they can be compared with the C restatement in a container without a GPU.
// Included into the emulator library (tests/emul/emul.cu).

EMUL_API void emul_cluster_neighbours(const uint64_t* keys, uint64_t count, int dx, int dy, int dz, int ds, uint32_t K, int has_z, uint64_t* out)
{
    for (uint64_t i = 0; i < count; i++) out[i] = kld_key_neighbour(keys[i], dx, dy, dz, ds, K, has_z != 0);
}
// the 81 (27 when z is not binned) keys k_pf_cluster_hook visits around each bin, the bin itself included: out[count][81 or 27]
EMUL_API void emul_cluster_offsets(const uint64_t* keys, uint64_t count, uint32_t K, int has_z, uint64_t* out)
{
    const uint32_t n_off = has_z ? 81u : 27u;
    for (uint64_t i = 0; i < count; i++)
        for (uint32_t o = 0; o < n_off; o++) out[i * n_off + o] = kld_key_offset(keys[i], o, K, has_z != 0);
}
