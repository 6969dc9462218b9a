// TEST PROGRAM: PCDSensorUpdaterB200::resampleKLD (include/rmcl_b200/rcc_b200.hpp) on device memory, as a node's resampling step would call
// it.  Usage: pf_kld_cpp IN OUT.  IN holds n, n_max (u32 each), then n poses (32 B) and n attributes (36 B).  OUT receives the b2_kld_result
// record (32 B), then the n_max output slots (zero-filled before the call) as n_max poses followed by n_max attributes, after one call with
// the default kld_config and resampler_config, seed 77, step 3; tests/test_gpu_pf_kld.py compares the file with the Python path.
#include <cstdio>
#include <cstdlib>
#include <vector>

#include <cuda_runtime.h>
#include <rmcl_b200/rcc_b200.hpp>

namespace rm = rmagine;

int main(int argc, char** argv)
{
    if (argc != 3) { std::fprintf(stderr, "usage: %s IN OUT\n", argv[0]); return 2; }
    FILE* in = std::fopen(argv[1], "rb");
    if (!in) return 4;
    uint32_t hd[2];
    if (std::fread(hd, 4, 2, in) != 2) return 4;
    const size_t n = hd[0], n_max = hd[1];
    std::vector<rm::Transform> hp(n);
    std::vector<rmcl::ParticleAttributes> ha(n);
    if (std::fread(hp.data(), sizeof(rm::Transform), n, in) != n || std::fread(ha.data(), sizeof(rmcl::ParticleAttributes), n, in) != n) return 4;
    std::fclose(in);
    // resampleKLD draws on the particles alone: a one-triangle map serves
    const float V[9] = {0, 0, 0, 1, 0, 0, 0, 1, 0};
    const uint32_t F[3] = {0, 1, 2};
    auto map = std::make_shared<rmcl::B200Map>(V, 3u, F, 1u);
    rmcl::PCDSensorUpdaterB200 up(map);

    rm::Transform *poses = nullptr, *poses_new = nullptr;
    rmcl::ParticleAttributes *attrs = nullptr, *attrs_new = nullptr;
    if (cudaMalloc((void**)&poses, n * sizeof(rm::Transform)) != cudaSuccess || cudaMalloc((void**)&attrs, n * sizeof(rmcl::ParticleAttributes)) != cudaSuccess ||
        cudaMalloc((void**)&poses_new, n_max * sizeof(rm::Transform)) != cudaSuccess ||
        cudaMalloc((void**)&attrs_new, n_max * sizeof(rmcl::ParticleAttributes)) != cudaSuccess)
        return 3;
    cudaMemcpy(poses, hp.data(), n * sizeof(rm::Transform), cudaMemcpyHostToDevice);
    cudaMemcpy(attrs, ha.data(), n * sizeof(rmcl::ParticleAttributes), cudaMemcpyHostToDevice);
    cudaMemset(poses_new, 0, n_max * sizeof(rm::Transform));
    cudaMemset(attrs_new, 0, n_max * sizeof(rmcl::ParticleAttributes));
    rm::MemoryView<rm::Transform, rm::VRAM_CUDA> pv{poses, n}, pnv{poses_new, n_max};
    rm::MemoryView<rmcl::ParticleAttributes, rm::VRAM_CUDA> av{attrs, n}, anv{attrs_new, n_max};

    const rmcl::ParticleUpdateDynamicResults res = up.resampleKLD(pv, av, pnv, anv, 77, 3);     // the node's resampling() (rmcl_localization.cpp:596-639)
    if (res.n_particles != up.last_kld.n_particles) return 5;
    std::vector<rm::Transform> op(n_max);
    std::vector<rmcl::ParticleAttributes> oa(n_max);
    cudaMemcpy(op.data(), poses_new, n_max * sizeof(rm::Transform), cudaMemcpyDeviceToHost);
    cudaMemcpy(oa.data(), attrs_new, n_max * sizeof(rmcl::ParticleAttributes), cudaMemcpyDeviceToHost);
    FILE* f = std::fopen(argv[2], "wb");
    if (!f) return 4;
    std::fwrite(&up.last_kld, sizeof(b2_kld_result), 1, f);
    std::fwrite(op.data(), sizeof(rm::Transform), n_max, f); std::fwrite(oa.data(), sizeof(rmcl::ParticleAttributes), n_max, f);
    std::fclose(f);

    // a refused config throws like every other failure of the classes
    up.kld_config.n_min = 0;
    try { up.resampleKLD(pv, av, pnv, anv, 77, 3); return 6; } catch (const std::runtime_error& e) { std::printf("REFUSED %s\n", e.what()); }
    cudaFree(poses); cudaFree(attrs); cudaFree(poses_new); cudaFree(attrs_new);
    return cudaGetLastError() == cudaSuccess ? 0 : 7;
}
