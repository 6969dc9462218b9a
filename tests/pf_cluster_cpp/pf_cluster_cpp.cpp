// TEST PROGRAM: PCDSensorUpdaterB200::estimateClusters (include/rmcl_b200/rcc_b200.hpp) on device memory, as a node's publishStats step would
// call it.  Usage: pf_cluster_cpp IN OUT.  IN holds n (u32), then n poses (32 B) and n attributes (36 B).  OUT receives the b2_cluster_result
// record (64 B), the n_records b2_cluster_record records (472 B each) and the n labels (u32), after one call with the default
// cluster_config; tests/test_gpu_pf_cluster.py compares the file with the Python path.
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
    uint32_t hd[1];
    if (std::fread(hd, 4, 1, in) != 1) return 4;
    const size_t n = hd[0];
    std::vector<rm::Transform> hp(n);
    std::vector<rmcl::ParticleAttributes> ha(n);
    if (std::fread(hp.data(), sizeof(rm::Transform), n, in) != n || std::fread(ha.data(), sizeof(rmcl::ParticleAttributes), n, in) != n) return 4;
    std::fclose(in);
    // estimateClusters reads the particles alone: a one-triangle map serves
    const float V[9] = {0, 0, 0, 1, 0, 0, 0, 1, 0};
    const uint32_t F[3] = {0, 1, 2};
    auto map = std::make_shared<rmcl::B200Map>(V, 3u, F, 1u);
    rmcl::PCDSensorUpdaterB200 up(map);

    rm::Transform* poses = nullptr;
    rmcl::ParticleAttributes* attrs = nullptr;
    uint32_t* labels = nullptr;
    if (cudaMalloc((void**)&poses, n * sizeof(rm::Transform)) != cudaSuccess || cudaMalloc((void**)&attrs, n * sizeof(rmcl::ParticleAttributes)) != cudaSuccess ||
        cudaMalloc((void**)&labels, n * sizeof(uint32_t)) != cudaSuccess)
        return 3;
    cudaMemcpy(poses, hp.data(), n * sizeof(rm::Transform), cudaMemcpyHostToDevice);
    cudaMemcpy(attrs, ha.data(), n * sizeof(rmcl::ParticleAttributes), cudaMemcpyHostToDevice);
    cudaMemset(labels, 0, n * sizeof(uint32_t));
    rm::MemoryView<rm::Transform, rm::VRAM_CUDA> pv{poses, n};
    rm::MemoryView<rmcl::ParticleAttributes, rm::VRAM_CUDA> av{attrs, n};

    const std::vector<b2_cluster_record> recs = up.estimateClusters(pv, av, labels);
    if (recs.size() != up.last_clusters.n_records) return 5;
    std::vector<uint32_t> hl(n);
    cudaMemcpy(hl.data(), labels, n * sizeof(uint32_t), cudaMemcpyDeviceToHost);
    FILE* f = std::fopen(argv[2], "wb");
    if (!f) return 4;
    std::fwrite(&up.last_clusters, sizeof(b2_cluster_result), 1, f);
    std::fwrite(recs.data(), sizeof(b2_cluster_record), recs.size(), f);
    std::fwrite(hl.data(), sizeof(uint32_t), n, f);
    std::fclose(f);

    // a refused config throws like every other failure of the classes
    up.cluster_config.max_records = 17;
    try { up.estimateClusters(pv, av); return 6; } catch (const std::runtime_error& e) { std::printf("REFUSED %s\n", e.what()); }
    cudaFree(poses); cudaFree(attrs); cudaFree(labels);
    return cudaGetLastError() == cudaSuccess ? 0 : 7;
}
