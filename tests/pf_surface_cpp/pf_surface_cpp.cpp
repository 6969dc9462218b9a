// TEST PROGRAM: PCDSensorUpdaterB200::projectToSurface (include/rmcl_b200/rcc_b200.hpp) on device memory, as a node's motion update would
// call it.  Usage: pf_surface_cpp IN OUT.  IN holds nv, nf, n (u32 each), then nv x 3 floats, nf x 3 u32, n poses (32 B) and n attributes
// (36 B).  OUT receives the particles after projectToSurface with surface_config(), then after a second call with align 0 and base_height
// 0.25, each as n poses followed by n attributes; tests/test_gpu_pf_surface.py compares the file with the Python path.
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
    uint32_t hd[3];
    if (std::fread(hd, 4, 3, in) != 3) return 4;
    const size_t nv = hd[0], nf = hd[1], n = hd[2];
    std::vector<float> V(3 * nv);
    std::vector<uint32_t> F(3 * nf);
    std::vector<rm::Transform> hp(n);
    std::vector<rmcl::ParticleAttributes> ha(n);
    if (std::fread(V.data(), 4, V.size(), in) != V.size() || std::fread(F.data(), 4, F.size(), in) != F.size() ||
        std::fread(hp.data(), sizeof(rm::Transform), n, in) != n || std::fread(ha.data(), sizeof(rmcl::ParticleAttributes), n, in) != n)
        return 4;
    std::fclose(in);
    auto map = std::make_shared<rmcl::B200Map>(V.data(), (uint32_t)nv, F.data(), (uint32_t)nf);
    rmcl::PCDSensorUpdaterB200 up(map);

    rm::Transform* poses = nullptr; rmcl::ParticleAttributes* attrs = nullptr;
    if (cudaMalloc((void**)&poses, n * sizeof(rm::Transform)) != cudaSuccess || cudaMalloc((void**)&attrs, n * sizeof(rmcl::ParticleAttributes)) != cudaSuccess) return 3;
    cudaMemcpy(poses, hp.data(), n * sizeof(rm::Transform), cudaMemcpyHostToDevice);
    cudaMemcpy(attrs, ha.data(), n * sizeof(rmcl::ParticleAttributes), cudaMemcpyHostToDevice);
    rm::MemoryView<rm::Transform, rm::VRAM_CUDA> pv{poses, n};
    rm::MemoryView<rmcl::ParticleAttributes, rm::VRAM_CUDA> av{attrs, n};
    FILE* f = std::fopen(argv[2], "wb");
    if (!f) return 4;
    auto dump = [&]() {
        cudaDeviceSynchronize();
        cudaMemcpy(hp.data(), poses, n * sizeof(rm::Transform), cudaMemcpyDeviceToHost);
        cudaMemcpy(ha.data(), attrs, n * sizeof(rmcl::ParticleAttributes), cudaMemcpyDeviceToHost);
        std::fwrite(hp.data(), sizeof(rm::Transform), n, f); std::fwrite(ha.data(), sizeof(rmcl::ParticleAttributes), n, f);
    };
    up.projectToSurface(pv, av);                                   // after motionUpdate (rmcl_localization.cpp:432-480)
    dump();
    b2_surface_config cfg = rmcl::PCDSensorUpdaterB200::surface_config();
    cfg.align = 0; cfg.base_height = 0.25f;
    up.projectToSurface(pv, av, cfg);
    dump();
    std::fclose(f);

    // a refused config throws like every other failure of the classes
    cfg.max_slope = 2.0f;
    try { up.projectToSurface(pv, av, cfg); return 5; } catch (const std::runtime_error& e) { std::printf("REFUSED %s\n", e.what()); }
    cudaFree(poses); cudaFree(attrs);
    return cudaGetLastError() == cudaSuccess ? 0 : 6;
}
