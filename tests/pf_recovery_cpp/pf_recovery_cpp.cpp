// TEST PROGRAM: the recovery of PCDSensorUpdaterB200 (include/rmcl_b200/rcc_b200.hpp: recoveryReset, recoveryObserve, recoveryInject) on
// device memory, as a node's cycle would call it.  Usage: pf_recovery_cpp IN OUT.  IN holds nv, nf, n (u32 each), the box bb_min, bb_max
// (6 doubles each), then nv x 3 floats, nf x 3 u32, n poses (32 B) and n attributes (36 B).  With recovery_config {0, 1}, two observes of
// n attributes of likelihood 1.0 and then 0.7 set p_inject = 0.3; recoveryInject with surface_config(), max_tries 16, seed 99, step 2
// follows.  OUT receives last_recovery_state (32 B), last_recovery (24 B), then the n poses and n attributes;
// tests/test_gpu_pf_recovery.py compares the file with the Python path.
#include <array>
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
    std::array<double, 6> lo, hi;
    if (std::fread(hd, 4, 3, in) != 3 || std::fread(lo.data(), 8, 6, in) != 6 || std::fread(hi.data(), 8, 6, in) != 6) return 4;
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

    rm::Transform* poses = nullptr; rmcl::ParticleAttributes *attrs = nullptr, *obs = nullptr;
    if (cudaMalloc((void**)&poses, n * sizeof(rm::Transform)) != cudaSuccess || cudaMalloc((void**)&attrs, n * sizeof(rmcl::ParticleAttributes)) != cudaSuccess ||
        cudaMalloc((void**)&obs, n * sizeof(rmcl::ParticleAttributes)) != cudaSuccess) return 3;
    cudaMemcpy(poses, hp.data(), n * sizeof(rm::Transform), cudaMemcpyHostToDevice);
    cudaMemcpy(attrs, ha.data(), n * sizeof(rmcl::ParticleAttributes), cudaMemcpyHostToDevice);
    rm::MemoryView<rm::Transform, rm::VRAM_CUDA> pv{poses, n};
    rm::MemoryView<rmcl::ParticleAttributes, rm::VRAM_CUDA> av{attrs, n}, ov{obs, n};
    std::vector<rmcl::ParticleAttributes> ho(n);
    auto observe = [&](float mean, bool want) {
        for (auto& a : ho) { a = rmcl::ParticleAttributes{}; a.likelihood.mean = mean; }
        cudaMemcpy(obs, ho.data(), n * sizeof(rmcl::ParticleAttributes), cudaMemcpyHostToDevice);
        up.recoveryObserve(ov, want);                              // after update (rmcl_localization.cpp's sensor update step)
    };
    up.recovery_config = b2_recovery_config{0.0, 1.0};
    up.recoveryReset();
    observe(1.0f, false);
    observe(0.7f, true);
    const b2_surface_config surface = rmcl::PCDSensorUpdaterB200::surface_config();
    up.recoveryInject(pv, av, lo, hi, &surface, 16, 99, 2, 0, true);   // after resampling
    cudaDeviceSynchronize();
    cudaMemcpy(hp.data(), poses, n * sizeof(rm::Transform), cudaMemcpyDeviceToHost);
    cudaMemcpy(ha.data(), attrs, n * sizeof(rmcl::ParticleAttributes), cudaMemcpyDeviceToHost);
    FILE* f = std::fopen(argv[2], "wb");
    if (!f) return 4;
    std::fwrite(&up.last_recovery_state, sizeof(b2_recovery_state), 1, f);
    std::fwrite(&up.last_recovery, sizeof(b2_recovery_result), 1, f);
    std::fwrite(hp.data(), sizeof(rm::Transform), n, f); std::fwrite(ha.data(), sizeof(rmcl::ParticleAttributes), n, f);
    std::fclose(f);

    // a refused setting throws like every other failure of the classes
    try { up.recoveryInject(pv, av, lo, hi, &surface, 0); return 5; } catch (const std::runtime_error& e) { std::printf("REFUSED %s\n", e.what()); }
    cudaFree(poses); cudaFree(attrs); cudaFree(obs);
    return cudaGetLastError() == cudaSuccess ? 0 : 6;
}
