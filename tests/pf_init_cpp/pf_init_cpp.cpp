// TEST PROGRAM: PCDSensorUpdaterB200::initSamplesUniform / initSamples (include/rmcl_b200/rcc_b200.hpp) on device memory, as a node's two
// initialisation callbacks would call them.  Usage: pf_init_cpp OUT N FIRST SEED.  Writes the N uniform particles, then the N Gaussian ones,
// each as N poses (32 B) followed by N attributes (36 B); tests/test_gpu_pf_init.py compares the file with the Python path.
#include <cstdio>
#include <cstdlib>
#include <vector>

#include <cuda_runtime.h>
#include <rmcl_b200/rcc_b200.hpp>

namespace rm = rmagine;

int main(int argc, char** argv)
{
    if (argc != 5) { std::fprintf(stderr, "usage: %s OUT N FIRST SEED\n", argv[0]); return 2; }
    const size_t n = std::strtoul(argv[2], nullptr, 10);
    const uint32_t first = (uint32_t)std::strtoul(argv[3], nullptr, 10);
    const uint64_t seed = std::strtoull(argv[4], nullptr, 10);
    const std::vector<float> V = {0, 0, 0, 1, 0, 0, 0, 1, 0};
    const std::vector<uint32_t> F = {0, 1, 2};
    auto map = std::make_shared<rmcl::B200Map>(V.data(), 3u, F.data(), 1u);
    rmcl::PCDSensorUpdaterB200 up(map);

    rm::Transform* poses = nullptr; rmcl::ParticleAttributes* attrs = nullptr;
    if (cudaMalloc((void**)&poses, n * sizeof(rm::Transform)) != cudaSuccess || cudaMalloc((void**)&attrs, n * sizeof(rmcl::ParticleAttributes)) != cudaSuccess) return 3;
    rm::MemoryView<rm::Transform, rm::VRAM_CUDA> pv{poses, n};
    rm::MemoryView<rmcl::ParticleAttributes, rm::VRAM_CUDA> av{attrs, n};
    std::vector<rm::Transform> hp(n);
    std::vector<rmcl::ParticleAttributes> ha(n);
    FILE* f = std::fopen(argv[1], "wb");
    if (!f) return 4;

    // global localisation (rmcl_localization.cpp:61-68, :110)
    up.initSamplesUniform(pv, av, {-5.0, -4.0, 0.5, -0.1, 0.0, -3.14159265358979}, {5.0, 4.0, 0.5, 0.1, 0.0, 3.14159265358979}, seed, first);
    cudaMemcpy(hp.data(), poses, n * sizeof(rm::Transform), cudaMemcpyDeviceToHost);
    cudaMemcpy(ha.data(), attrs, n * sizeof(rmcl::ParticleAttributes), cudaMemcpyDeviceToHost);
    std::fwrite(hp.data(), sizeof(rm::Transform), n, f); std::fwrite(ha.data(), sizeof(rmcl::ParticleAttributes), n, f);

    // /initialpose (rmcl_localization.cpp:54-58): rviz's covariance
    rm::Transform pose = rm::Transform::Identity();
    pose.t = {2.0f, -1.0f, 0.0f}; pose.R = {0.0f, 0.0f, 0.38268343f, 0.92387953f};
    std::array<double, 36> cov{};
    cov[0] = 0.25; cov[7] = 0.25; cov[35] = 0.06853891909122467;
    up.initSamples(pv, av, pose, cov, seed, first);
    cudaMemcpy(hp.data(), poses, n * sizeof(rm::Transform), cudaMemcpyDeviceToHost);
    cudaMemcpy(ha.data(), attrs, n * sizeof(rmcl::ParticleAttributes), cudaMemcpyDeviceToHost);
    std::fwrite(hp.data(), sizeof(rm::Transform), n, f); std::fwrite(ha.data(), sizeof(rmcl::ParticleAttributes), n, f);
    std::fclose(f);

    // a refused covariance throws like every other failure of the classes
    cov[14] = -1.0;
    try { up.initSamples(pv, av, pose, cov, seed, first); return 5; } catch (const std::runtime_error& e) { std::printf("REFUSED %s\n", e.what()); }
    cudaFree(poses); cudaFree(attrs);
    return cudaGetLastError() == cudaSuccess ? 0 : 6;
}
