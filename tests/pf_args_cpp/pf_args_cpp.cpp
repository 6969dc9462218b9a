// TEST PROGRAM: the argument check of PCDSensorUpdaterB200 (include/rmcl_b200/rcc_b200.hpp).  Every entry point that passes one count for
// poses and attributes is called once with views one attribute short, which must throw std::invalid_argument with no kernel launched, and
// once with views that agree, which must run.  Prints one line per call (REFUSED / RAN name) and exits 0 when every call behaved;
// tests/test_gpu_binding_args.py checks the lines.
#include <cstdio>
#include <stdexcept>
#include <vector>

#include <cuda_runtime.h>
#include <rmcl_b200/rcc_b200.hpp>

namespace rm = rmagine;

static int failures = 0;

template <typename F> static void refused(const char* name, F call)
{
    const uint64_t before = b2_kernel_launch_count();
    try {
        call();
        std::printf("FAIL %s: views of different sizes were accepted\n", name);
    } catch (const std::invalid_argument& e) {
        if (b2_kernel_launch_count() == before) { std::printf("REFUSED %s: %s\n", name, e.what()); return; }
        std::printf("FAIL %s: refused after a launch\n", name);
    } catch (const std::exception& e) {
        std::printf("FAIL %s: %s\n", name, e.what());
    }
    failures++;
}

template <typename F> static void runs(const char* name, F call)
{
    try {
        call();
        std::printf("RAN %s\n", name);
    } catch (const std::exception& e) {
        std::printf("FAIL %s: %s\n", name, e.what());
        failures++;
    }
}

int main()
{
    const std::vector<float> V = {-10, -10, 0, 10, -10, 0, 0, 10, 0};
    const std::vector<uint32_t> F = {0, 1, 2};
    auto map = std::make_shared<rmcl::B200Map>(V.data(), 3u, F.data(), 1u);
    auto field = std::make_shared<rmcl::B200DistanceField>(map, 0.25f, 1.0f);
    rmcl::PCDSensorUpdaterB200 up(map);
    rmcl::RangeMeasurement beam{{0.f, 0.f, 1.f}, {0.f, 0.f, -1.f}, 1.f, {}};
    up.setBeams(std::vector<rmcl::RangeMeasurement>(4, beam));

    const size_t n = 64;
    std::vector<rm::Transform> hp(n, rm::Transform::Identity());
    std::vector<rmcl::ParticleAttributes> ha(n);
    for (size_t i = 0; i < n; i++) { hp[i].t = {0.1f * float(i % 8), 0.1f * float(i / 8), 1.f}; ha[i] = rmcl::ParticleAttributes{{0.5f, 0.1f, 1u}, {}}; }
    rm::Transform* poses = nullptr; rmcl::ParticleAttributes* attrs = nullptr; rm::Transform* poses_new = nullptr; rmcl::ParticleAttributes* attrs_new = nullptr;
    if (cudaMalloc((void**)&poses, n * sizeof(rm::Transform)) != cudaSuccess || cudaMalloc((void**)&attrs, n * sizeof(rmcl::ParticleAttributes)) != cudaSuccess ||
        cudaMalloc((void**)&poses_new, n * sizeof(rm::Transform)) != cudaSuccess || cudaMalloc((void**)&attrs_new, n * sizeof(rmcl::ParticleAttributes)) != cudaSuccess)
        return 3;
    cudaMemcpy(poses, hp.data(), n * sizeof(rm::Transform), cudaMemcpyHostToDevice);
    cudaMemcpy(attrs, ha.data(), n * sizeof(rmcl::ParticleAttributes), cudaMemcpyHostToDevice);

    using PV = rm::MemoryView<rm::Transform, rm::VRAM_CUDA>;
    using AV = rm::MemoryView<rmcl::ParticleAttributes, rm::VRAM_CUDA>;
    const PV P{poses, n}, Pn{poses_new, n};
    const AV A{attrs, n}, An{attrs_new, n}, A_short{attrs, n - 1}, An_short{attrs_new, n - 1};
    const rm::MemoryView<rm::Transform, rm::RAM> hP{hp.data(), n};
    const rm::MemoryView<rmcl::ParticleAttributes, rm::RAM> hA{ha.data(), n}, hA_short{ha.data(), n - 1};
    const std::array<double, 6> lo{-1, -1, 1, 0, 0, -3}, hi{1, 1, 1, 0, 0, 3};
    const std::array<double, 36> cov{0.01, 0, 0, 0, 0, 0, 0, 0.01, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0.01};

    refused("update RAM", [&] { up.update(hP, hA_short); });
    runs("update RAM", [&] { up.update(hP, hA); });
    refused("update VRAM", [&] { up.update(P, A_short); });
    runs("update VRAM", [&] { up.update(P, A); });
    up.setDistanceField(field);
    refused("update field", [&] { up.update(P, A_short); });
    runs("update field", [&] { up.update(P, A); });
    up.setDistanceField(nullptr);
    refused("motionUpdate", [&] { up.motionUpdate(P, A_short, rm::Transform::Identity(), 0.01); });
    runs("motionUpdate", [&] { up.motionUpdate(P, A, rm::Transform::Identity(), 0.01); });
    refused("projectToSurface", [&] { up.projectToSurface(P, A_short); });
    runs("projectToSurface", [&] { up.projectToSurface(P, A); });
    cudaMemcpy(attrs, ha.data(), n * sizeof(rmcl::ParticleAttributes), cudaMemcpyHostToDevice);
    refused("resample all", [&] { up.resample(P, A_short, Pn, An); });
    refused("resample new", [&] { up.resample(P, A, Pn, An_short); });
    runs("resample", [&] { up.resample(P, A, Pn, An); });
    refused("resampleResidual all", [&] { up.resampleResidual(P, A_short, Pn, An); });
    refused("resampleResidual new", [&] { up.resampleResidual(P, A, Pn, An_short); });
    runs("resampleResidual", [&] { up.resampleResidual(P, A, Pn, An); });
    up.kld_config.n_min = 16;                                                   // at most the n slots of the output
    refused("resampleKLD all", [&] { up.resampleKLD(P, A_short, Pn, An); });
    refused("resampleKLD new", [&] { up.resampleKLD(P, A, Pn, An_short); });
    runs("resampleKLD", [&] { up.resampleKLD(P, A, Pn, An); });
    refused("initSamplesUniform", [&] { up.initSamplesUniform(P, A_short, lo, hi, 7); });
    runs("initSamplesUniform", [&] { up.initSamplesUniform(P, A, lo, hi, 7); });
    refused("initSamples", [&] { up.initSamples(P, A_short, rm::Transform::Identity(), cov, 7); });
    runs("initSamples", [&] { up.initSamples(P, A, rm::Transform::Identity(), cov, 7); });
    cudaMemcpy(attrs, ha.data(), n * sizeof(rmcl::ParticleAttributes), cudaMemcpyHostToDevice);
    refused("estimateStats", [&] { up.estimateStats(P, A_short); });
    runs("estimateStats", [&] { up.estimateStats(P, A); });
    refused("estimateClusters", [&] { up.estimateClusters(P, A_short); });
    runs("estimateClusters", [&] { up.estimateClusters(P, A); });
    up.recoveryReset();
    refused("recoveryInject", [&] { up.recoveryInject(P, A_short, lo, hi); });
    runs("recoveryInject", [&] { up.recoveryInject(P, A, lo, hi); });

    const bool clean = cudaDeviceSynchronize() == cudaSuccess && cudaGetLastError() == cudaSuccess;
    cudaFree(poses); cudaFree(attrs); cudaFree(poses_new); cudaFree(attrs_new);
    return failures ? 1 : clean ? 0 : 4;
}
