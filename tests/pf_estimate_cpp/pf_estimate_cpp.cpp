// TEST PROGRAM: PCDSensorUpdaterB200::estimateStats (include/rmcl_b200/rcc_b200.hpp) and rmcl::b200::fillParticleStats
// (rmcl_msgs_adapters.hpp) as RmclNode::resampling would call them: the induction slice of a device particle set in, a message-shaped
// stand-in for rmcl_msgs::msg::ParticleStats out.  Usage: pf_estimate_cpp PARTICLES OUT K.  PARTICLES holds N poses (32 B) then N attributes
// (36 B); the program estimates over the first K and writes the message's fields as doubles in b2_particle_stats order (nparticles as
// uint64 last); tests/test_gpu_pf_estimate.py compares the file with the Python path byte for byte.
#include <array>
#include <cstdio>
#include <cstdlib>
#include <vector>

#include <cuda_runtime.h>
#include <rmcl_b200/rmcl_msgs_adapters.hpp>

namespace rm = rmagine;

// the field names of rmcl_msgs/ParticleStats, geometry_msgs/PoseWithCovariance, geometry_msgs/Point and rmcl_msgs/LikelihoodStats
struct PointMsg { double x = 0, y = 0, z = 0; };
struct QuatMsg { double x = 0, y = 0, z = 0, w = 0; };
struct PoseMsg { PointMsg position; QuatMsg orientation; };
struct PoseWithCovarianceMsg { PoseMsg pose; std::array<double, 36> covariance{}; };
struct LikelihoodStatsMsg { double min = 0, max = 0, mean = 0, sigma = 0; };
struct ParticleStatsMsg { uint64_t nparticles = 0; PoseWithCovarianceMsg pose; double shift = 0; PointMsg trans_bb_min, trans_bb_max; LikelihoodStatsMsg likelihood; };

int main(int argc, char** argv)
{
    if (argc != 4) { std::fprintf(stderr, "usage: %s PARTICLES OUT K\n", argv[0]); return 2; }
    FILE* f = std::fopen(argv[1], "rb");
    if (!f) return 3;
    std::fseek(f, 0, SEEK_END);
    const size_t n = (size_t)std::ftell(f) / 68;
    std::fseek(f, 0, SEEK_SET);
    std::vector<rm::Transform> hp(n);
    std::vector<rmcl::ParticleAttributes> ha(n);
    if (std::fread(hp.data(), sizeof(rm::Transform), n, f) != n || std::fread(ha.data(), sizeof(rmcl::ParticleAttributes), n, f) != n) return 4;
    std::fclose(f);
    const size_t k = std::strtoul(argv[3], nullptr, 10);

    const std::vector<float> V = {0, 0, 0, 1, 0, 0, 0, 1, 0};
    const std::vector<uint32_t> F = {0, 1, 2};
    auto map = std::make_shared<rmcl::B200Map>(V.data(), 3u, F.data(), 1u);
    rmcl::PCDSensorUpdaterB200 up(map);
    rm::Transform* poses = nullptr; rmcl::ParticleAttributes* attrs = nullptr;
    if (cudaMalloc((void**)&poses, n * sizeof(rm::Transform)) != cudaSuccess || cudaMalloc((void**)&attrs, n * sizeof(rmcl::ParticleAttributes)) != cudaSuccess) return 5;
    cudaMemcpy(poses, hp.data(), n * sizeof(rm::Transform), cudaMemcpyHostToDevice);
    cudaMemcpy(attrs, ha.data(), n * sizeof(rmcl::ParticleAttributes), cudaMemcpyHostToDevice);

    // RmclNode::resampling (rmcl_localization.cpp:557-558): estimateStats over poses(0, k), then publishStats
    ParticleStatsMsg msg;
    rmcl::b200::fillParticleStats(msg, up.estimateStats(rm::MemoryView<rm::Transform, rm::VRAM_CUDA>{poses, k},
                                                        rm::MemoryView<rmcl::ParticleAttributes, rm::VRAM_CUDA>{attrs, k}));
    FILE* o = std::fopen(argv[2], "wb");
    if (!o) return 6;
    const PoseMsg& p = msg.pose.pose;
    const double head[7] = {p.position.x, p.position.y, p.position.z, p.orientation.x, p.orientation.y, p.orientation.z, p.orientation.w};
    std::fwrite(head, sizeof(double), 7, o);
    std::fwrite(msg.pose.covariance.data(), sizeof(double), 36, o);
    const double tail[11] = {msg.shift, msg.trans_bb_min.x, msg.trans_bb_min.y, msg.trans_bb_min.z, msg.trans_bb_max.x, msg.trans_bb_max.y, msg.trans_bb_max.z,
                             msg.likelihood.min, msg.likelihood.max, msg.likelihood.mean, msg.likelihood.sigma};
    std::fwrite(tail, sizeof(double), 11, o);
    std::fwrite(&msg.nparticles, sizeof(uint64_t), 1, o);
    std::fclose(o);

    // an empty slice is refused like every other failure of the classes
    try {
        up.estimateStats(rm::MemoryView<rm::Transform, rm::VRAM_CUDA>{poses, 0}, rm::MemoryView<rmcl::ParticleAttributes, rm::VRAM_CUDA>{attrs, 0});
        return 7;
    } catch (const std::runtime_error& e) { std::printf("REFUSED %s\n", e.what()); }
    cudaFree(poses); cudaFree(attrs);
    return cudaGetLastError() == cudaSuccess ? 0 : 8;
}
