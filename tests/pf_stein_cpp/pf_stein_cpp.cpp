// TEST PROGRAM: PCDSensorUpdaterB200's sharded Stein steps (steinBegin / steinScore / steinMove / steinResult, include/rmcl_b200/rcc_b200.hpp)
// on device memory, two handles on one device playing two ranks, against steinUpdate of the whole set.  Usage: pf_stein_cpp IN OUT.
// IN holds nv, nf, n, n_beams, iterations, n_ref (u32 each), resolution, truncation, dist_sigma (f32 each), then nv vertices (3 f32), nf
// faces (3 u32), Tsb (32 B), n poses (32 B) and n_beams beams (64 B).  OUT receives steinUpdate's b2_stein_result (32 B) and poses (n x 32 B),
// then the two ranks' b2_stein_slice_result (40 B each) and their concatenated poses, with seed 1234 and step 7.  Rank r moves
// [r n / 2, (r + 1) n / 2) and scores [r m / 2, (r + 1) m / 2) of J; per iteration both score into one snapshot, both move into their own
// buffers, and the buffers are copied back into the whole set (the all-gathers of a multi-GPU node).  tests/test_gpu_pf_stein_sharded.py
// compares the file with the Python path.
#include <cstdio>
#include <memory>
#include <vector>

#include <cuda_runtime.h>
#include <rmcl_b200/rcc_b200.hpp>

namespace rm = rmagine;

int main(int argc, char** argv)
{
    if (argc != 3) { std::fprintf(stderr, "usage: %s IN OUT\n", argv[0]); return 2; }
    FILE* in = std::fopen(argv[1], "rb");
    if (!in) return 4;
    uint32_t hd[6];
    float hf[3];
    if (std::fread(hd, 4, 6, in) != 6 || std::fread(hf, 4, 3, in) != 3) return 4;
    const uint32_t nv = hd[0], nf = hd[1], n = hd[2], n_beams = hd[3];
    std::vector<float> V(3 * (size_t)nv);
    std::vector<uint32_t> F(3 * (size_t)nf);
    rm::Transform Tsb;
    std::vector<rm::Transform> hp(n);
    std::vector<b2_range_meas> beams(n_beams);
    if (std::fread(V.data(), 4, V.size(), in) != V.size() || std::fread(F.data(), 4, F.size(), in) != F.size() || std::fread(&Tsb, 32, 1, in) != 1 ||
        std::fread(hp.data(), 32, n, in) != n || std::fread(beams.data(), sizeof(b2_range_meas), n_beams, in) != n_beams)
        return 4;
    std::fclose(in);
    auto map = std::make_shared<rmcl::B200Map>(V.data(), nv, F.data(), nf);
    auto field = std::make_shared<rmcl::B200DistanceField>(map, hf[0], hf[1]);
    b2_stein_config cfg = rmcl::PCDSensorUpdaterB200::stein_config();
    cfg.iterations = hd[4]; cfg.n_ref = hd[5];
    const uint32_t m = (cfg.n_ref == 0 || cfg.n_ref >= n) ? n : cfg.n_ref;
    rmcl::PCDSensorUpdaterB200 whole(map), rank[2] = {rmcl::PCDSensorUpdaterB200(map), rmcl::PCDSensorUpdaterB200(map)};
    for (rmcl::PCDSensorUpdaterB200* u : {&whole, &rank[0], &rank[1]}) { u->setDistanceField(field); u->setTsb(Tsb); u->config.dist_sigma = hf[2]; }

    rm::Transform *poses = nullptr, *poses_all = nullptr, *out[2] = {nullptr, nullptr};
    b2_stein_ref* snap = nullptr;
    const size_t bytes = (size_t)n * sizeof(rm::Transform);
    if (cudaMalloc((void**)&poses, bytes) != cudaSuccess || cudaMalloc((void**)&poses_all, bytes) != cudaSuccess ||
        cudaMalloc((void**)&out[0], bytes) != cudaSuccess || cudaMalloc((void**)&out[1], bytes) != cudaSuccess ||
        cudaMalloc((void**)&snap, (size_t)(m ? m : 1) * sizeof(b2_stein_ref)) != cudaSuccess)
        return 3;
    cudaMemcpy(poses, hp.data(), bytes, cudaMemcpyHostToDevice);
    cudaMemcpy(poses_all, hp.data(), bytes, cudaMemcpyHostToDevice);

    const b2_stein_result res = whole.steinUpdate(rm::MemoryView<rm::Transform, rm::VRAM_CUDA>{poses, n}, beams.data(), n_beams, cfg, 1234, 7);

    const uint32_t first[3] = {0, n / 2, n}, j_first[3] = {0, m / 2, m};
    for (int r = 0; r < 2; r++) rank[r].steinBegin(n, first[r], first[r + 1] - first[r], j_first[r], j_first[r + 1] - j_first[r], beams.data(), n_beams, cfg, 1234, 7);
    rm::MemoryView<rm::Transform, rm::VRAM_CUDA> all{poses_all, n};
    for (uint32_t k = 0; k < cfg.iterations; k++) {
        for (int r = 0; r < 2; r++) rank[r].steinScore(all, k, snap + j_first[r]);
        for (int r = 0; r < 2; r++) rank[r].steinMove(all, snap, k, rm::MemoryView<rm::Transform, rm::VRAM_CUDA>{out[r], first[r + 1] - first[r]});
        for (int r = 0; r < 2; r++) cudaMemcpy(poses_all + first[r], out[r], (size_t)(first[r + 1] - first[r]) * sizeof(rm::Transform), cudaMemcpyDeviceToDevice);
    }
    const b2_stein_slice_result sr[2] = {rank[0].steinResult(), rank[1].steinResult()};

    std::vector<rm::Transform> op(n), os(n);
    cudaMemcpy(op.data(), poses, bytes, cudaMemcpyDeviceToHost);
    cudaMemcpy(os.data(), poses_all, bytes, cudaMemcpyDeviceToHost);
    FILE* f = std::fopen(argv[2], "wb");
    if (!f) return 4;
    std::fwrite(&res, sizeof(res), 1, f); std::fwrite(op.data(), 32, n, f);
    std::fwrite(sr, sizeof(b2_stein_slice_result), 2, f); std::fwrite(os.data(), 32, n, f);
    std::fclose(f);

    // a call out of sequence throws like every other failure of the classes
    try { rank[0].steinMove(all, snap, 0, rm::MemoryView<rm::Transform, rm::VRAM_CUDA>{out[0], first[1]}); return 6; }
    catch (const std::runtime_error& e) { std::printf("REFUSED %s\n", e.what()); }
    cudaFree(poses); cudaFree(poses_all); cudaFree(out[0]); cudaFree(out[1]); cudaFree(snap);
    return cudaGetLastError() == cudaSuccess ? 0 : 7;
}
