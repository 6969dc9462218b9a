// TEST PROGRAM: PCDSensorUpdaterB200::globalSearchBnB (include/rmcl_b200/rcc_b200.hpp) against the C ABI.  Usage: pf_search_bnb_cpp IN OUT.
// IN holds nv, nf, n_beams (u32 each), resolution, truncation, dist_sigma, min_ratio (f32 each), the b2_search_config (40 B), then nv
// vertices (3 f32), nf faces (3 u32), Tsb (32 B) and n_beams beams (64 B).  OUT receives the class's b2_search_bnb_result (384 B) and its
// records (n_records x 48 B), with the surface rule's suggested values.  tests/test_gpu_pf_search_bnb_cpp.py compares the file with the
// Python path.
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
    uint32_t hd[3];
    float hf[4];
    b2_search_config cfg;
    if (std::fread(hd, 4, 3, in) != 3 || std::fread(hf, 4, 4, in) != 4 || std::fread(&cfg, sizeof(cfg), 1, in) != 1) return 4;
    const uint32_t nv = hd[0], nf = hd[1], n_beams = hd[2];
    std::vector<float> V(3 * (size_t)nv);
    std::vector<uint32_t> F(3 * (size_t)nf);
    rm::Transform Tsb;
    std::vector<b2_range_meas> beams(n_beams);
    if (std::fread(V.data(), 4, V.size(), in) != V.size() || std::fread(F.data(), 4, F.size(), in) != F.size() || std::fread(&Tsb, 32, 1, in) != 1 ||
        std::fread(beams.data(), sizeof(b2_range_meas), n_beams, in) != n_beams)
        return 4;
    std::fclose(in);
    auto map = std::make_shared<rmcl::B200Map>(V.data(), nv, F.data(), nf);
    rmcl::B200DistanceField field(map, hf[0], hf[1]);
    rmcl::PCDSensorUpdaterB200 up(map);
    up.setTsb(Tsb);
    up.config.dist_sigma = hf[2];
    const b2_surface_config surface = rmcl::PCDSensorUpdaterB200::surface_config();
    b2_search_bnb_result res{};
    const std::vector<b2_search_record> recs = up.globalSearchBnB(field, beams.data(), n_beams, cfg, &surface, hf[3], &res);
    FILE* f = std::fopen(argv[2], "wb");
    if (!f) return 4;
    std::fwrite(&res, sizeof(res), 1, f); std::fwrite(recs.data(), sizeof(b2_search_record), recs.size(), f);
    std::fclose(f);

    // a refused min_ratio throws like every other failure of the classes
    try { up.globalSearchBnB(field, beams.data(), n_beams, cfg, nullptr, 1.5f); return 6; }
    catch (const std::runtime_error& e) { std::printf("REFUSED %s\n", e.what()); }
    return cudaGetLastError() == cudaSuccess ? 0 : 7;
}
