// TEST PROGRAM: rmcl::micp_pose_covariance (include/rmcl_b200/rcc_b200.hpp) after rmcl::micp_correct, as a node's publishPose step would call
// them.  Usage: micp_cov_cpp IN OUT.  IN holds nv, nf, n (u32), the vertices (3 nv floats), the faces (3 nf u32), a b2_spherical_model (32 B),
// Tsb and Tom (32 B each) and n ranges.  OUT receives Tom after a 3-step correction (32 B) and the b2_micp_covariance record (984 B) of its last
// step; tests/test_gpu_micp_cov.py compares the file with the Python path.
#include <cstdio>
#include <vector>

#include <rmcl_b200/rcc_b200.hpp>

namespace rm = rmagine;

int main(int argc, char** argv)
{
    if (argc != 3) { std::fprintf(stderr, "usage: %s IN OUT\n", argv[0]); return 2; }
    FILE* in = std::fopen(argv[1], "rb");
    if (!in) return 4;
    uint32_t hd[3];
    if (std::fread(hd, 4, 3, in) != 3) return 4;
    std::vector<float> V(3 * (size_t)hd[0]), ranges(hd[2]);
    std::vector<uint32_t> F(3 * (size_t)hd[1]);
    b2_spherical_model m;
    rm::Transform Tsb, Tom;
    if (std::fread(V.data(), 4, V.size(), in) != V.size() || std::fread(F.data(), 4, F.size(), in) != F.size() || std::fread(&m, sizeof(m), 1, in) != 1 ||
        std::fread(&Tsb, sizeof(Tsb), 1, in) != 1 || std::fread(&Tom, sizeof(Tom), 1, in) != 1 || std::fread(ranges.data(), 4, ranges.size(), in) != ranges.size())
        return 4;
    std::fclose(in);
    auto map = std::make_shared<rmcl::B200Map>(V.data(), hd[0], F.data(), hd[1]);
    rmcl::RCCB200Spherical s(map);
    s.setTsb(Tsb);
    s.setModel(rm::SphericalModel{{m.phi_min, m.phi_inc, m.phi_size}, {m.theta_min, m.theta_inc, m.theta_size}, {m.range_min, m.range_max}});
    s.setRanges(ranges.data(), ranges.size());
    const std::vector<rm::Transform> Tbo{rm::Transform{{0.f, 0.f, 0.f, 1.f}, {0.f, 0.f, 0.f}, 0u}};
    double cp = 0.0;
    std::vector<b2_micp_step> steps;
    rmcl::micp_correct({&s}, Tbo, {}, Tom, cp, true, 3, 5, &steps);
    const rm::Transform& Td = *reinterpret_cast<const rm::Transform*>(&steps[2].T_onew_oold);       // the same 32-byte layout
    const b2_micp_covariance cov = rmcl::micp_pose_covariance({&s}, Tbo, {}, Td, steps[1].convergence_progress);
    FILE* f = std::fopen(argv[2], "wb");
    if (!f) return 4;
    std::fwrite(&Tom, sizeof(Tom), 1, f);
    std::fwrite(&cov, sizeof(cov), 1, f);
    std::fclose(f);
    // a refused setting throws like every other failure of the classes
    try { rmcl::micp_pose_covariance({&s}, Tbo, {}, Td, 0.0, nullptr, b2_micp_cov_config{1.0, 1e2}); return 6; }
    catch (const std::runtime_error& e) { std::printf("REFUSED %s\n", e.what()); }
    return 0;
}
