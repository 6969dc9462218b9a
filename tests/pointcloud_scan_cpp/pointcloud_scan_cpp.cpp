// TEST PROGRAM: RCCB200Spherical::setPointCloud through rmcl::b200::unpackPointCloud (include/rmcl_b200/rmcl_msgs_adapters.hpp) over plain structs
// with the field names of sensor_msgs/PointCloud2 and sensor_msgs/PointField, as a spherical sensor's callback would call it in place of the
// pc2_to_scan node + unpackMessage.
// Usage: pointcloud_scan_cpp MESH CLOUD OUT.  MESH: u32 nv, nf, then vertices and faces.  CLOUD: u32 width, height, point_step, row_step,
// is_bigendian, n_fields, then per field {char name[16], u32 offset, u32 datatype}, then the spherical model (b2_spherical_model, 32 B), then
// T_sensor_cloud and Tom (rm::Transform, 32 B each), then the data bytes.  OUT: the dataset points and mask, then Tom_new of one
// correctOnce(Tom, identity, 5, 0) -- tests/test_gpu_pointcloud_scan.py compares it with the Python path byte for byte.
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include <rmcl_b200/rmcl_msgs_adapters.hpp>

namespace rm = rmagine;

struct PointFieldMsg { std::string name; uint32_t offset = 0; uint8_t datatype = 0; uint32_t count = 1; };
struct PointCloud2Msg { uint32_t height = 0, width = 0; std::vector<PointFieldMsg> fields; bool is_bigendian = false; uint32_t point_step = 0, row_step = 0;
                        std::vector<uint8_t> data; bool is_dense = false; };

static bool rd(FILE* f, void* p, size_t n) { return std::fread(p, 1, n, f) == n; }

int main(int argc, char** argv)
{
    if (argc != 4) { std::fprintf(stderr, "usage: %s MESH CLOUD OUT\n", argv[0]); return 2; }
    FILE* f = std::fopen(argv[1], "rb");
    if (!f) return 3;
    uint32_t nvf[2];
    if (!rd(f, nvf, 8)) return 3;
    std::vector<float> V(3 * (size_t)nvf[0]); std::vector<uint32_t> F(3 * (size_t)nvf[1]);
    if (!rd(f, V.data(), 4 * V.size()) || !rd(f, F.data(), 4 * F.size())) return 3;
    std::fclose(f);

    f = std::fopen(argv[2], "rb");
    if (!f) return 4;
    uint32_t hd[6];
    if (!rd(f, hd, sizeof(hd))) return 4;
    PointCloud2Msg cloud;
    cloud.width = hd[0]; cloud.height = hd[1]; cloud.point_step = hd[2]; cloud.row_step = hd[3]; cloud.is_bigendian = hd[4] != 0;
    for (uint32_t k = 0; k < hd[5]; k++) {
        char name[16]; uint32_t od[2];
        if (!rd(f, name, 16) || !rd(f, od, 8)) return 4;
        name[15] = 0;
        cloud.fields.push_back(PointFieldMsg{name, od[0], (uint8_t)od[1], 1});
    }
    b2_spherical_model sm;
    rm::Transform T_sensor_cloud, Tom;
    if (!rd(f, &sm, sizeof(sm)) || !rd(f, &T_sensor_cloud, sizeof(T_sensor_cloud)) || !rd(f, &Tom, sizeof(Tom))) return 4;
    std::fseek(f, 0, SEEK_END);
    const long end = std::ftell(f);
    const long begin = (long)(sizeof(hd) + 24 * hd[5] + sizeof(sm) + sizeof(T_sensor_cloud) + sizeof(Tom));
    cloud.data.resize((size_t)(end - begin));
    std::fseek(f, begin, SEEK_SET);
    if (!rd(f, cloud.data.data(), cloud.data.size())) return 4;
    std::fclose(f);

    auto map = std::make_shared<rmcl::B200Map>(V.data(), nvf[0], F.data(), nvf[1]);
    rmcl::RCCB200Spherical rcc(map);
    rm::SphericalModel model;
    model.phi.min = sm.phi_min; model.phi.inc = sm.phi_inc; model.phi.size = sm.phi_size;
    model.theta.min = sm.theta_min; model.theta.inc = sm.theta_inc; model.theta.size = sm.theta_size;
    model.range.min = sm.range_min; model.range.max = sm.range_max;
    rcc.setModel(model);
    rmcl::b200::unpackPointCloud(rcc, cloud, T_sensor_cloud);
    float* p = nullptr; uint8_t* m = nullptr; uint32_t n = 0;
    rmcl::b2_check(b2_rcc_dataset_view(rcc.handle(), &p, &m, &n), "dataset_view");
    std::vector<float> pts(3 * (size_t)n); std::vector<uint8_t> mask(n);
    rmcl::b2_check(b2_rcc_download_dataset(rcc.handle(), pts.data(), mask.data()), "download_dataset");
    const rm::Transform I = rm::Transform::Identity();
    const rm::Transform T = rcc.correctOnce(Tom, I, 5, 0.0);

    FILE* o = std::fopen(argv[3], "wb");
    if (!o) return 6;
    std::fwrite(pts.data(), 4, pts.size(), o);
    std::fwrite(mask.data(), 1, mask.size(), o);
    std::fwrite(&T, sizeof(T), 1, o);
    std::fclose(o);

    // a cloud without a field named z is refused like every other failure of the classes
    for (size_t k = 0; k < cloud.fields.size(); k++) if (cloud.fields[k].name == "z") { cloud.fields.erase(cloud.fields.begin() + k); break; }
    try { rmcl::b200::unpackPointCloud(rcc, cloud, T_sensor_cloud); return 7; }
    catch (const std::runtime_error& e) { std::printf("REFUSED %s\n", e.what()); }
    return 0;
}
