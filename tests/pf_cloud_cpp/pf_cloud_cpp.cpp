// TEST PROGRAM: PCDSensorUpdaterB200 fed through rmcl::b200::setInput (include/rmcl_b200/rmcl_msgs_adapters.hpp) with a plain struct carrying
// the field names of sensor_msgs/PointCloud2, as RmclNode::sensorUpdate hands each cloud to its updater and then updates the particles.
// Usage: pf_cloud_cpp IN OUT.  IN: u32 nv, nf, vertices, faces; u32 n_particles, step; u64 seed; Tsb (rm::Transform); the six float
// parameters of b2_pf_params (ray casting, ng_mode 0); the particles (n poses, n attributes); u32 width, height, point_step, row_step,
// is_bigendian, n_fields; per field {char name[16], u32 offset, u32 datatype}; the data bytes.  OUT: the attributes after two updates of
// device particles (after each), then after one update of host particles -- tests/test_gpu_pf_cloud.py compares them with the Python path.
#include <cstdio>
#include <cstring>
#include <memory>
#include <string>
#include <vector>

#include <cuda_runtime.h>
#include <rmcl_b200/rmcl_msgs_adapters.hpp>

namespace rm = rmagine;

struct PointFieldMsg { std::string name; uint32_t offset = 0; uint8_t datatype = 0; uint32_t count = 1; };
struct PointCloud2Msg { uint32_t height = 0, width = 0; std::vector<PointFieldMsg> fields; bool is_bigendian = false; uint32_t point_step = 0, row_step = 0;
                        std::vector<uint8_t> data; bool is_dense = false; };

static bool rd(FILE* f, void* p, size_t n) { return std::fread(p, 1, n, f) == n; }

int main(int argc, char** argv)
{
    if (argc != 3) { std::fprintf(stderr, "usage: %s IN OUT\n", argv[0]); return 2; }
    FILE* f = std::fopen(argv[1], "rb");
    if (!f) return 3;
    uint32_t nvf[2];
    if (!rd(f, nvf, 8)) return 3;
    std::vector<float> V(3 * (size_t)nvf[0]); std::vector<uint32_t> F(3 * (size_t)nvf[1]);
    if (!rd(f, V.data(), 4 * V.size()) || !rd(f, F.data(), 4 * F.size())) return 3;
    uint32_t ns[2]; uint64_t seed; rm::Transform Tsb; float prm[6];
    if (!rd(f, ns, 8) || !rd(f, &seed, 8) || !rd(f, &Tsb, sizeof(Tsb)) || !rd(f, prm, sizeof(prm))) return 3;
    const size_t n = ns[0];
    std::vector<rm::Transform> poses(n); std::vector<rmcl::ParticleAttributes> attrs(n);
    if (!rd(f, poses.data(), n * sizeof(rm::Transform)) || !rd(f, attrs.data(), n * sizeof(rmcl::ParticleAttributes))) return 3;
    uint32_t hd[6];
    if (!rd(f, hd, sizeof(hd))) return 3;
    auto cloud = std::make_shared<PointCloud2Msg>();
    cloud->width = hd[0]; cloud->height = hd[1]; cloud->point_step = hd[2]; cloud->row_step = hd[3]; cloud->is_bigendian = hd[4] != 0;
    for (uint32_t k = 0; k < hd[5]; k++) {
        char name[16]; uint32_t od[2];
        if (!rd(f, name, 16) || !rd(f, od, 8)) return 3;
        name[15] = 0;
        cloud->fields.push_back(PointFieldMsg{name, od[0], (uint8_t)od[1], 1});
    }
    const long begin = std::ftell(f);
    std::fseek(f, 0, SEEK_END);
    cloud->data.resize((size_t)(std::ftell(f) - begin));
    std::fseek(f, begin, SEEK_SET);
    if (!rd(f, cloud->data.data(), cloud->data.size())) return 3;
    std::fclose(f);

    auto map = std::make_shared<rmcl::B200Map>(V.data(), nvf[0], F.data(), nvf[1]);
    rmcl::PCDSensorUpdaterB200 up(map);
    up.config = b2_pf_params{prm[0], prm[1], prm[2], prm[3], prm[4], prm[5], 0, 0};
    up.seed = seed; up.step = ns[1];
    up.setTsb(Tsb);
    rmcl::b200::setInput(up, std::shared_ptr<const PointCloud2Msg>(cloud));
    cloud.reset();                                                          // the updater holds the message, as Input<> holds input_

    rm::Transform* pd = nullptr; rmcl::ParticleAttributes* ad = nullptr;
    if (cudaMalloc((void**)&pd, n * sizeof(rm::Transform)) != cudaSuccess || cudaMalloc((void**)&ad, n * sizeof(rmcl::ParticleAttributes)) != cudaSuccess) return 4;
    cudaMemcpy(pd, poses.data(), n * sizeof(rm::Transform), cudaMemcpyHostToDevice);
    cudaMemcpy(ad, attrs.data(), n * sizeof(rmcl::ParticleAttributes), cudaMemcpyHostToDevice);
    rm::MemoryView<rm::Transform, rm::VRAM_CUDA> pv{pd, n};
    rm::MemoryView<rmcl::ParticleAttributes, rm::VRAM_CUDA> av{ad, n};
    FILE* o = std::fopen(argv[2], "wb");
    if (!o) return 5;
    std::vector<rmcl::ParticleAttributes> out(n);
    for (int u = 0; u < 2; u++) {
        up.update(pv, av);
        cudaMemcpy(out.data(), ad, n * sizeof(rmcl::ParticleAttributes), cudaMemcpyDeviceToHost);
        std::fwrite(out.data(), sizeof(rmcl::ParticleAttributes), n, o);
    }
    out = attrs;
    up.update(rm::MemoryView<rm::Transform, rm::RAM>{poses.data(), n}, rm::MemoryView<rmcl::ParticleAttributes, rm::RAM>{out.data(), n});
    std::fwrite(out.data(), sizeof(rmcl::ParticleAttributes), n, o);
    std::fclose(o);

    // a cloud without a field named z is refused like every other failure of the classes, when the update samples it
    auto bad = std::make_shared<PointCloud2Msg>();
    bad->width = 2; bad->height = 1; bad->point_step = 16; bad->row_step = 32; bad->data.assign(32, 0);
    bad->fields = {PointFieldMsg{"x", 0, 7, 1}, PointFieldMsg{"y", 4, 7, 1}};
    rmcl::b200::setInput(up, std::shared_ptr<const PointCloud2Msg>(bad));
    try { up.update(pv, av); return 6; } catch (const std::runtime_error& e) { std::printf("REFUSED %s\n", e.what()); }
    cudaFree(pd); cudaFree(ad);
    return cudaGetLastError() == cudaSuccess ? 0 : 7;
}
