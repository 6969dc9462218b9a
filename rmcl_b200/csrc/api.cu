// api.cu -- C ABI (include/rmcl_b200.h) over the sm_90a kernels.  No CPU fallback anywhere: every entry point either runs
// the CUDA path or fails with B2_ERR_CUDA.
#include "kernels.cuh"
#include "lbvh.cuh"
#include <cub/device/device_scan.cuh>

#include <algorithm>
#include <atomic>
#include <chrono>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <deque>
#include <mutex>
#include <new>
#include <vector>

// ---------------------------------------------------------------------------------------------------------------------
static thread_local char g_err[512] = "";
static std::atomic<uint64_t> g_launches{0};

static int fail(int code, const char* fmt, ...)
{
    va_list ap; va_start(ap, fmt); vsnprintf(g_err, sizeof(g_err), fmt, ap); va_end(ap);
    return code;
}
#define CU(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) { (void)cudaGetLastError(); } if (e_ != cudaSuccess) return fail(B2_ERR_CUDA, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(e_), __FILE__, __LINE__); } while (0)
#define LAUNCHED() do { g_launches.fetch_add(1, std::memory_order_relaxed); cudaError_t e_ = cudaGetLastError(); if (e_ != cudaSuccess) return fail(B2_ERR_CUDA, "kernel launch failed: %s (%s:%d)", cudaGetErrorString(e_), __FILE__, __LINE__); } while (0)
#define NOTNULL(p) do { if (!(p)) return fail(B2_ERR_INVALID, "%s: null argument '%s'", __func__, #p); } while (0)

extern "C" const char* b2_last_error(void) { return g_err; }
extern "C" int b2_version(void) { return 100; }
extern "C" uint64_t b2_kernel_launch_count(void) { return g_launches.load(); }
// pending (not yet consumed) CUDA runtime error of the calling thread, "" if none; does not clear it (test hygiene: no entry point may leave one behind)
extern "C" const char* b2_peek_cuda_error(void) { const cudaError_t e = cudaPeekAtLastError(); return e == cudaSuccess ? "" : cudaGetErrorString(e); }
extern "C" int b2_device_count(int* n) { NOTNULL(n); CU(cudaGetDeviceCount(n)); return B2_OK; }

// ---------------------------------------------------------------------------------------------------------------------
struct b2_mesh {
    std::atomic<int> refs{1};           // the creator's reference + one per b2_rcc / b2_pf handle: the BVH stays resident until the last user is gone
    int device = 0; int build_mode = 0;
    B2Node8* d_nodes = nullptr; B2Tri* d_tris = nullptr;
    uint32_t n_nodes = 0, n_tris = 0, n_faces = 0, n_verts = 0, max_depth = 0;
    float build_ms = 0.f, sah = 0.f, abs_max[3] = {0.f, 0.f, 0.f};
    std::vector<uint32_t> level_begin;          // device-built maps: node index ranges per tree level (for b2_mesh_refit)
    uint32_t* d_faces = nullptr;                // device-built maps keep the face list for b2_mesh_refit (12 B per face)
    BvhView view() const
    {
        BvhView v; v.nodes = reinterpret_cast<const float4*>(d_nodes); v.tris = reinterpret_cast<const float4*>(d_tris);
        v.bx = abs_max[0]; v.by = abs_max[1]; v.bz = abs_max[2]; return v;
    }
};

template <typename T> struct DevBuf {
    T* p = nullptr; size_t cap = 0;
    int reserve(size_t n) {
        if (n <= cap) return B2_OK;
        if (p) cudaFree(p);
        p = nullptr; cap = 0;
        cudaError_t e = cudaMalloc((void**)&p, sizeof(T) * n);
        if (e != cudaSuccess) return fail(B2_ERR_OOM, "cudaMalloc(%zu bytes) failed: %s", sizeof(T) * n, cudaGetErrorString(e));
        cap = n; return B2_OK;
    }
    void release() { if (p) cudaFree(p); p = nullptr; cap = 0; }
};
#define RES(call) do { int r_ = (call); if (r_ != B2_OK) return r_; } while (0)

extern "C" int b2_mesh_create(const float* verts, uint32_t nv, const uint32_t* faces, uint32_t nf, int device, int build_mode, b2_mesh** out)
{
    NOTNULL(out); *out = nullptr;
    if (nf == 0 || nv == 0) return fail(B2_ERR_NO_MAP, "EMPTY MAP: %u vertices, %u faces", nv, nf);
    NOTNULL(verts); NOTNULL(faces);
    if (build_mode != B2_BUILD_HOST_SAH && build_mode != B2_BUILD_DEVICE_LBVH) return fail(B2_ERR_UNSUPPORTED, "unknown build_mode %d", build_mode);
    int ndev = 0; CU(cudaGetDeviceCount(&ndev));
    if (device < 0 || device >= ndev) return fail(B2_ERR_INVALID, "device %d out of range (%d devices)", device, ndev);
    CU(cudaSetDevice(device));
    if (build_mode == B2_BUILD_DEVICE_LBVH) {
        for (size_t i = 0; i < 3 * (size_t)nf; i++) if (faces[i] >= nv) return fail(B2_ERR_INVALID, "BVH build failed: face index out of range");
        if (!b2_vertices_ok(verts, 3 * (size_t)nv)) return fail(B2_ERR_INVALID, "BVH build failed: a vertex coordinate is not finite or exceeds 2^62 in magnitude");
        const auto t0 = std::chrono::steady_clock::now();
        float* d_v = nullptr; uint32_t* d_f = nullptr;
        cudaError_t e = cudaMalloc((void**)&d_v, sizeof(float) * 3 * (size_t)nv);
        if (e == cudaSuccess) e = cudaMalloc((void**)&d_f, sizeof(uint32_t) * 3 * (size_t)nf);
        if (e == cudaSuccess) e = cudaMemcpy(d_v, verts, sizeof(float) * 3 * (size_t)nv, cudaMemcpyHostToDevice);
        if (e == cudaSuccess) e = cudaMemcpy(d_f, faces, sizeof(uint32_t) * 3 * (size_t)nf, cudaMemcpyHostToDevice);
        if (e != cudaSuccess) { cudaFree(d_v); cudaFree(d_f); return fail(B2_ERR_CUDA, "mesh upload failed: %s", cudaGetErrorString(e)); }
        b2_mesh* m = new (std::nothrow) b2_mesh();
        if (!m) { cudaFree(d_v); cudaFree(d_f); return fail(B2_ERR_OOM, "out of host memory"); }
        const char* err = "";
        const int rc = lbvh_build_device(d_v, nv, d_f, nf, &m->d_nodes, &m->n_nodes, &m->d_tris, &m->n_tris, &m->max_depth, m->abs_max, &err, &m->level_begin);
        g_launches.fetch_add(5 + m->max_depth);
        cudaFree(d_v);
        if (rc == 0) m->d_faces = d_f; else cudaFree(d_f);
        if (rc != 0) { delete m; return fail(rc == -5 ? B2_ERR_INVALID : B2_ERR_CUDA, "BVH build failed: %s (%s)", err, cudaGetErrorString(cudaGetLastError())); }
        m->device = device; m->build_mode = build_mode; m->n_faces = nf; m->n_verts = nv; m->sah = 0.f;
        m->build_ms = std::chrono::duration<float, std::milli>(std::chrono::steady_clock::now() - t0).count();
        *out = m;
        return B2_OK;
    }
    const auto t0 = std::chrono::steady_clock::now();
    B2BvhHost hb; const char* err = "";
    const int rc = b2_build_bvh8_host(verts, nv, faces, nf, &hb, &err);
    if (rc != 0) return fail(rc == -3 ? B2_ERR_NO_MAP : (rc == -4 ? B2_ERR_OOM : B2_ERR_INVALID), "BVH build failed: %s", err);
    b2_mesh* m = new (std::nothrow) b2_mesh();
    if (!m) { b2_free_bvh8_host(&hb); return fail(B2_ERR_OOM, "out of host memory"); }
    m->device = device; m->build_mode = build_mode; m->n_nodes = hb.n_nodes; m->n_tris = hb.n_tris; m->n_faces = nf; m->n_verts = nv;
    m->max_depth = hb.max_depth; m->sah = hb.sah_cost;
    for (int k = 0; k < 3; k++) m->abs_max[k] = hb.abs_max[k];
    cudaError_t e = cudaMalloc((void**)&m->d_nodes, sizeof(B2Node8) * (size_t)hb.n_nodes);
    if (e == cudaSuccess) e = cudaMalloc((void**)&m->d_tris, sizeof(B2Tri) * (size_t)std::max(hb.n_tris, 1u));
    if (e == cudaSuccess) e = cudaMemcpy(m->d_nodes, hb.nodes, sizeof(B2Node8) * (size_t)hb.n_nodes, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMemcpy(m->d_tris, hb.tris, sizeof(B2Tri) * (size_t)hb.n_tris, cudaMemcpyHostToDevice);
    b2_free_bvh8_host(&hb);
    if (e != cudaSuccess) { if (m->d_nodes) cudaFree(m->d_nodes); if (m->d_tris) cudaFree(m->d_tris); delete m; return fail(B2_ERR_CUDA, "map upload failed: %s", cudaGetErrorString(e)); }
    m->build_ms = std::chrono::duration<float, std::milli>(std::chrono::steady_clock::now() - t0).count();
    *out = m;
    return B2_OK;
}

int b2_load_mesh_file(const char* path, std::vector<float>& V, std::vector<uint32_t>& F, const char** err_out);   // mesh_io.cpp

extern "C" int b2_mesh_file_load(const char* path, float** verts, uint32_t* nv, uint32_t** faces, uint32_t* nf)
{
    NOTNULL(path); NOTNULL(verts); NOTNULL(nv); NOTNULL(faces); NOTNULL(nf);
    *verts = nullptr; *faces = nullptr; *nv = 0; *nf = 0;
    std::vector<float> V; std::vector<uint32_t> F; const char* err = "";
    const int rc = b2_load_mesh_file(path, V, F, &err);
    if (rc != 0) return fail(rc == -3 ? B2_ERR_NO_MAP : (rc == -4 ? B2_ERR_OOM : B2_ERR_INVALID), "mesh import of '%s' failed: %s", path, err);
    float* v = (float*)malloc(sizeof(float) * V.size()); uint32_t* f = (uint32_t*)malloc(sizeof(uint32_t) * F.size());
    if (!v || !f) { free(v); free(f); return fail(B2_ERR_OOM, "out of host memory"); }
    memcpy(v, V.data(), sizeof(float) * V.size()); memcpy(f, F.data(), sizeof(uint32_t) * F.size());
    *verts = v; *faces = f; *nv = (uint32_t)(V.size() / 3); *nf = (uint32_t)(F.size() / 3);
    return B2_OK;
}
extern "C" void b2_mesh_file_free(float* verts, uint32_t* faces) { free(verts); free(faces); }

extern "C" int b2_mesh_create_from_file(const char* path, int device, int build_mode, b2_mesh** out)
{
    NOTNULL(out); *out = nullptr; NOTNULL(path);
    std::vector<float> V; std::vector<uint32_t> F; const char* err = "";
    const int rc = b2_load_mesh_file(path, V, F, &err);
    if (rc != 0) return fail(rc == -3 ? B2_ERR_NO_MAP : (rc == -4 ? B2_ERR_OOM : B2_ERR_INVALID), "mesh import of '%s' failed: %s", path, err);
    return b2_mesh_create(V.data(), (uint32_t)(V.size() / 3), F.data(), (uint32_t)(F.size() / 3), device, build_mode, out);
}

// Embree / OptiX scene re-commit after the vertices moved (SURVEY.md 8f1; the reference flags dependants with `outdated`,
// Correspondences.hpp:26-31): refit of the resident tree, no rebuild.  Only for device-built maps (they keep their level ranges and faces).
extern "C" int b2_mesh_refit(b2_mesh* m, const float* verts, uint32_t nv, int src_is_device)
{
    NOTNULL(m); NOTNULL(verts);
    if (m->level_begin.size() < 2 || !m->d_faces)
        return fail(B2_ERR_UNSUPPORTED, "refit is not available for this map: it needs the level ranges and face list only b2_mesh_create(..., B2_BUILD_DEVICE_LBVH) keeps "
                                        "(host-SAH maps and maps imported from a blob do not have them)");
    if (nv != m->n_verts) return fail(B2_ERR_INVALID, "refit keeps the topology: %u vertices given, the map has %u", nv, m->n_verts);
    CU(cudaSetDevice(m->device));
    const auto t0 = std::chrono::steady_clock::now();
    if (!src_is_device && !b2_vertices_ok(verts, 3 * (size_t)nv)) return fail(B2_ERR_INVALID, "refit: a vertex coordinate is not finite or exceeds 2^62 in magnitude");
    DevBuf<float> d_v; DevBuf<unsigned int> d_bits;
    const float* vp = verts;
    if (!src_is_device) {
        RES(d_v.reserve(3 * (size_t)nv));
        cudaError_t e = cudaMemcpy(d_v.p, verts, sizeof(float) * 3 * (size_t)nv, cudaMemcpyHostToDevice);
        if (e != cudaSuccess) { d_v.release(); return fail(B2_ERR_CUDA, "refit upload failed: %s", cudaGetErrorString(e)); }
        vp = d_v.p;
    }
    int rc = d_bits.reserve(3);
    if (rc == B2_OK && cudaMemset(d_bits.p, 0, 3 * sizeof(unsigned int)) != cudaSuccess) rc = fail(B2_ERR_CUDA, "refit: memset failed");
    if (rc == B2_OK) {
        cudaDeviceSynchronize();                                            // no trace of any handle may be in flight on the old boxes
        for (size_t l = m->level_begin.size() - 1; l-- > 0;) {
            const uint32_t b = m->level_begin[l], e = m->level_begin[l + 1];
            if (e > b) { k_bvh8_refit_level<<<(e - b + 127) / 128, 128>>>(b, e, m->d_nodes, m->d_tris, vp, m->d_faces); g_launches.fetch_add(1); }
        }
        k_abs_max<<<296, 256>>>(vp, nv, d_bits.p); g_launches.fetch_add(1);
        unsigned int bits[3] = {0, 0, 0};
        cudaError_t e = cudaMemcpy(bits, d_bits.p, sizeof(bits), cudaMemcpyDeviceToHost);
        if (e == cudaSuccess) e = cudaGetLastError();
        if (e != cudaSuccess) rc = fail(B2_ERR_CUDA, "refit failed: %s", cudaGetErrorString(e));
        else for (int k = 0; k < 3; k++) memcpy(&m->abs_max[k], &bits[k], 4);
    }
    d_v.release(); d_bits.release();
    if (rc == B2_OK) m->build_ms = std::chrono::duration<float, std::milli>(std::chrono::steady_clock::now() - t0).count();
    return rc;
}

// ---- BVH blob: build once, ship to the other ranks / to disk (SURVEY.md 8b: b2_mesh_bvh_blob for broadcast); layout in bvh8.h --------
static const char kBlobMagic[8] = {'B', '2', 'B', 'V', 'H', '8', 'F', 0};

extern "C" int b2_mesh_blob_size(const b2_mesh* m, uint64_t* bytes)
{
    NOTNULL(m); NOTNULL(bytes);
    *bytes = sizeof(B2BlobHeader) + (uint64_t)m->n_nodes * sizeof(B2Node8) + (uint64_t)m->n_tris * sizeof(B2Tri);
    return B2_OK;
}

extern "C" int b2_mesh_export_blob(const b2_mesh* m, void* dst_host, uint64_t capacity)
{
    NOTNULL(m); NOTNULL(dst_host);
    uint64_t need = 0; b2_mesh_blob_size(m, &need);
    if (capacity < need) return fail(B2_ERR_INVALID, "blob buffer too small: %llu < %llu bytes", (unsigned long long)capacity, (unsigned long long)need);
    CU(cudaSetDevice(m->device));
    B2BlobHeader hd; memset(&hd, 0, sizeof(hd));
    memcpy(hd.magic, kBlobMagic, 8);
    hd.version = 2; hd.node_bytes = sizeof(B2Node8); hd.tri_bytes = sizeof(B2Tri); hd.n_nodes = m->n_nodes; hd.n_tris = m->n_tris; hd.n_faces = m->n_faces;
    hd.n_verts = m->n_verts; hd.max_depth = m->max_depth; hd.build_mode = m->build_mode; hd.sah = m->sah;
    for (int k = 0; k < 3; k++) hd.abs_max[k] = m->abs_max[k];
    char* p = static_cast<char*>(dst_host);
    memcpy(p, &hd, sizeof(hd));
    CU(cudaMemcpy(p + sizeof(hd), m->d_nodes, (size_t)m->n_nodes * sizeof(B2Node8), cudaMemcpyDeviceToHost));
    CU(cudaMemcpy(p + sizeof(hd) + (size_t)m->n_nodes * sizeof(B2Node8), m->d_tris, (size_t)m->n_tris * sizeof(B2Tri), cudaMemcpyDeviceToHost));
    return B2_OK;
}

extern "C" int b2_mesh_create_from_blob(const void* blob_host, uint64_t bytes, int device, b2_mesh** out)
{
    NOTNULL(out); *out = nullptr; NOTNULL(blob_host);
    if (bytes < sizeof(B2BlobHeader)) return fail(B2_ERR_INVALID, "BVH blob truncated (%llu bytes)", (unsigned long long)bytes);
    B2BlobHeader hd; memcpy(&hd, blob_host, sizeof(hd));
    if (memcmp(hd.magic, kBlobMagic, 8) != 0 || hd.version != 2 || hd.node_bytes != sizeof(B2Node8) || hd.tri_bytes != sizeof(B2Tri))
        return fail(B2_ERR_INVALID, "not a BVH blob of this library version");
    const uint64_t need = sizeof(hd) + (uint64_t)hd.n_nodes * sizeof(B2Node8) + (uint64_t)hd.n_tris * sizeof(B2Tri);
    if (hd.n_nodes == 0 || hd.n_tris == 0) return fail(B2_ERR_NO_MAP, "EMPTY MAP in BVH blob");
    if (bytes < need || hd.max_depth > B2_TRAVERSAL_STACK - 4) return fail(B2_ERR_INVALID, "BVH blob inconsistent (%llu of %llu bytes, depth %u)", (unsigned long long)bytes, (unsigned long long)need, hd.max_depth);
    // structural check of the indices the traversal follows (a corrupt blob must not turn into out-of-bounds device reads)
    const B2Node8* nodes = reinterpret_cast<const B2Node8*>(static_cast<const char*>(blob_host) + sizeof(hd));
    for (uint32_t i = 0; i < hd.n_nodes; i++) {
        uint32_t n_inner = 0, tri_end = 0;
        for (int sl = 0; sl < 8; sl++) {
            const uint8_t meta = nodes[i].meta[sl];
            if ((nodes[i].imask() >> sl) & 1u) n_inner++;
            else if (meta) { const uint32_t cnt = (meta >> 5) == 7 ? 3 : ((meta >> 5) == 3 ? 2 : 1); tri_end = std::max(tri_end, (uint32_t)(meta & 0x1fu) + cnt); }
        }
        if ((n_inner && (uint64_t)nodes[i].child_base + n_inner > hd.n_nodes) || (tri_end && (uint64_t)nodes[i].tri_base + tri_end > hd.n_tris))
            return fail(B2_ERR_INVALID, "BVH blob corrupt: node %u points outside the arrays", i);
        if (nodes[i].masks != b2_masks_from_meta(nodes[i].meta)) return fail(B2_ERR_INVALID, "BVH blob corrupt: node %u has inconsistent child masks", i);
        // children sit strictly behind their parent (breadth-first layout): makes the structure acyclic, so the depth below is well defined
        if (n_inner && nodes[i].child_base <= i) return fail(B2_ERR_INVALID, "BVH blob corrupt: node %u has a child at or before itself", i);
    }
    {
        // the real depth, not the header's claim: the traversal stack has B2_TRAVERSAL_STACK entries
        std::vector<uint8_t> depth;
        try { depth.assign(hd.n_nodes, 0); } catch (const std::exception&) { return fail(B2_ERR_OOM, "out of host memory"); }
        uint32_t max_depth = 0;
        for (uint32_t i = 0; i < hd.n_nodes; i++) {            // parents precede children: one forward pass
            uint32_t n_inner = 0;
            for (int sl = 0; sl < 8; sl++) if ((nodes[i].imask() >> sl) & 1u) n_inner++;
            for (uint32_t c = 0; c < n_inner; c++) { const uint32_t d = (uint32_t)depth[i] + 1u; if (d > 250u) return fail(B2_ERR_INVALID, "BVH blob corrupt: tree too deep"); depth[nodes[i].child_base + c] = (uint8_t)std::max<uint32_t>(depth[nodes[i].child_base + c], d); max_depth = std::max(max_depth, d); }
        }
        if (max_depth + 1 > B2_TRAVERSAL_STACK - 4) return fail(B2_ERR_INVALID, "BVH blob: tree depth %u exceeds the traversal stack", max_depth + 1);
    }
    int ndev = 0; CU(cudaGetDeviceCount(&ndev));
    if (device < 0 || device >= ndev) return fail(B2_ERR_INVALID, "device %d out of range (%d devices)", device, ndev);
    CU(cudaSetDevice(device));
    const auto t0 = std::chrono::steady_clock::now();
    b2_mesh* m = new (std::nothrow) b2_mesh();
    if (!m) return fail(B2_ERR_OOM, "out of host memory");
    m->device = device; m->build_mode = hd.build_mode; m->n_nodes = hd.n_nodes; m->n_tris = hd.n_tris; m->n_faces = hd.n_faces; m->n_verts = hd.n_verts;
    m->max_depth = hd.max_depth; m->sah = hd.sah;
    for (int k = 0; k < 3; k++) m->abs_max[k] = hd.abs_max[k];
    cudaError_t e = cudaMalloc((void**)&m->d_nodes, sizeof(B2Node8) * (size_t)hd.n_nodes);
    if (e == cudaSuccess) e = cudaMalloc((void**)&m->d_tris, sizeof(B2Tri) * (size_t)hd.n_tris);
    if (e == cudaSuccess) e = cudaMemcpy(m->d_nodes, nodes, sizeof(B2Node8) * (size_t)hd.n_nodes, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMemcpy(m->d_tris, reinterpret_cast<const char*>(nodes) + sizeof(B2Node8) * (size_t)hd.n_nodes, sizeof(B2Tri) * (size_t)hd.n_tris, cudaMemcpyHostToDevice);
    if (e != cudaSuccess) { if (m->d_nodes) cudaFree(m->d_nodes); if (m->d_tris) cudaFree(m->d_tris); delete m; (void)cudaGetLastError(); return fail(B2_ERR_CUDA, "BVH blob upload failed: %s", cudaGetErrorString(e)); }
    m->build_ms = std::chrono::duration<float, std::milli>(std::chrono::steady_clock::now() - t0).count();
    *out = m;
    return B2_OK;
}

static void mesh_unref(b2_mesh* m)
{
    if (!m || m->refs.fetch_sub(1) != 1) return;
    cudaSetDevice(m->device);
    if (m->d_nodes) cudaFree(m->d_nodes);
    if (m->d_tris) cudaFree(m->d_tris);
    if (m->d_faces) cudaFree(m->d_faces);
    delete m;
    (void)cudaGetLastError();
}
// Drops the creator's reference.  Handles created on the map keep it alive (rm::EmbreeMapPtr is a shared_ptr in the reference as well,
// micp_localization.cpp:545), so the order in which a garbage collector destroys map and handles does not matter.
extern "C" int b2_mesh_destroy(b2_mesh* m) { mesh_unref(m); return B2_OK; }

extern "C" int b2_mesh_get_info(const b2_mesh* m, b2_mesh_info* info)
{
    NOTNULL(m); NOTNULL(info);
    info->n_faces = m->n_faces; info->n_vertices = m->n_verts; info->n_nodes = m->n_nodes; info->n_leaf_tris = m->n_tris; info->max_depth = m->max_depth;
    info->bvh_bytes = (uint64_t)m->n_nodes * sizeof(B2Node8) + (uint64_t)m->n_tris * sizeof(B2Tri);
    info->build_ms = m->build_ms; info->device = m->device; info->build_mode = m->build_mode; info->sah_cost = m->sah;
    return B2_OK;
}

static int intersect_impl(const b2_mesh* m, const float* origs, const float* dirs, uint32_t n, float tfar,
                          float* t_out, uint32_t* face_out, float* ng_out, uint8_t* hit_out, double* mean_nodes, double* mean_tris)
{
    NOTNULL(m);
    if (n == 0) return B2_OK;
    NOTNULL(origs); NOTNULL(dirs);
    CU(cudaSetDevice(m->device));
    DevBuf<float> d_o, d_d, d_t, d_ng; DevBuf<uint32_t> d_f; DevBuf<uint8_t> d_h; DevBuf<unsigned long long> d_c;
    int rc = B2_OK;
    auto cleanup = [&]() { d_o.release(); d_d.release(); d_t.release(); d_ng.release(); d_f.release(); d_h.release(); d_c.release(); };
    if ((rc = d_o.reserve(3 * (size_t)n)) || (rc = d_d.reserve(3 * (size_t)n)) || (rc = d_t.reserve(n)) || (rc = d_ng.reserve(3 * (size_t)n)) ||
        (rc = d_f.reserve(n)) || (rc = d_h.reserve(n)) || (rc = d_c.reserve(2))) { cleanup(); return rc; }
    cudaError_t e = cudaMemcpy(d_o.p, origs, sizeof(float) * 3 * (size_t)n, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMemcpy(d_d.p, dirs, sizeof(float) * 3 * (size_t)n, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMemset(d_c.p, 0, 2 * sizeof(unsigned long long));
    if (e == cudaSuccess) {
        const uint32_t grid = (n + 127) / 128;
        if (mean_nodes || mean_tris) k_intersect<true><<<grid, 128>>>(m->view(), d_o.p, d_d.p, n, tfar, d_t.p, d_f.p, d_ng.p, d_h.p, d_c.p);
        else k_intersect<false><<<grid, 128>>>(m->view(), d_o.p, d_d.p, n, tfar, d_t.p, d_f.p, d_ng.p, d_h.p, d_c.p);
        g_launches.fetch_add(1);
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
    if (e == cudaSuccess && t_out) e = cudaMemcpy(t_out, d_t.p, sizeof(float) * n, cudaMemcpyDeviceToHost);
    if (e == cudaSuccess && face_out) e = cudaMemcpy(face_out, d_f.p, sizeof(uint32_t) * n, cudaMemcpyDeviceToHost);
    if (e == cudaSuccess && ng_out) e = cudaMemcpy(ng_out, d_ng.p, sizeof(float) * 3 * (size_t)n, cudaMemcpyDeviceToHost);
    if (e == cudaSuccess && hit_out) e = cudaMemcpy(hit_out, d_h.p, n, cudaMemcpyDeviceToHost);
    unsigned long long c[2] = {0, 0};
    if (e == cudaSuccess && (mean_nodes || mean_tris)) e = cudaMemcpy(c, d_c.p, sizeof(c), cudaMemcpyDeviceToHost);
    cleanup();
    if (e != cudaSuccess) return fail(B2_ERR_CUDA, "b2_mesh_intersect: %s", cudaGetErrorString(e));
    if (mean_nodes) *mean_nodes = (double)c[0] / (double)n;
    if (mean_tris) *mean_tris = (double)c[1] / (double)n;
    return B2_OK;
}

extern "C" int b2_mesh_intersect(const b2_mesh* m, const float* origs, const float* dirs, uint32_t n, float tfar,
                                 float* t_out, uint32_t* face_out, float* ng_out, uint8_t* hit_out)
{
    return intersect_impl(m, origs, dirs, n, tfar, t_out, face_out, ng_out, hit_out, nullptr, nullptr);
}
extern "C" int b2_mesh_intersect_stats(const b2_mesh* m, const float* origs, const float* dirs, uint32_t n, float tfar, double* mean_nodes, double* mean_tris)
{
    double a = 0, b = 0;
    int rc = intersect_impl(m, origs, dirs, n, tfar, nullptr, nullptr, nullptr, nullptr, &a, &b);
    if (rc == B2_OK) { if (mean_nodes) *mean_nodes = a; if (mean_tris) *mean_tris = b; }
    return rc;
}

// ---------------------------------------------------------------------------------------------------------------------
// RCC handle
// ---------------------------------------------------------------------------------------------------------------------
#define B2_RING 8                // correctOnce calls that may be in flight per handle (b2_rcc_correct_once_async)
struct HostPin {            // pinned (mapped) staging for small results
    b2_transform T[3]; b2_cross_stats S[2]; IcpState icp;
    uint4 chunks[B2_RING][B2_ICP_RESULT_CHUNKS + 1];   // results of k_icp_loop: 16-byte chunks {3 payload words, sequence number} written by the kernel
    IcpResult res[B2_RING];                         // D2H staging of the non-spin path
    unsigned long long dbg[8];
    unsigned int flag_src[B2_RING];                 // source words of the "scan copy complete" flag copies
};

// What is still to be collected from an enqueued correctOnce (b2_rcc_correct_once_async .. _wait)
struct PendingCall {
    int kind = 0;                       // 0: result already in `res`, 1: spin on the mapped chunks, 2: D2H copy of d_res enqueued (stream sync), 3: D2H copy of d_icp (multi-launch chain)
    unsigned int seq = 0; int slot = 0;
    bool barrier_used = false, rerun = false;
    IcpLaunch launch{}; size_t smem = 0; int grid = 0;      // kept for the cooperative re-run after a barrier abort:
    b2_rcc* sensors[B2_MAX_SENSORS] = {nullptr, nullptr, nullptr, nullptr}; b2_transform Tbm[B2_MAX_SENSORS];   //   the finds are repeated as well (later calls overwrote the model buffers)
    IcpResult res{};
};

struct b2_rcc {
    b2_mesh* map = nullptr; cudaStream_t stream = 0;
    b2_transform Tsb{};
    bool has_model = false; uint32_t n = 0, width = 0, height = 0, n_origs = 1; float range_min = 0.f, range_max = 0.f;
    float max_dist = 1.0f, adaptive_max_dist_min = 0.15f;
    DevBuf<float> d_dirs, d_origs;
    DevBuf<float> d_dpts; DevBuf<uint8_t> d_dmask; uint32_t n_dataset = 0; DevBuf<float> d_ranges_in;
    DevBuf<float> d_mpts, d_mnrm, d_mranges; DevBuf<uint8_t> d_mhits; DevBuf<uint32_t> d_mfaces; uint32_t n_model = 0; bool found = false;
    DevBuf<double> d_partials; DevBuf<unsigned int> d_ticket; DevBuf<b2_cross_stats> d_stats; DevBuf<IcpState> d_icp;
    DevBuf<IcpResult> d_res; DevBuf<unsigned long long> d_dbg;
    DevBuf<b2_transform> d_poses, d_tdelta; DevBuf<uint32_t> d_ncorr; DevBuf<b2_cross_stats> d_bstats;
    HostPin* pin = nullptr; uint4* pin_chunks_dev = nullptr;
    int red_grid = 0;
    int fused_grid = 0;                 // blocks of k_icp_loop, one per SM (0: a whole-grid barrier is not available on this device)
    int smem_u_cap = 0;                 // pairs per thread k_icp_loop can keep in shared memory (beyond the two in registers)
    int exec_mode = 2;                  // b2_rcc_set_exec_mode: 2 software grid barrier + programmatic launch (default), 1 cooperative launch, 0 one launch per reduction
    bool pdl_next = false, pdl_armed = false;   // the next find is followed by k_icp_loop launched with programmatic stream serialization / the find let it start early
    DevBuf<uint32_t> d_tile_cost; DevBuf<uint16_t> d_tile_perm; uint32_t perm_tiles = 0, cost_tiles = 0;    // tile schedule of k_rcc_find: tile durations of the last launch (cost_tiles of them if it recorded any), order for the next (always a permutation of perm_tiles tiles)
    DevBuf<unsigned int> d_find_tickets; unsigned int find_ticket = 0; uint32_t find_grid = 0;   // k_rcc_find's tile queue: device counter, its value at the next launch, grid of the last launch
    DevBuf<uint8_t> d_cloud; bool model_from_cloud = false;      // b2_rcc_set_cloud_o1dn: uploaded host cloud; the model came from that call (its tile schedule carries over)
    b2_spherical_model sph{}; bool model_spherical = false;    // the model b2_rcc_set_model_spherical set, while it is the current one (b2_rcc_set_cloud_spherical bins into it)
    DevBuf<unsigned long long> d_scan_keys;                     // b2_rcc_set_cloud_spherical: one key per cell, all 0 between calls
    unsigned long long n_reruns = 0;                            // calls that were run again through the cooperative launch (exchange abort: co-residency or range)
    uint32_t loop_geom[2 + 4 * B2_MAX_SENSORS] = {};            // last fused call: sensors, grid, per sensor {n, blk0, nblk, smem_u} (b2_rcc_debug_loop_geometry)
    DevBuf<unsigned int> d_bar; unsigned int zc_seq = 0;        // [0] = "scan copy complete" flag (value: zc_seq of the call), [1] = abort word of the ICP loop
    DevBuf<unsigned long long> d_slots; unsigned int tag_base = 0; // exchange buffers of the ICP loop (icp_loop.cuh: accumulators, base, FP64 slots); round number of the next launch
    unsigned int seq = 0;               // sequence number of the last k_icp_loop launch (carried by every result chunk)
    std::deque<PendingCall> pending;    // enqueued, not yet collected (oldest first), at most B2_RING
    unsigned int slot_counter = 0;
    DevBuf<unsigned char> d_chain;      // b2_micp_correct with this handle in the lead: IcpChainState, then one b2_micp_step per correction
    DevBuf<double> d_cov_part; DevBuf<unsigned int> d_cov_ticket; DevBuf<b2_micp_covariance> d_cov_rec;   // b2_micp_pose_covariance with this handle in the lead
    bool timing = false; cudaEvent_t ev[3] = {nullptr, nullptr, nullptr}; bool timing_valid = false;
    cudaStream_t aux = nullptr; cudaEvent_t ev_aux = nullptr;     // side stream: scan upload + unpack overlap the find kernel
    cudaEvent_t ev_join = nullptr;      // multi-sensor correctOnce: orders this handle's stream against the lead handle's
    uint32_t n_ranges_in = 0;           // real ranges resident in d_ranges_in (set_ranges / correct_once_ranges), needed by b2_rcc_segment
    DevBuf<uint32_t> d_seg_counts, d_seg_offsets, d_seg_totals; DevBuf<float> d_seg_scan, d_seg_map; DevBuf<uint8_t> d_seg_labels;
    // caller-owned device memory (b2_rcc_bind_dataset / b2_rcc_bind_model_buffers): the reference's public `dataset` member and protected
    // `model_buffers_` (Correspondences.hpp:24,81-85) live in rm::Memory<.., VRAM_CUDA>; a subclass binds them so that nothing is copied
    const float* b_dpts = nullptr; const uint8_t* b_dmask = nullptr;        // borrowed dataset (read only)
    float* b_mpts = nullptr; float* b_mnrm = nullptr; uint8_t* b_mhits = nullptr; uint32_t b_mcap = 0;
    const float* dpts() const { return b_dpts ? b_dpts : d_dpts.p; }
    const uint8_t* dmask() const { return b_dpts ? b_dmask : d_dmask.p; }
    float* mpts() const { return b_mpts ? b_mpts : d_mpts.p; }
    float* mnrm() const { return b_mpts ? b_mnrm : d_mnrm.p; }
    uint8_t* mhits() const { return b_mpts ? b_mhits : d_mhits.p; }
    bool cpc_skip_masked = false;       // b2_rcc_set_cpc_options
    uint32_t sim_opts = 0;              // b2_rcc_set_sim_options
    int corr_type = B2_CORR_RCC;        // B2_CORR_CPC: find() is a closest-point query per dataset point (CPCEmbree), no sensor model needed
    uint32_t work_n() const { return corr_type == B2_CORR_CPC ? n_dataset : n; }   // correspondences per find
};

// Per device: k_icp_loop launches with the software grid barrier must never overlap each other (two partially resident grids would wait
// for each other's SMs).  Handles on different streams are therefore chained through one event per device; a single handle on a single
// stream -- the common case -- pays nothing (stream order already serialises its launches).
struct DeviceCtx { std::mutex m; cudaEvent_t loop_done = nullptr; bool recorded = false, multi = false; int n_handles = 0; b2_rcc* last = nullptr; cudaStream_t last_stream = nullptr; };
static DeviceCtx g_dev[64];

static b2_transform tf_identity_pod() { b2_transform T; memset(&T, 0, sizeof(T)); T.R.w = 1.0f; return T; }

extern "C" int b2_rcc_destroy(b2_rcc* h);

// device resources of a fresh handle; any failure leaves the handle in a state b2_rcc_destroy can clean up
static int rcc_init(b2_rcc* h)
{
    b2_mesh* map = h->map;
    cudaDeviceProp prop; CU(cudaGetDeviceProperties(&prop, map->device));
    h->red_grid = prop.multiProcessorCount;
    {
        // k_icp_loop: one 512-thread block per SM; the shared memory the block does not need statically holds pairs (18 KB per pair-per-thread)
        int coop = 0, per_sm = 0, optin = 0;
        cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, map->device);
        cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, map->device);
        cudaFuncAttributes fa{}, fb{};
        if (cudaFuncGetAttributes(&fa, k_icp_loop<false>) == cudaSuccess && cudaFuncGetAttributes(&fb, k_icp_loop<true>) == cudaSuccess) {
            const int room = optin - (int)std::max(fa.sharedSizeBytes, fb.sharedSizeBytes) - 1024;       // both variants must accept the same launch
            h->smem_u_cap = std::max(0, room / (9 * B2_ICP_BLOCK * 4));
            const int dyn = h->smem_u_cap * 9 * B2_ICP_BLOCK * 4;
            if (dyn > 0 && (cudaFuncSetAttribute(k_icp_loop<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, dyn) != cudaSuccess ||
                            cudaFuncSetAttribute(k_icp_loop<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, dyn) != cudaSuccess)) h->smem_u_cap = 0;
        }
        if (coop && cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_icp_loop<true>, B2_ICP_BLOCK, (size_t)h->smem_u_cap * 9 * B2_ICP_BLOCK * 4) == cudaSuccess && per_sm > 0)
            h->fused_grid = std::min(prop.multiProcessorCount, B2_ICP_MAX_GRID);      // one block per SM
        (void)cudaGetLastError();
    }
    { const char* e = getenv("B2_FUSED"); h->exec_mode = e ? atoi(e) : 2; if (h->exec_mode < 0 || h->exec_mode > 2) h->exec_mode = 2; }
    RES(h->d_partials.reserve((size_t)(B2_NACC + 1) * std::max(h->red_grid, 2 * B2_ICP_MAX_GRID))); RES(h->d_ticket.reserve(1)); RES(h->d_stats.reserve(1)); RES(h->d_icp.reserve(1));
    RES(h->d_bar.reserve(2)); RES(h->d_res.reserve(1)); RES(h->d_dbg.reserve(16 + 4 * B2_ICP_MAX_GRID)); RES(h->d_slots.reserve((size_t)B2_ICP_ACC_WORDS + B2_ICP_BASE_WORDS + B2_ICP_SLOT_WORDS));
    RES(h->d_find_tickets.reserve(1));
    CU(cudaMemset(h->d_ticket.p, 0, sizeof(unsigned int)));
    CU(cudaMemset(h->d_find_tickets.p, 0, sizeof(unsigned int)));
    CU(cudaMemset(h->d_bar.p, 0, 2 * sizeof(unsigned int)));
    CU(cudaMemset(h->d_slots.p, 0, ((size_t)B2_ICP_ACC_WORDS + B2_ICP_BASE_WORDS + B2_ICP_SLOT_WORDS) * sizeof(unsigned long long)));      // accumulators and base agree (0); slot tag 0 is never used
    CU(cudaMemset(h->d_dbg.p, 0, (16 + 4 * B2_ICP_MAX_GRID) * sizeof(unsigned long long)));
    CU(cudaHostAlloc((void**)&h->pin, sizeof(HostPin), cudaHostAllocMapped));
    memset((void*)h->pin, 0, sizeof(HostPin));
    CU(cudaHostGetDevicePointer((void**)&h->pin_chunks_dev, (void*)&h->pin->chunks[0][0], 0));
    CU(cudaStreamCreateWithFlags(&h->aux, cudaStreamNonBlocking));
    CU(cudaEventCreateWithFlags(&h->ev_aux, cudaEventDisableTiming));
    CU(cudaEventCreateWithFlags(&h->ev_join, cudaEventDisableTiming));
    return B2_OK;
}

extern "C" int b2_rcc_create(b2_mesh* map, b2_rcc** out)
{
    NOTNULL(out); *out = nullptr;
    if (!map) return fail(B2_ERR_NO_MAP, "NO MAP");
    CU(cudaSetDevice(map->device));
    b2_rcc* h = new (std::nothrow) b2_rcc();
    if (!h) return fail(B2_ERR_OOM, "out of host memory");
    h->map = map; h->Tsb = tf_identity_pod();
    map->refs.fetch_add(1);             // released in b2_rcc_destroy
    { DeviceCtx& dc = g_dev[map->device & 63]; std::lock_guard<std::mutex> lk(dc.m); if (++dc.n_handles > 1) dc.multi = true; }
    const int rc = rcc_init(h);
    if (rc != B2_OK) { b2_rcc_destroy(h); return rc; }      // the error text of the failing call stays in b2_last_error
    *out = h;
    return B2_OK;
}

extern "C" int b2_rcc_destroy(b2_rcc* h)
{
    if (!h) return B2_OK;
    cudaSetDevice(h->map->device);
    cudaStreamSynchronize(h->stream);
    h->d_dirs.release(); h->d_origs.release(); h->d_dpts.release(); h->d_dmask.release(); h->d_ranges_in.release();
    h->d_mpts.release(); h->d_mnrm.release(); h->d_mranges.release(); h->d_mhits.release(); h->d_mfaces.release();
    h->d_partials.release(); h->d_ticket.release(); h->d_stats.release(); h->d_icp.release(); h->d_bar.release(); h->d_res.release(); h->d_dbg.release(); h->d_slots.release(); h->d_tile_cost.release(); h->d_tile_perm.release(); h->d_find_tickets.release();
    h->d_chain.release(); h->d_cloud.release(); h->d_scan_keys.release();
    h->d_cov_part.release(); h->d_cov_ticket.release(); h->d_cov_rec.release();
    { DeviceCtx& dc = g_dev[h->map->device & 63]; std::lock_guard<std::mutex> lk(dc.m); dc.n_handles--; if (dc.last == h) { dc.last = nullptr; dc.recorded = false; } }
    h->d_poses.release(); h->d_tdelta.release(); h->d_ncorr.release(); h->d_bstats.release();
    if (h->pin) cudaFreeHost(h->pin);
    if (h->aux) { cudaStreamSynchronize(h->aux); cudaStreamDestroy(h->aux); }
    if (h->ev_aux) cudaEventDestroy(h->ev_aux);
    if (h->ev_join) cudaEventDestroy(h->ev_join);
    for (int i = 0; i < 3; i++) if (h->ev[i]) cudaEventDestroy(h->ev[i]);
    h->d_seg_counts.release(); h->d_seg_offsets.release(); h->d_seg_totals.release(); h->d_seg_scan.release(); h->d_seg_map.release(); h->d_seg_labels.release();
    b2_mesh* map = h->map;
    delete h;
    (void)cudaGetLastError();
    mesh_unref(map);
    return B2_OK;
}

extern "C" int b2_rcc_enable_timing(b2_rcc* h, int enable)
{
    NOTNULL(h);
    CU(cudaSetDevice(h->map->device));
    if (enable) for (int i = 0; i < 3; i++) if (!h->ev[i]) CU(cudaEventCreate(&h->ev[i]));
    h->timing = enable != 0; h->timing_valid = false;
    return B2_OK;
}
extern "C" int b2_rcc_last_timing(b2_rcc* h, float* find_ms, float* reduce_ms)
{
    NOTNULL(h);
    if (!h->timing || !h->timing_valid) return fail(B2_ERR_INVALID, "no timing recorded (b2_rcc_enable_timing + a correct_once call first)");
    CU(cudaSetDevice(h->map->device));
    CU(cudaEventSynchronize(h->ev[2]));
    float a = 0.f, b = 0.f;
    CU(cudaEventElapsedTime(&a, h->ev[0], h->ev[1])); CU(cudaEventElapsedTime(&b, h->ev[1], h->ev[2]));
    if (find_ms) *find_ms = a; if (reduce_ms) *reduce_ms = b;
    return B2_OK;
}

// profiling aid (not part of the public header): SM-clock durations of the last reduction's phases
extern "C" __attribute__((visibility("default"))) int b2_rcc_debug_clocks(b2_rcc* h, unsigned long long* out16)
{
    NOTNULL(h); NOTNULL(out16);
    CU(cudaSetDevice(h->map->device));
    CU(cudaStreamSynchronize(h->stream));
    CU(cudaMemcpy(out16, h->d_dbg.p, 16 * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
    return B2_OK;
}
// test aid (not part of the public header): how many correctOnce calls of this handle were run again through the cooperative launch
extern "C" __attribute__((visibility("default"))) int b2_rcc_debug_reruns(b2_rcc* h, unsigned long long* out)
{
    NOTNULL(h); NOTNULL(out);
    *out = h->n_reruns;
    return B2_OK;
}
// test aid (not part of the public header): the launch shape of k_icp_loop, so that tests can place pair counts on its tier boundaries.
// out[0] = blocks of a full grid, out[1] = pairs per thread shared memory can hold, out[2] = sensors of this handle's last fused call (0: none yet),
// out[3] = its grid, out[4 + 4k ..] = sensor k's {pairs, first block, blocks, pairs per thread in shared memory}; 4 + 4 * B2_MAX_SENSORS words
extern "C" __attribute__((visibility("default"))) int b2_rcc_debug_loop_geometry(b2_rcc* h, uint32_t* out)
{
    NOTNULL(h); NOTNULL(out);
    out[0] = (uint32_t)h->fused_grid; out[1] = (uint32_t)h->smem_u_cap;
    memcpy(out + 2, h->loop_geom, sizeof(h->loop_geom));
    return B2_OK;
}
// test aid (not part of the public header): the tile order the next find of this handle will use (host copy; *n_tiles = 0 when the schedule is off)
extern "C" __attribute__((visibility("default"))) int b2_rcc_debug_tile_perm(b2_rcc* h, uint16_t* out, uint32_t capacity, uint32_t* n_tiles)
{
    NOTNULL(h); NOTNULL(n_tiles);
    CU(cudaSetDevice(h->map->device));
    CU(cudaStreamSynchronize(h->stream));
    *n_tiles = h->perm_tiles;
    if (out && h->perm_tiles && capacity >= h->perm_tiles) CU(cudaMemcpy(out, h->d_tile_perm.p, h->perm_tiles * sizeof(uint16_t), cudaMemcpyDeviceToHost));
    return B2_OK;
}
// test aid (not part of the public header): host copies of the sensor model's ray directions (3 n floats) and the resident ranges (n floats);
// either may be null.  *n receives the model's ray count.
extern "C" __attribute__((visibility("default"))) int b2_rcc_debug_model_tables(b2_rcc* h, float* dirs, float* ranges, uint32_t* n)
{
    NOTNULL(h); NOTNULL(n);
    CU(cudaSetDevice(h->map->device));
    CU(cudaStreamSynchronize(h->stream));
    *n = h->has_model ? h->n : 0;
    if (dirs && *n) CU(cudaMemcpy(dirs, h->d_dirs.p, 3 * sizeof(float) * *n, cudaMemcpyDeviceToHost));
    if (ranges && *n && h->n_ranges_in == *n) CU(cudaMemcpy(ranges, h->d_ranges_in.p, sizeof(float) * *n, cudaMemcpyDeviceToHost));
    return B2_OK;
}
// test aid (not part of the public header): k_rcc_find's tile queue.  set != nullptr: after the stream drains, the device counter and the
// handle's copy both become *set (a test starts them just below 2^32 to cross the wrap).  out (may be null): {device counter, handle's
// value for the next launch, grid of the last launch}.
extern "C" __attribute__((visibility("default"))) int b2_rcc_debug_find_tickets(b2_rcc* h, const unsigned int* set, unsigned int* out)
{
    NOTNULL(h);
    CU(cudaSetDevice(h->map->device));
    CU(cudaStreamSynchronize(h->stream));
    if (set) { CU(cudaMemcpy(h->d_find_tickets.p, set, sizeof(unsigned int), cudaMemcpyHostToDevice)); h->find_ticket = *set; }
    if (out) { CU(cudaMemcpy(out, h->d_find_tickets.p, sizeof(unsigned int), cudaMemcpyDeviceToHost)); out[1] = h->find_ticket; out[2] = h->find_grid; }
    return B2_OK;
}
// test aid (not part of the public header): host copy of the tile durations the last find recorded (*n_tiles = 0 when it recorded none);
// poison != 0: afterwards every entry is set to 0xffffffff on the device, so that the next find must rewrite each one
extern "C" __attribute__((visibility("default"))) int b2_rcc_debug_tile_cost(b2_rcc* h, uint32_t* out, uint32_t capacity, uint32_t* n_tiles, int poison)
{
    NOTNULL(h); NOTNULL(n_tiles);
    CU(cudaSetDevice(h->map->device));
    CU(cudaStreamSynchronize(h->stream));
    *n_tiles = h->cost_tiles;
    if (out && h->cost_tiles && capacity >= h->cost_tiles) CU(cudaMemcpy(out, h->d_tile_cost.p, h->cost_tiles * sizeof(uint32_t), cudaMemcpyDeviceToHost));
    if (poison && h->cost_tiles) CU(cudaMemset(h->d_tile_cost.p, 0xff, h->cost_tiles * sizeof(uint32_t)));
    return B2_OK;
}
// make PROFILE=1 only: per block {ns at publish, ns at collect, cycles since the block reduce at publish, at collect} of iteration 1
extern "C" __attribute__((visibility("default"))) int b2_rcc_debug_blocks(b2_rcc* h, unsigned long long* out /* 4 * B2_ICP_MAX_GRID */)
{
    NOTNULL(h); NOTNULL(out);
    CU(cudaSetDevice(h->map->device));
    CU(cudaStreamSynchronize(h->stream));
    CU(cudaMemcpy(out, h->d_dbg.p + 16, 4 * B2_ICP_MAX_GRID * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
    return B2_OK;
}

// profiling aid (not part of the public header): per-tile {start, end} %globaltimer stamps of the NEXT k_rcc_find launches.
// buf_dev: device buffer of 2 x ceil(n_rays / 32) u64 (one pair per tile of 32 rays), or nullptr to switch the stamps off again.
extern "C" __attribute__((visibility("default"))) int b2_rcc_debug_find_warp_times(b2_rcc* h, unsigned long long* buf_dev)
{
    NOTNULL(h);
    CU(cudaSetDevice(h->map->device));
    CU(cudaStreamSynchronize(h->stream));
    CU(cudaMemcpyToSymbol(g_find_warp_times, &buf_dev, sizeof(buf_dev)));
    return B2_OK;
}

extern "C" int b2_rcc_set_stream(b2_rcc* h, void* s) { NOTNULL(h); h->stream = (cudaStream_t)s; return B2_OK; }
extern "C" int b2_rcc_set_tsb(b2_rcc* h, const b2_transform* Tsb) { NOTNULL(h); NOTNULL(Tsb); h->Tsb = *Tsb; return B2_OK; }
extern "C" int b2_rcc_set_params(b2_rcc* h, float max_dist, float amin) { NOTNULL(h); h->max_dist = max_dist; h->adaptive_max_dist_min = amin; return B2_OK; }

// upload sensor-frame ray tables.  Direction tables are evaluated on the host with libm cosf/sinf exactly like
// rmagine's SphericalModel::getDirection does on the CPU path (witness rmcl_ros/src/util/conversions.cpp:174-188), so the
// rays are bit-identical to the reference's; this runs once per setModel, not per scan.
static int set_model_tables(b2_rcc* h, uint32_t w, uint32_t hgt, const float* origs, uint32_t n_origs, const float* dirs, float rmin, float rmax)
{
    CU(cudaSetDevice(h->map->device));
    const size_t n = (size_t)w * hgt;
    if (n == 0) { h->has_model = true; h->n = 0; h->width = w; h->height = hgt; h->model_from_cloud = false; h->model_spherical = false; return B2_OK; }   // zero-size model: find() silently returns (RCCOptix.cpp:30-34)
    if (n > 0xffffffffu / 4) return fail(B2_ERR_INVALID, "model too large");
    RES(h->d_dirs.reserve(3 * n)); RES(h->d_origs.reserve(3 * (size_t)n_origs));
    CU(cudaStreamSynchronize(h->stream));
    CU(cudaMemcpy(h->d_dirs.p, dirs, sizeof(float) * 3 * n, cudaMemcpyHostToDevice));
    CU(cudaMemcpy(h->d_origs.p, origs, sizeof(float) * 3 * (size_t)n_origs, cudaMemcpyHostToDevice));
    h->has_model = true; h->n = (uint32_t)n; h->width = w; h->height = hgt; h->n_origs = n_origs; h->range_min = rmin; h->range_max = rmax;
    h->perm_tiles = 0;                                             // the tile schedule belongs to the previous model
    h->model_from_cloud = false; h->model_spherical = false;
    return B2_OK;
}

extern "C" int b2_rcc_set_model_spherical(b2_rcc* h, const b2_spherical_model* m)
{
    NOTNULL(h); NOTNULL(m);
    const size_t n = (size_t)m->phi_size * m->theta_size;
    if (n > 0xffffffffu / 4) return fail(B2_ERR_INVALID, "model too large");
    std::vector<float> dirs;
    try { dirs.resize(3 * n); } catch (const std::exception&) { return fail(B2_ERR_OOM, "out of host memory (%zu rays)", n); }
    for (uint32_t vid = 0; vid < m->phi_size; vid++) {
        const float phi = m->phi_min + (float)vid * m->phi_inc;
        const float cp = cosf(phi), sp = sinf(phi);
        for (uint32_t hid = 0; hid < m->theta_size; hid++) {
            const float theta = m->theta_min + (float)hid * m->theta_inc;
            float* d = &dirs[3 * ((size_t)vid * m->theta_size + hid)];
            d[0] = cp * cosf(theta); d[1] = cp * sinf(theta); d[2] = sp;
        }
    }
    const float o[3] = {0.f, 0.f, 0.f};
    RES(set_model_tables(h, m->theta_size, m->phi_size, o, 1, dirs.data(), m->range_min, m->range_max));
    h->sph = *m; h->model_spherical = true;
    return B2_OK;
}

extern "C" int b2_rcc_set_model_pinhole(b2_rcc* h, const b2_pinhole_model* m)
{
    NOTNULL(h); NOTNULL(m);
    const size_t n = (size_t)m->width * m->height;
    if (n > 0xffffffffu / 4) return fail(B2_ERR_INVALID, "model too large");
    std::vector<float> dirs;
    try { dirs.resize(3 * n); } catch (const std::exception&) { return fail(B2_ERR_OOM, "out of host memory (%zu rays)", n); }
    for (uint32_t vid = 0; vid < m->height; vid++)
        for (uint32_t hid = 0; hid < m->width; hid++) {
            const float px = ((float)hid - m->cx) / m->fx, py = ((float)vid - m->cy) / m->fy;
            const float nrm = sqrtf(px * px + py * py + 1.0f * 1.0f);
            const float ox = px / nrm, oy = py / nrm, oz = 1.0f / nrm;            // optical frame, normalised
            float* d = &dirs[3 * ((size_t)vid * m->width + hid)];
            d[0] = oz; d[1] = -ox; d[2] = -oy;                                     // x forward, y left, z up
        }
    const float o[3] = {0.f, 0.f, 0.f};
    return set_model_tables(h, m->width, m->height, o, 1, dirs.data(), m->range_min, m->range_max);
}

extern "C" int b2_rcc_set_model_o1dn(b2_rcc* h, uint32_t w, uint32_t hgt, const float orig[3], const float* dirs, float rmin, float rmax)
{
    NOTNULL(h); if ((size_t)w * hgt) { NOTNULL(orig); NOTNULL(dirs); }
    return set_model_tables(h, w, hgt, orig, 1, dirs, rmin, rmax);
}
extern "C" int b2_rcc_set_model_ondn(b2_rcc* h, uint32_t w, uint32_t hgt, const float* origs, const float* dirs, float rmin, float rmax)
{
    NOTNULL(h); if ((size_t)w * hgt) { NOTNULL(origs); NOTNULL(dirs); }
    return set_model_tables(h, w, hgt, origs, (uint32_t)((size_t)w * hgt), dirs, rmin, rmax);
}

extern "C" int b2_rcc_set_dataset(b2_rcc* h, const float* pts, const uint8_t* mask, uint32_t n, int src_is_device)
{
    NOTNULL(h);
    CU(cudaSetDevice(h->map->device));
    if (n) { NOTNULL(pts); }
    h->b_dpts = nullptr; h->b_dmask = nullptr;                                        // own buffers from now on
    RES(h->d_dpts.reserve(3 * (size_t)std::max(n, 1u))); RES(h->d_dmask.reserve(std::max(n, 1u)));
    const cudaMemcpyKind kind = src_is_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice;
    if (n) {
        CU(cudaMemcpyAsync(h->d_dpts.p, pts, sizeof(float) * 3 * (size_t)n, kind, h->stream));
        if (mask) CU(cudaMemcpyAsync(h->d_dmask.p, mask, n, kind, h->stream));
        else CU(cudaMemsetAsync(h->d_dmask.p, 1, n, h->stream));                  // empty mask == all valid (statistics_p2l semantics)
        if (!src_is_device) CU(cudaStreamSynchronize(h->stream));                 // caller may reuse its buffers
    }
    h->n_dataset = n;
    return B2_OK;
}

static int ranges_to_dataset(b2_rcc* h, const float* ranges, uint32_t n, int src_is_device)
{
    if (!h->has_model) return fail(B2_ERR_INVALID, "set_ranges before setModel");
    if (n != h->n) return fail(B2_ERR_INVALID, "ranges size %u != model size %u", n, h->n);
    if (n == 0) { h->n_dataset = 0; return B2_OK; }
    NOTNULL(ranges);
    h->b_dpts = nullptr; h->b_dmask = nullptr;
    RES(h->d_dpts.reserve(3 * (size_t)n)); RES(h->d_dmask.reserve(n)); RES(h->d_ranges_in.reserve(n));
    CU(cudaMemcpyAsync(h->d_ranges_in.p, ranges, sizeof(float) * n, src_is_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, h->stream));
    k_dataset_from_ranges<<<(n + 255) / 256, 256, 0, h->stream>>>(h->d_ranges_in.p, h->d_dirs.p, h->d_origs.p, h->n_origs, n, h->range_min, h->range_max, h->d_dpts.p, h->d_dmask.p);
    LAUNCHED();
    h->n_dataset = n; h->n_ranges_in = n;
    return B2_OK;
}

extern "C" int b2_rcc_set_ranges(b2_rcc* h, const float* ranges, uint32_t n, int src_is_device)
{
    NOTNULL(h);
    CU(cudaSetDevice(h->map->device));
    RES(ranges_to_dataset(h, ranges, n, src_is_device));
    if (!src_is_device) CU(cudaStreamSynchronize(h->stream));
    return B2_OK;
}

// The layout checks every cloud entry point makes before it reads a byte: x, y and z present, FLOAT32 or FLOAT64, little-endian, each
// field inside point_step, and -- when the call reads any point -- `bytes` reaching the end of the last point it reads (row last_row,
// column last_col).  *need receives that end (0 when nothing is read).  `who` prefixes every message; the two refs follow the messages
// on a missing field and on the datatype.
static int check_cloud_layout(const b2_cloud_layout* L, uint64_t bytes, bool reads, uint64_t last_row, uint64_t last_col, const char* who,
                              const char* no_field_ref, const char* datatype_ref, uint64_t* need)
{
    const uint32_t off[3] = {L->offset_x, L->offset_y, L->offset_z};
    if (off[0] == B2_CLOUD_NO_FIELD || off[1] == B2_CLOUD_NO_FIELD || off[2] == B2_CLOUD_NO_FIELD)
        return fail(B2_ERR_INVALID, "%s: the cloud has no x, y or z field%s", who, no_field_ref);
    if (L->datatype != 7 && L->datatype != 8)
        return fail(B2_ERR_INVALID, "%s: field x has datatype %u; FLOAT32 (7) and FLOAT64 (8) are read%s", who, (unsigned)L->datatype, datatype_ref);
    if (L->is_bigendian) return fail(B2_ERR_INVALID, "%s: big-endian clouds are not read", who);
    const uint32_t fsz = L->datatype == 8 ? 8u : 4u;
    for (int c = 0; c < 3; c++)
        if ((uint64_t)off[c] + fsz > L->point_step) return fail(B2_ERR_INVALID, "%s: field %c at offset %u ends beyond point_step %u", who, "xyz"[c], off[c], L->point_step);
    *need = 0;
    if (!reads) return B2_OK;
    const unsigned __int128 last = (unsigned __int128)last_row * L->row_step + (unsigned __int128)last_col * L->point_step +
                                   std::max(off[0], std::max(off[1], off[2])) + fsz;
    if (last > (unsigned __int128)bytes)
        return fail(B2_ERR_INVALID, "%s: %llu bytes given, the last point read ends at byte %llu", who, (unsigned long long)bytes,
                    last > (unsigned __int128)UINT64_MAX ? (unsigned long long)UINT64_MAX : (unsigned long long)last);
    *need = (uint64_t)last;
    return B2_OK;
}

// Pc2ToO1DnNode::convert + MICPO1DnSensorCUDA::unpackMessage + setModel (conversions.cpp:869-1073, scan_operations.cpp:41-143,
// MICPO1DnSensorCUDA.cpp:142-148,171-230) as one kernel.  Every check runs before anything of the handle changes: where the reference
// throws, divides by zero, underflows size_t or reads past the message, the call is refused.  A host cloud is uploaded whole up to the last
// byte the filter reads (one copy; scripts/bench_pointcloud.py measures it against the host path).
extern "C" int b2_rcc_set_cloud_o1dn(b2_rcc* h, const void* data, uint64_t bytes, const b2_cloud_layout* L, const b2_o1dn_cloud_filter* F, int src_is_device)
{
    NOTNULL(data); NOTNULL(L); NOTNULL(F);          // the arguments are checked before the handle: the checks need no device
    if (F->height_increment == 0 || F->width_increment == 0) return fail(B2_ERR_INVALID, "set_cloud_o1dn: increment 0 (height %u, width %u)", F->height_increment, F->width_increment);
    if ((uint64_t)F->height_skip_begin + F->height_skip_end > L->height || (uint64_t)F->width_skip_begin + F->width_skip_end > L->width)
        return fail(B2_ERR_INVALID, "set_cloud_o1dn: skips %u+%u of height %u / %u+%u of width %u", F->height_skip_begin, F->height_skip_end, L->height,
                    F->width_skip_begin, F->width_skip_end, L->width);
    const uint64_t w_out = (L->width - F->width_skip_begin - F->width_skip_end) / F->width_increment;
    const uint64_t h_out = (L->height - F->height_skip_begin - F->height_skip_end) / F->height_increment;
    const uint64_t n = w_out * h_out;
    if (n > 0xffffffffu / 4) return fail(B2_ERR_INVALID, "set_cloud_o1dn: model too large (%llu rays)", (unsigned long long)n);
    uint64_t need = 0;
    RES(check_cloud_layout(L, bytes, n != 0, n ? (h_out - 1) * F->height_increment + F->height_skip_begin : 0, n ? (w_out - 1) * F->width_increment + F->width_skip_begin : 0,
                           "set_cloud_o1dn", " (\"NO POINT FIELD IN CLOUD!\", conversions.cpp:955-958)", " (conversions.cpp:977-990)", &need));
    const uint32_t off[3] = {L->offset_x, L->offset_y, L->offset_z};
    NOTNULL(h);
    CU(cudaSetDevice(h->map->device));
    const bool keep_schedule = h->model_from_cloud && h->has_model && h->width == (uint32_t)w_out && h->height == (uint32_t)h_out;
    if (n) {
        RES(h->d_dirs.reserve(3 * n)); RES(h->d_origs.reserve(3)); RES(h->d_dpts.reserve(3 * n)); RES(h->d_dmask.reserve(n)); RES(h->d_ranges_in.reserve(n));
        const uint8_t* src = static_cast<const uint8_t*>(data);
        if (!src_is_device) {
            RES(h->d_cloud.reserve(need));
            CU(cudaMemcpyAsync(h->d_cloud.p, data, need, cudaMemcpyHostToDevice, h->stream));
            src = h->d_cloud.p;
        }
        CU(cudaMemsetAsync(h->d_origs.p, 0, 3 * sizeof(float), h->stream));
        CloudO1Dn c;
        c.w_out = (uint32_t)w_out; c.h_out = (uint32_t)h_out; c.row_step = L->row_step; c.point_step = L->point_step;
        for (int k = 0; k < 3; k++) c.off[k] = off[k];
        c.f64 = L->datatype == 8 ? 1u : 0u;
        c.h_inc = F->height_increment; c.h_begin = F->height_skip_begin; c.w_inc = F->width_increment; c.w_begin = F->width_skip_begin;
        c.range_min = F->range_min; c.range_max = F->range_max;
        k_o1dn_from_cloud<<<(uint32_t)((n + 255) / 256), 256, 0, h->stream>>>(src, c, h->d_dirs.p, h->d_ranges_in.p, h->d_dpts.p, h->d_dmask.p);
        LAUNCHED();
    }
    h->has_model = true; h->n = (uint32_t)n; h->width = (uint32_t)w_out; h->height = (uint32_t)h_out; h->n_origs = 1;
    h->range_min = F->range_min; h->range_max = F->range_max;
    if (!keep_schedule) h->perm_tiles = 0;
    h->model_from_cloud = true; h->model_spherical = false;
    h->b_dpts = nullptr; h->b_dmask = nullptr;
    h->n_dataset = (uint32_t)n; h->n_ranges_in = (uint32_t)n;
    if (!src_is_device) CU(cudaStreamSynchronize(h->stream));
    return B2_OK;
}

static bool all_finite(const float* v, int n)
{
    for (int k = 0; k < n; k++) if (!std::isfinite(v[k])) return false;
    return true;
}

// Pc2ToScanNode::convert + fillEmpty + MICPSphericalSensorCUDA::unpackMessage (pc2_to_scan.cpp:105-213, scan_operations.cpp:25-39,
// MICPSphericalSensorCUDA.cpp:176-235) as two kernels on the handle's stream with no host round trip between them.  The model stays the
// one b2_rcc_set_model_spherical set: its direction table and find's tile schedule are kept.  Every check runs before anything of the
// handle changes.  A host cloud is uploaded whole up to the last byte read (scripts/bench_pointcloud_scan.py measures the call).
extern "C" int b2_rcc_set_cloud_spherical(b2_rcc* h, const void* data, uint64_t bytes, const b2_cloud_layout* L, const b2_transform* T, int src_is_device)
{
    NOTNULL(L); NOTNULL(T);                         // the arguments are checked before the handle: the checks need no device
    const uint64_t n_points = (uint64_t)L->width * L->height;
    if (n_points) NOTNULL(data);
    if (n_points > 0xfffffffeull) return fail(B2_ERR_INVALID, "set_cloud_spherical: %llu points, at most 2^32 - 2 are read", (unsigned long long)n_points);
    uint64_t need = 0;
    RES(check_cloud_layout(L, bytes, n_points != 0, n_points ? L->height - 1 : 0, n_points ? L->width - 1 : 0, "set_cloud_spherical", "",
                           " (pc2_to_scan.cpp:167-184)", &need));
    const uint32_t off[3] = {L->offset_x, L->offset_y, L->offset_z};
    const float Tv[7] = {T->R.x, T->R.y, T->R.z, T->R.w, T->t.x, T->t.y, T->t.z};
    if (!all_finite(Tv, 7)) return fail(B2_ERR_INVALID, "set_cloud_spherical: T_sensor_cloud is not finite");
    NOTNULL(h);
    if (!h->model_spherical) return fail(B2_ERR_INVALID, "set_cloud_spherical: the handle's current model is not spherical (b2_rcc_set_model_spherical first)");
    const b2_spherical_model& m = h->sph;
    const float mv[6] = {m.phi_min, m.phi_inc, m.theta_min, m.theta_inc, m.range_min, m.range_max};
    if (!all_finite(mv, 6)) return fail(B2_ERR_INVALID, "set_cloud_spherical: the spherical model has a non-finite parameter");
    if ((m.phi_inc == 0.f && m.phi_size > 1) || (m.theta_inc == 0.f && m.theta_size > 1))
        return fail(B2_ERR_INVALID, "set_cloud_spherical: model increment 0 with more than one bin (phi %u, theta %u)", m.phi_size, m.theta_size);
    CU(cudaSetDevice(h->map->device));
    const uint32_t n = h->n;
    if (n == 0) { h->n_dataset = 0; return B2_OK; }                             // as b2_rcc_set_ranges on a zero-size model
    RES(h->d_dpts.reserve(3 * (size_t)n)); RES(h->d_dmask.reserve(n)); RES(h->d_ranges_in.reserve(n));
    if (h->d_scan_keys.cap < n) {
        RES(h->d_scan_keys.reserve(n));
        CU(cudaMemsetAsync(h->d_scan_keys.p, 0, sizeof(unsigned long long) * h->d_scan_keys.cap, h->stream));   // k_scan_cells keeps them 0 from here on
    }
    CloudScan c;
    c.width = L->width; c.n_points = (uint32_t)n_points; c.row_step = L->row_step; c.point_step = L->point_step;
    for (int k = 0; k < 3; k++) c.off[k] = off[k];
    c.f64 = L->datatype == 8 ? 1u : 0u;
    c.T = tf_from_pod(*T);
    c.phi_min = m.phi_min; c.phi_inc = m.phi_inc; c.theta_min = m.theta_min; c.theta_inc = m.theta_inc; c.phi_n = m.phi_size; c.theta_n = m.theta_size;
    c.range_min = m.range_min; c.range_max = m.range_max;
    c.fill = (float)((double)m.range_max + 1.0);                                  // scan.info.range_max + 1.0 stored as float
    if (n_points) {
        const uint8_t* src = static_cast<const uint8_t*>(data);
        if (!src_is_device) {
            RES(h->d_cloud.reserve(need));
            CU(cudaMemcpyAsync(h->d_cloud.p, data, need, cudaMemcpyHostToDevice, h->stream));
            src = h->d_cloud.p;
        }
        k_scan_bin_cloud<<<(uint32_t)((n_points + 255) / 256), 256, 0, h->stream>>>(src, c, h->d_scan_keys.p);
        LAUNCHED();
    }
    k_scan_cells<<<(n + 255) / 256, 256, 0, h->stream>>>(c, h->d_scan_keys.p, h->d_dirs.p, h->d_origs.p, h->d_ranges_in.p, h->d_dpts.p, h->d_dmask.p);
    LAUNCHED();
    h->b_dpts = nullptr; h->b_dmask = nullptr;
    h->n_dataset = n; h->n_ranges_in = n;
    if (!src_is_device) CU(cudaStreamSynchronize(h->stream));
    return B2_OK;
}

static int reserve_model(b2_rcc* h, size_t n)
{
    // buffers only ever grow (RCCEmbree.cpp:28-33)
    if (h->b_mpts && n > h->b_mcap) return fail(B2_ERR_INVALID, "bound model buffers hold %u entries, find needs %zu (resize them and bind again, RCCOptix.cpp:36-40)", h->b_mcap, n);
    RES(h->d_mpts.reserve(h->b_mpts ? 1 : 3 * n)); RES(h->d_mnrm.reserve(h->b_mpts ? 1 : 3 * n)); RES(h->d_mranges.reserve(n)); RES(h->d_mhits.reserve(h->b_mpts ? 1 : n)); RES(h->d_mfaces.reserve(n));
    return B2_OK;
}

static RayModel ray_model(const b2_rcc* h)
{
    RayModel m; m.dirs = h->d_dirs.p; m.origs = h->d_origs.p; m.n_origs = h->n_origs; m.n = h->n; m.range_min = h->range_min; m.range_max = h->range_max;
    m.width = h->width; m.height = h->height; m.sim_opts = h->sim_opts; return m;
}
static ModelBuffers model_buffers(const b2_rcc* h)
{
    ModelBuffers b; b.pts = h->mpts(); b.nrm = h->mnrm(); b.hits = h->mhits(); b.faces = h->d_mfaces.p; b.ranges = h->d_mranges.p; return b;
}

// k_rcc_find as one resident wave (kernels.cuh): the blocks that fit on the device at once, computed once per device
static int find_slots(int device, uint32_t* slots)
{
    static std::atomic<uint32_t> per_device[64];
    uint32_t v = per_device[device & 63].load(std::memory_order_relaxed);
    if (v == 0) {
        int per_sm = 0, n_sm = 0;
        CU(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_rcc_find, B2_FIND_BLOCK, 0));
        CU(cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, device));
        if (per_sm < 1 || n_sm < 1) return fail(B2_ERR_CUDA, "k_rcc_find cannot be resident on device %d", device);
        v = (uint32_t)per_sm * (uint32_t)n_sm;
        per_device[device & 63].store(v, std::memory_order_relaxed);
    }
    *slots = v;
    return B2_OK;
}

// k_rcc_find over `total` rays (all poses) on h's stream: the grid is one resident wave, at most one warp per tile, and the tickets
// of the launch are taken from h's queue counter.  The launch consumes exactly n_tiles tickets (kernels.cuh); h->find_ticket follows
// the device counter modulo 2^32.
static int launch_rcc_find(b2_rcc* h, uint64_t total, int prefetch_mode, const b2_transform* Tbm_dev, const IcpState* icp_dev, const b2_transform& Tbm_val,
                           uint32_t n_poses, const ModelBuffers& out, int early, const uint16_t* perm, uint32_t* cost)
{
    const uint64_t n_tiles = (total + 31u) / 32u;
    if (n_tiles > 0x7fffffffull) return fail(B2_ERR_INVALID, "too many rays for one find (%llu)", (unsigned long long)total);
    uint32_t slots = 0;
    RES(find_slots(h->map->device, &slots));
    const uint32_t warps_per_block = B2_FIND_BLOCK / 32u, grid = (uint32_t)std::min<uint64_t>(slots, (n_tiles + warps_per_block - 1u) / warps_per_block);
    const unsigned int base = h->find_ticket;
    k_rcc_find<<<grid, B2_FIND_BLOCK, 0, h->stream>>>(h->map->view(), h->map->n_nodes, h->map->n_tris, prefetch_mode, Tbm_dev, icp_dev, Tbm_val, h->Tsb, ray_model(h), n_poses, out, early,
                                                      perm, cost, h->d_find_tickets.p, base, (uint32_t)n_tiles);
    h->find_ticket = base + (unsigned int)n_tiles;                              // unsigned: wraps like the device counter
    h->find_grid = grid;
    return B2_OK;
}

static int launch_find(b2_rcc* h, const b2_transform* Tbm_host, const IcpState* icp_dev)
{
    static const int prefetch_mode_cp = [] { const char* e = getenv("B2_FIND_PREFETCH"); return e ? atoi(e) : 0; }();
    if (h->corr_type == B2_CORR_CPC) {
        // CPCEmbree::find (CPCEmbree.cpp:17-43): one closest-point query per dataset point
        const uint32_t n = h->n_dataset;
        if (n == 0) { h->n_model = 0; h->found = true; return B2_OK; }
        RES(reserve_model(h, n));
        k_cpc_find<<<(n + B2_FIND_BLOCK - 1) / B2_FIND_BLOCK, B2_FIND_BLOCK, 0, h->stream>>>(h->map->view(), h->map->n_nodes, h->map->n_tris, prefetch_mode_cp, icp_dev,
                                                                                             Tbm_host ? *Tbm_host : tf_identity_pod(), h->Tsb, h->dpts(), n, h->max_dist, model_buffers(h), h->cpc_skip_masked ? h->dmask() : nullptr);
        LAUNCHED();
        h->n_model = n; h->found = true;
        return B2_OK;
    }
    if (!h->has_model) return fail(B2_ERR_INVALID, "find before setModel");
    if (h->n == 0) return B2_OK;
    RES(reserve_model(h, h->n));
    // no L2 prefetch by default: on an H100 (50 MB L2) prefetching the 37 MB node array of a 1M-triangle map slowed the C2 step from
    // 80 to 86 us (nodes + triangles, mode 2: 91 us)
    static const int prefetch_mode = [] { const char* e = getenv("B2_FIND_PREFETCH"); return e ? atoi(e) : 0; }();
    // early_dependents: the grid is one resident wave, so an early-resident dependent block never takes a slot a find block waits for
    const int early = h->pdl_next ? 1 : 0;
    h->pdl_armed = early != 0;
    // tile schedule (kernels.cuh): whole tiles only, as many as the ICP loop's idle warps sort in the time they have (icp_loop.cuh)
    static const int use_sched = [] { const char* e = getenv("B2_FIND_SCHED"); return e ? atoi(e) : 1; }();
    const uint32_t n_tiles = h->n / 32u;
    const bool sched = use_sched && (h->n % 32u) == 0u && n_tiles >= 2u && n_tiles <= (uint32_t)B2_PERM_MAX_TILES;
    uint32_t* cost = nullptr; const uint16_t* perm = nullptr;
    if (sched) {
        if (h->perm_tiles != n_tiles) {      // first launch with this model: identity order; from then on d_tile_perm always holds a permutation of the tiles
            RES(h->d_tile_cost.reserve(n_tiles)); RES(h->d_tile_perm.reserve(n_tiles));
            k_perm_identity<<<(n_tiles + 255u) / 256u, 256, 0, h->stream>>>(h->d_tile_perm.p, n_tiles);
            LAUNCHED();
            h->perm_tiles = n_tiles;
        }
        cost = h->d_tile_cost.p; perm = h->d_tile_perm.p; h->cost_tiles = n_tiles;
    } else h->cost_tiles = 0;
    RES(launch_rcc_find(h, h->n, prefetch_mode, nullptr, icp_dev, Tbm_host ? *Tbm_host : tf_identity_pod(), 1u, model_buffers(h), early, perm, cost));
    LAUNCHED();
    h->n_model = h->n; h->found = true;
    return B2_OK;
}

extern "C" int b2_rcc_set_cpc_options(b2_rcc* h, int skip_masked)
{
    NOTNULL(h);
    h->cpc_skip_masked = skip_masked != 0; h->found = false;
    return B2_OK;
}
extern "C" int b2_rcc_bind_dataset(b2_rcc* h, const float* points_dev, const uint8_t* mask_dev, uint32_t n)
{
    NOTNULL(h);
    if (n) { NOTNULL(points_dev); NOTNULL(mask_dev); }
    if (!h->pending.empty()) return fail(B2_ERR_INVALID, "bind_dataset while correctOnce calls are in flight");
    h->b_dpts = n ? points_dev : nullptr; h->b_dmask = n ? mask_dev : nullptr; h->n_dataset = n;
    return B2_OK;
}
extern "C" int b2_rcc_bind_model_buffers(b2_rcc* h, float* points_dev, float* normals_dev, uint8_t* hits_dev, uint32_t capacity)
{
    NOTNULL(h);
    if (!h->pending.empty()) return fail(B2_ERR_INVALID, "bind_model_buffers while correctOnce calls are in flight");
    if (capacity == 0 || !points_dev) { h->b_mpts = nullptr; h->b_mnrm = nullptr; h->b_mhits = nullptr; h->b_mcap = 0; h->found = false; return B2_OK; }
    NOTNULL(normals_dev); NOTNULL(hits_dev);
    if (h->b_mpts == points_dev && h->b_mnrm == normals_dev && h->b_mhits == hits_dev && h->b_mcap == capacity) return B2_OK;      // bound already: the last find stays valid
    h->b_mpts = points_dev; h->b_mnrm = normals_dev; h->b_mhits = hits_dev; h->b_mcap = capacity; h->found = false;
    return B2_OK;
}

extern "C" int b2_rcc_set_sim_options(b2_rcc* h, int tfar_mode, int min_mode, int miss_fill)
{
    NOTNULL(h);
    if ((tfar_mode | min_mode | miss_fill) & ~1) return fail(B2_ERR_INVALID, "sim options are 0 or 1");
    h->sim_opts = (uint32_t)(tfar_mode | (min_mode << 1) | (miss_fill << 2)); h->found = false;
    return B2_OK;
}

extern "C" int b2_rcc_set_correspondence_type(b2_rcc* h, int type)
{
    NOTNULL(h);
    if (type != B2_CORR_RCC && type != B2_CORR_CPC) return fail(B2_ERR_INVALID, "unknown correspondence type %d", type);
    h->corr_type = type; h->found = false;
    return B2_OK;
}

extern "C" int b2_rcc_find(b2_rcc* h, const b2_transform* Tbm)
{
    NOTNULL(h); NOTNULL(Tbm);
    CU(cudaSetDevice(h->map->device));
    return launch_find(h, Tbm, nullptr);
}

static int launch_reduce(b2_rcc* h, const b2_transform* Tpre_host, float max_dist, IcpState* icp_dev, b2_cross_stats* out_dev)
{
    const uint32_t n = std::min(h->n_dataset, h->n_model);
    int grid = (int)std::min<uint32_t>((uint32_t)h->red_grid, (n + B2_RED_BLOCK - 1) / B2_RED_BLOCK);
    if (grid < 1) grid = 1;
    k_p2l_reduce<<<grid, B2_RED_BLOCK, 0, h->stream>>>(h->dpts(), h->dmask(), h->mpts(), h->mnrm(), h->mhits(), n,
                                                       Tpre_host ? *Tpre_host : tf_identity_pod(), max_dist, icp_dev, h->d_partials.p, h->d_ticket.p, out_dev);
    LAUNCHED();
    return B2_OK;
}

static float adaptive_max_dist(const b2_rcc* h, double cp)
{
    // CorrespondencesCPU.cpp:21-23
    return (float)(h->max_dist * (1.0 - cp) + h->adaptive_max_dist_min * cp);
}

extern "C" int b2_rcc_cross_statistics(b2_rcc* h, const b2_transform* T, double cp, b2_cross_stats* out)
{
    NOTNULL(h); NOTNULL(T); NOTNULL(out);
    CU(cudaSetDevice(h->map->device));
    if (!h->found) return fail(B2_ERR_INVALID, "computeCrossStatistics before find");
    RES(launch_reduce(h, T, adaptive_max_dist(h, cp), nullptr, h->d_stats.p));
    CU(cudaMemcpyAsync(&h->pin->S[0], h->d_stats.p, sizeof(b2_cross_stats), cudaMemcpyDeviceToHost, h->stream));
    CU(cudaStreamSynchronize(h->stream));
    *out = h->pin->S[0];
    return B2_OK;
}

extern "C" int b2_rcc_segment(b2_rcc* h, float min_dist_outlier_scan, float min_dist_outlier_map, float* outlier_scan, uint32_t cap_scan, uint32_t* n_scan,
                              float* outlier_map, uint32_t cap_map, uint32_t* n_map, uint8_t* labels)
{
    NOTNULL(h); NOTNULL(n_scan); NOTNULL(n_map);
    *n_scan = 0; *n_map = 0;
    CU(cudaSetDevice(h->map->device));
    if (h->corr_type != B2_CORR_RCC || !h->has_model) return fail(B2_ERR_INVALID, "segmentation needs a ray-casting handle with a sensor model");
    if (!h->found || h->n_model != h->n) return fail(B2_ERR_INVALID, "segmentation before find");
    if (h->n_ranges_in != h->n) return fail(B2_ERR_INVALID, "segmentation needs the real ranges (set_ranges), have %u of %u", h->n_ranges_in, h->n);
    const uint32_t n = h->n;
    if (n == 0) return B2_OK;
    const uint32_t blocks = (n + B2_SEG_BLOCK - 1) / B2_SEG_BLOCK;
    RES(h->d_seg_counts.reserve(2 * (size_t)blocks)); RES(h->d_seg_offsets.reserve(2 * (size_t)blocks)); RES(h->d_seg_totals.reserve(2));
    RES(h->d_seg_scan.reserve(3 * (size_t)n)); RES(h->d_seg_map.reserve(3 * (size_t)n)); RES(h->d_seg_labels.reserve(n));
    const RayModel m = ray_model(h);
    k_segment<<<blocks, B2_SEG_BLOCK, 0, h->stream>>>(m, h->d_ranges_in.p, h->d_mranges.p, h->mnrm(), min_dist_outlier_scan, min_dist_outlier_map, h->d_seg_counts.p, nullptr, nullptr, nullptr, nullptr);
    LAUNCHED();
    k_segment_scan<<<1, 1024, 0, h->stream>>>(h->d_seg_counts.p, blocks, h->d_seg_offsets.p, h->d_seg_totals.p);
    LAUNCHED();
    k_segment<<<blocks, B2_SEG_BLOCK, 0, h->stream>>>(m, h->d_ranges_in.p, h->d_mranges.p, h->mnrm(), min_dist_outlier_scan, min_dist_outlier_map, h->d_seg_counts.p, h->d_seg_offsets.p,
                                                      h->d_seg_scan.p, h->d_seg_map.p, h->d_seg_labels.p);
    LAUNCHED();
    uint32_t tot[2] = {0, 0};
    CU(cudaMemcpyAsync(tot, h->d_seg_totals.p, sizeof(tot), cudaMemcpyDeviceToHost, h->stream));
    CU(cudaStreamSynchronize(h->stream));
    *n_scan = tot[0]; *n_map = tot[1];
    if (outlier_scan && std::min(tot[0], cap_scan)) CU(cudaMemcpyAsync(outlier_scan, h->d_seg_scan.p, sizeof(float) * 3 * (size_t)std::min(tot[0], cap_scan), cudaMemcpyDeviceToHost, h->stream));
    if (outlier_map && std::min(tot[1], cap_map)) CU(cudaMemcpyAsync(outlier_map, h->d_seg_map.p, sizeof(float) * 3 * (size_t)std::min(tot[1], cap_map), cudaMemcpyDeviceToHost, h->stream));
    if (labels) CU(cudaMemcpyAsync(labels, h->d_seg_labels.p, n, cudaMemcpyDeviceToHost, h->stream));
    CU(cudaStreamSynchronize(h->stream));
    return B2_OK;
}

extern "C" int b2_rcc_model_view(b2_rcc* h, float** p, float** nr, uint8_t** hi, uint32_t** f, float** r, uint32_t* n)
{
    NOTNULL(h);
    if (p) *p = h->mpts(); if (nr) *nr = h->mnrm(); if (hi) *hi = h->mhits(); if (f) *f = h->d_mfaces.p; if (r) *r = h->d_mranges.p; if (n) *n = h->n_model;
    return B2_OK;
}
extern "C" int b2_rcc_dataset_view(b2_rcc* h, float** p, uint8_t** m, uint32_t* n)
{
    NOTNULL(h);
    if (p) *p = const_cast<float*>(h->dpts()); if (m) *m = const_cast<uint8_t*>(h->dmask()); if (n) *n = h->n_dataset;
    return B2_OK;
}
extern "C" int b2_rcc_download_model(b2_rcc* h, float* p, float* nr, uint8_t* hi, uint32_t* f, float* r)
{
    NOTNULL(h);
    CU(cudaSetDevice(h->map->device));
    const size_t n = h->n_model;
    CU(cudaStreamSynchronize(h->stream));
    if (n == 0) return B2_OK;
    if (p) CU(cudaMemcpy(p, h->mpts(), sizeof(float) * 3 * n, cudaMemcpyDeviceToHost));
    if (nr) CU(cudaMemcpy(nr, h->mnrm(), sizeof(float) * 3 * n, cudaMemcpyDeviceToHost));
    if (hi) CU(cudaMemcpy(hi, h->mhits(), n, cudaMemcpyDeviceToHost));
    if (f) CU(cudaMemcpy(f, h->d_mfaces.p, sizeof(uint32_t) * n, cudaMemcpyDeviceToHost));
    if (r) CU(cudaMemcpy(r, h->d_mranges.p, sizeof(float) * n, cudaMemcpyDeviceToHost));
    return B2_OK;
}
extern "C" int b2_rcc_download_dataset(b2_rcc* h, float* p, uint8_t* m)
{
    NOTNULL(h);
    CU(cudaSetDevice(h->map->device));
    const size_t n = h->n_dataset;
    CU(cudaStreamSynchronize(h->stream));
    if (n == 0) return B2_OK;
    if (p) CU(cudaMemcpy(p, h->dpts(), sizeof(float) * 3 * n, cudaMemcpyDeviceToHost));
    if (m) CU(cudaMemcpy(m, h->dmask(), n, cudaMemcpyDeviceToHost));
    return B2_OK;
}

// ---------------------------------------------------------------------------------------------------------------------
// correctOnce (micp_localization.cpp:899-984) for 1..B2_MAX_SENSORS sensors.  sc[0].h is the LEAD handle: its stream carries the launches,
// its buffers hold the partial sums / the barrier / the result.
// ---------------------------------------------------------------------------------------------------------------------
struct SensorCall { b2_rcc* h; b2_transform Tbo; double weight; const float* ranges_host; uint32_t n_ranges; };

// Tbm = Tom * Tbo (MICPSensor.hpp:148), same inline ops as the kernels
static b2_transform body_in_map(const b2_transform& Tom, const b2_transform& Tbo)
{
    b2_transform Tbm; memset(&Tbm, 0, sizeof(Tbm)); tf_store(&Tbm, tf_mul(tf_from_pod(Tom), tf_from_pod(Tbo))); return Tbm;
}

// Sensor list of b2_micp_correct_once / b2_micp_correct (`fn`, messages prefixed `what`): 1..B2_MAX_SENSORS distinct handles, nothing in flight
// on the lead.  ranges_host NULL: every sensor keeps its dataset.
static int sensor_list(const char* fn, const char* what, b2_rcc* const* sensors, const b2_transform* Tbo, const double* merge_weights,
                       const float* const* ranges_host, uint32_t n_sensors, SensorCall* sc)
{
    if (n_sensors == 0 || n_sensors > B2_MAX_SENSORS) return fail(B2_ERR_INVALID, "%s: %u sensors (1..%d supported per call)", what, n_sensors, B2_MAX_SENSORS);
    for (uint32_t k = 0; k < n_sensors; k++) {
        if (!sensors[k]) return fail(B2_ERR_INVALID, "%s: null argument '%s'", fn, "sensors[k]");
        for (uint32_t j = 0; j < k; j++) if (sensors[j] == sensors[k]) return fail(B2_ERR_INVALID, "%s: sensor %u given twice", what, k);
        sc[k].h = sensors[k]; sc[k].Tbo = Tbo[k]; sc[k].weight = merge_weights ? merge_weights[k] : 1.0;
        sc[k].ranges_host = ranges_host ? ranges_host[k] : nullptr; sc[k].n_ranges = sc[k].ranges_host ? sensors[k]->n : 0;
    }
    const b2_rcc* H = sc[0].h;
    CU(cudaSetDevice(H->map->device));
    if (!H->pending.empty()) return fail(B2_ERR_INVALID, "%s: asynchronous calls are still in flight on the lead handle, collect them first", what);
    return B2_OK;
}

// Checks every sensor of a call and changes none, so that a refused call leaves all handles as they were.  *pairs = correspondences of all.
static int check_sensors(const SensorCall* sc, uint32_t ns, const char* what, uint64_t* pairs)
{
    *pairs = 0;
    for (uint32_t k = 0; k < ns; k++) {
        const b2_rcc* h = sc[k].h;
        if (h->map->device != sc[0].h->map->device) return fail(B2_ERR_INVALID, "%s: all sensors must live on the same device", what);
        const bool cpc = h->corr_type == B2_CORR_CPC;
        if (sc[k].ranges_host && cpc) return fail(B2_ERR_INVALID, "correctOnce(ranges) needs ray-casting correspondences (the handle is in closest-point mode)");
        if (!cpc && !h->has_model) return fail(B2_ERR_INVALID, "%s before setModel", what);
        if (sc[k].ranges_host && sc[k].n_ranges != h->n) return fail(B2_ERR_INVALID, "ranges size %u != model size %u", sc[k].n_ranges, h->n);
        if (!sc[k].ranges_host && h->n_dataset != h->work_n()) return fail(B2_ERR_INVALID, "dataset size %u != model size %u", h->n_dataset, h->n);
        *pairs += h->work_n();
    }
    return B2_OK;
}

// into_lead: the lead stream waits for the other sensors' streams (pending set_ranges / set_dataset copies); otherwise they wait for the lead
// stream, so that later work on them sees the model buffers the call wrote
static int join_streams(const SensorCall* sc, uint32_t ns, bool into_lead)
{
    for (uint32_t k = 1; k < ns; k++) {
        b2_rcc* h = sc[k].h;
        CU(cudaEventRecord(h->ev_join, into_lead ? h->stream : sc[0].h->stream));
        CU(cudaStreamWaitEvent(into_lead ? sc[0].h->stream : h->stream, h->ev_join, 0));
    }
    return B2_OK;
}

// h's find on the lead H's stream, which carries all launches of a call.  arm_pdl: the loop follows this find and may start early behind it,
// programmatically (B2_PDL, default 1; behind the last find only: event records / other kernels in between would serialise them anyway)
static int find_on_lead(b2_rcc* H, b2_rcc* h, const b2_transform* Tbm_host, const IcpState* icp_dev, bool arm_pdl)
{
    static const int use_pdl = [] { const char* e = getenv("B2_PDL"); return e ? atoi(e) : 1; }();
    const cudaStream_t own = h->stream;
    h->stream = H->stream; h->pdl_next = arm_pdl && use_pdl && h->corr_type == B2_CORR_RCC;
    const int rc = launch_find(h, Tbm_host, icp_dev);
    h->pdl_next = false; h->stream = own;
    return rc;
}

// sequence number of the next k_icp_loop launch; never 0, which the result chunks hold before the first launch
static unsigned int next_seq(b2_rcc* H) { unsigned int seq = ++H->seq; if (seq == 0) seq = ++H->seq; return seq; }

// slot < 0: no result chunks in mapped host memory (chain steps: their results stay on the device)
static int launch_icp_loop(b2_rcc* H, const IcpLaunch& L, int grid, size_t smem, int mode, bool pdl, int slot)
{
    unsigned long long* parts = H->d_slots.p; IcpResult* res_dev = H->d_res.p; uint4* host_out = slot >= 0 ? H->pin_chunks_dev + (size_t)slot * (B2_ICP_RESULT_CHUNKS + 1) : nullptr;
    unsigned int tag_base = H->tag_base; unsigned int* bar_abort = H->d_bar.p + 1; unsigned long long* dbg = H->d_dbg.p;
    H->tag_base += L.iterations;                                  // tags tag_base + 1 .. tag_base + iterations belong to this launch
    if (H->tag_base > 0xfffffff0u - 64u) H->tag_base = 0;          // wrap far away from anything a live slot can still hold
    if (mode == 1) {
        IcpLaunch Lc = L;
        void* args[] = {&Lc, &parts, &res_dev, &host_out, &tag_base, &bar_abort, &dbg};
        CU(cudaLaunchCooperativeKernel((const void*)k_icp_loop<true>, dim3((unsigned)grid), dim3(B2_ICP_BLOCK), args, smem, H->stream));
    } else {
        // One software-barrier loop at a time per device: launches of different handles / streams are chained through the device's event
        DeviceCtx& dc = g_dev[H->map->device & 63];
        std::lock_guard<std::mutex> lk(dc.m);
        if (!dc.loop_done) CU(cudaEventCreateWithFlags(&dc.loop_done, cudaEventDisableTiming));
        const bool foreign = dc.last && (dc.last != H || dc.last_stream != H->stream);
        if (foreign) {
            dc.multi = true;
            if (dc.recorded) CU(cudaStreamWaitEvent(H->stream, dc.loop_done, 0));
            else CU(cudaDeviceSynchronize());            // the previous launch left no marker (first change of handle / stream): drain once
            pdl = false;
        }
        cudaLaunchConfig_t cfg{};
        cfg.gridDim = dim3((unsigned)grid); cfg.blockDim = dim3(B2_ICP_BLOCK); cfg.dynamicSmemBytes = smem; cfg.stream = H->stream;
        cudaLaunchAttribute attr[1];
        attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
        attr[0].val.programmaticStreamSerializationAllowed = pdl ? 1 : 0;
        cfg.attrs = attr; cfg.numAttrs = 1;
        CU(cudaLaunchKernelEx(&cfg, k_icp_loop<false>, L, parts, res_dev, host_out, tag_base, bar_abort, dbg));
        dc.recorded = false;
        if (dc.multi) { CU(cudaEventRecord(dc.loop_done, H->stream)); dc.recorded = true; }     // the marker the next foreign launch waits on
        dc.last = H; dc.last_stream = H->stream;
    }
    LAUNCHED();
    return B2_OK;
}

// k_icp_loop's launch L for `total` pairs and its grid (returned).  Blocks per sensor: in proportion to the pairs, at least one for each sensor
// with pairs.  A sensor without pairs gets none, so the other sensors' pairs are summed by exactly the blocks a call without it would use: its
// presence cannot change a bit of the result.  Then per sensor the pairs per thread in shared memory, merge weight, range limits, frames and
// dataset; the gate (max_dist) is the caller's.
// The blocks of a grid of at most grid_cap blocks of `block` threads, split among ns sensors with n[k] pairs (total in all) as described above.
// Returns the grid; nblk[k] receives sensor k's blocks.
static int split_blocks(const uint32_t* n, uint32_t ns, uint64_t total, int grid_cap, int block, uint32_t* nblk)
{
    uint32_t ns_busy = 0;
    for (uint32_t k = 0; k < ns; k++) if (n[k] > 0) ns_busy++;
    const int grid = std::min<int>(grid_cap, (int)std::max<uint64_t>((total + block - 1) / block, ns_busy));
    int assigned = 0;
    for (uint32_t k = 0; k < ns; k++) {
        const uint32_t nw = n[k];
        nblk[k] = nw ? std::max<uint32_t>(1u, (uint32_t)((uint64_t)grid * nw / total)) : 0u; assigned += (int)nblk[k];
    }
    while (assigned > grid) { uint32_t big = 0; for (uint32_t k = 1; k < ns; k++) if (nblk[k] > nblk[big]) big = k; nblk[big]--; assigned--; }
    while (assigned < grid) {
        uint32_t best = 0; double load = -1.0;
        for (uint32_t k = 0; k < ns; k++) { if (!nblk[k]) continue; const double l = (double)n[k] / nblk[k]; if (l > load) { load = l; best = k; } }
        nblk[best]++; assigned++;
    }
    return grid;
}

static int loop_layout(const b2_rcc* H, const SensorCall* sc, uint32_t ns, uint64_t total, const b2_transform& Tom, uint32_t iterations, IcpLaunch& L)
{
    memset(&L, 0, sizeof(L));
    L.Tom = Tom; L.n_sensors = ns; L.iterations = iterations;
    uint32_t nw[B2_MAX_SENSORS], nblk[B2_MAX_SENSORS];
    for (uint32_t k = 0; k < ns; k++) nw[k] = sc[k].h->work_n();
    const int grid = split_blocks(nw, ns, total, H->fused_grid, B2_ICP_BLOCK, nblk);
    uint32_t blk0 = 0;
    for (uint32_t k = 0; k < ns; k++) {
        const b2_rcc* h = sc[k].h;
        IcpSensor& S = L.s[k];
        S.n = h->work_n(); S.blk0 = blk0; S.nblk = nblk[k]; blk0 += nblk[k];
        const uint32_t stride = S.nblk * B2_ICP_BLOCK, per_thread = stride ? (S.n + stride - 1) / stride : 0u;
        S.smem_u = per_thread > B2_ICP_REG_PAIRS ? std::min<uint32_t>(per_thread - B2_ICP_REG_PAIRS, (uint32_t)H->smem_u_cap) : 0u;
        L.smem_u_max = std::max(L.smem_u_max, S.smem_u);
        S.merge_weight = sc[k].weight; S.range_min = h->range_min; S.range_max = h->range_max;
        const Tf Tos = tf_mul(tf_from_pod(sc[k].Tbo), tf_from_pod(h->Tsb));
        memset(&S.Tos, 0, sizeof(S.Tos)); memset(&S.Tso, 0, sizeof(S.Tso));
        tf_store(&S.Tos, Tos); tf_store(&S.Tso, tf_inv(Tos)); quat_to_mat(Tos.R, S.Ros);
        S.dpts = h->dpts(); S.dmask = h->dmask();
    }
    return grid;
}

// k_icp_loop behind the finds of a call: their model buffers (a find may have grown them), tile-sort fields, dynamic shared memory (*smem_out),
// sequence number; a programmatic launch if the last find armed it and pdl_ok.  Records the geometry for b2_rcc_debug_loop_geometry.
static int launch_loop_after_finds(b2_rcc* H, const SensorCall* sc, uint32_t ns, IcpLaunch& L, int grid, int mode, bool pdl_ok, int slot, size_t* smem_out)
{
    uint32_t sort_tiles_max = 0;
    for (uint32_t k = 0; k < ns; k++) {
        const b2_rcc* h = sc[k].h;
        IcpSensor& S = L.s[k];
        S.mpts = h->mpts(); S.mnrm = h->mnrm(); S.mmask = h->mhits();
        S.tile_cost = nullptr; S.tile_perm = nullptr; S.n_tiles = 0;
        if (h->corr_type == B2_CORR_RCC && h->cost_tiles && L.iterations >= 3u) {
            S.tile_cost = h->d_tile_cost.p; S.tile_perm = h->d_tile_perm.p; S.n_tiles = h->cost_tiles;
            sort_tiles_max = std::max(sort_tiles_max, h->cost_tiles);
        }
    }
    size_t smem = (size_t)L.smem_u_max * 9 * B2_ICP_BLOCK * sizeof(float);
    if (sort_tiles_max) {
        // the tile sort stages the durations behind the pair cache (2 bytes per tile); no room (very large scans): no sort, the order stays as it is
        const size_t want = smem + 2 * (size_t)sort_tiles_max;
        if (want <= (size_t)H->smem_u_cap * 9 * B2_ICP_BLOCK * sizeof(float)) smem = want;
        else for (uint32_t k = 0; k < ns; k++) { L.s[k].tile_cost = nullptr; L.s[k].tile_perm = nullptr; L.s[k].n_tiles = 0; }
    }
    if (smem_out) *smem_out = smem;
    L.seq = next_seq(H);
    const bool pdl = mode == 2 && sc[ns - 1].h->pdl_armed && pdl_ok;
    sc[ns - 1].h->pdl_armed = false;
    RES(launch_icp_loop(H, L, grid, smem, mode, pdl, slot));
    memset(H->loop_geom, 0, sizeof(H->loop_geom));
    H->loop_geom[0] = ns; H->loop_geom[1] = (uint32_t)grid;
    for (uint32_t k = 0; k < ns; k++) { uint32_t* g = H->loop_geom + 2 + 4 * k; g[0] = L.s[k].n; g[1] = L.s[k].blk0; g[2] = L.s[k].nblk; g[3] = L.s[k].smem_u; }
    return B2_OK;
}

// Did the grid-wide exchange of a mode-2 loop give up (its blocks were not co-resident: SMs held by something that itself waits; or code 2: a
// block's partial sum left the fixed-point range of the atomic exchange)?  That is a scheduling condition, not an error: the abort word and the
// accumulator words the aborted rounds left inconsistent are reset, and the caller runs the work again through the cooperative launch, whose
// co-residency the driver guarantees and which exchanges FP64.
static int exchange_aborted(b2_rcc* H, bool* aborted)
{
    unsigned int bar_state[2] = {0u, 0u};
    CU(cudaMemcpy(bar_state, H->d_bar.p, sizeof(bar_state), cudaMemcpyDeviceToHost));
    *aborted = bar_state[1] != 0u;
    if (*aborted) {
        CU(cudaMemset(H->d_bar.p + 1, 0, sizeof(unsigned int)));
        CU(cudaMemset(H->d_slots.p, 0, ((size_t)B2_ICP_ACC_WORDS + B2_ICP_BASE_WORDS) * sizeof(unsigned long long)));
    }
    return B2_OK;
}

static int micp_enqueue(SensorCall* sc, uint32_t ns, const b2_transform* Tom, uint32_t iterations, double cp)
{
    b2_rcc* H = sc[0].h;
    if (H->pending.size() >= B2_RING) return fail(B2_ERR_INVALID, "correctOnce: %d asynchronous calls are in flight already, collect one first (b2_rcc_correct_once_wait)", B2_RING);
    static const int use_zc = [] { const char* e = getenv("B2_ZEROCOPY"); return e ? atoi(e) : 1; }();
    static const int use_spin = [] { const char* e = getenv("B2_SPIN"); return e ? atoi(e) : 1; }();
    int mode = H->exec_mode;
    if (H->fused_grid <= 0) mode = 0;
    if (ns > 1 && mode == 0) mode = H->fused_grid > 0 ? 1 : 0;
    if (ns > 1 && mode == 0) return fail(B2_ERR_UNSUPPORTED, "multi-sensor correctOnce needs a device with cooperative launch");
    uint64_t total = 0;
    RES(check_sensors(sc, ns, "correctOnce", &total));
    if (mode == 0 && !H->pending.empty()) return fail(B2_ERR_INVALID, "correctOnce: exec mode 0 keeps its state in one staging block: collect the pending call first");
    for (const PendingCall& q : H->pending) if (q.kind == 3) return fail(B2_ERR_INVALID, "correctOnce: an exec-mode-0 call is pending: collect it first");
    for (uint32_t k = 0; k < ns; k++) if (sc[k].ranges_host) {          // accepted: the scans replace the datasets (uploaded below)
        b2_rcc* h = sc[k].h;
        h->n_dataset = h->n; h->n_ranges_in = h->n; h->b_dpts = nullptr; h->b_dmask = nullptr;
        if (h->n > 0) { RES(h->d_dpts.reserve(3 * (size_t)h->n)); RES(h->d_dmask.reserve(h->n)); RES(h->d_ranges_in.reserve(h->n)); }
    }
    H->pending.emplace_back();
    PendingCall& pc = H->pending.back();
    struct Guard { b2_rcc* H; bool ok = false; ~Guard() { if (!ok) H->pending.pop_back(); } } guard{H};
    // ---- nothing to do on the device: identity update (micp_localization.cpp:974: Tom stays when n_meas == 0) ----
    if (total == 0 || iterations == 0) {
        memset(&pc.res, 0, sizeof(pc.res));
        pc.res.Tom_new = *Tom; pc.res.T_onew_oold = tf_identity_pod();
        if (total > 0) for (uint32_t k = 0; k < ns; k++) {          // iterations == 0: the reference still runs findCorrespondences (:900-908)
            const b2_transform Tbm = body_in_map(*Tom, sc[k].Tbo);
            if (sc[k].ranges_host && sc[k].h->n) { RES(ranges_to_dataset(sc[k].h, sc[k].ranges_host, sc[k].n_ranges, 0)); CU(cudaStreamSynchronize(sc[k].h->stream)); }
            RES(launch_find(sc[k].h, &Tbm, nullptr));
        }
        pc.kind = 0; guard.ok = true;
        return B2_OK;
    }
    // ---- the multi-launch chain (exec mode 0): find + one k_p2l_reduce per inner iteration, state in device memory ----
    if (mode == 0) {
        b2_rcc* h = H;
        if (sc[0].ranges_host && h->n) RES(ranges_to_dataset(h, sc[0].ranges_host, sc[0].n_ranges, 0));
        IcpState& st = h->pin->icp;
        memset(&st, 0, sizeof(st));
        st.Tom = *Tom; st.Tbo = sc[0].Tbo; st.Tsb = h->Tsb; st.max_dist = adaptive_max_dist(h, cp);
        st.T_onew_oold = tf_identity_pod(); st.Tom_new = *Tom;
        tf_store(&st.T_snew_sold, icp_pretransform(tf_from_pod(sc[0].Tbo), tf_from_pod(h->Tsb), tf_identity()));
        CU(cudaMemcpyAsync(h->d_icp.p, &st, sizeof(IcpState), cudaMemcpyHostToDevice, h->stream));
        if (h->timing) CU(cudaEventRecord(h->ev[0], h->stream));
        RES(launch_find(h, nullptr, h->d_icp.p));
        if (h->timing) CU(cudaEventRecord(h->ev[1], h->stream));
        for (uint32_t it = 0; it < iterations; it++) RES(launch_reduce(h, nullptr, 0.f, h->d_icp.p, nullptr));
        if (h->timing) { CU(cudaEventRecord(h->ev[2], h->stream)); h->timing_valid = true; }
        CU(cudaMemcpyAsync(&st, h->d_icp.p, sizeof(IcpState), cudaMemcpyDeviceToHost, h->stream));
        pc.kind = 3; guard.ok = true;
        return B2_OK;
    }
    // ---- fused path: find per sensor, then ALL inner iterations of ALL sensors in one k_icp_loop ----
    IcpLaunch& L = pc.launch;
    const int grid = loop_layout(H, sc, ns, total, *Tom, iterations, L);
    RES(join_streams(sc, ns, true));
    bool aux_any = false;
    if (H->timing) CU(cudaEventRecord(H->ev[0], H->stream));
    for (uint32_t k = 0; k < ns; k++) {
        b2_rcc* h = sc[k].h;
        IcpSensor& S = L.s[k];
        const uint32_t nw = S.n;
        S.max_dist = adaptive_max_dist(h, cp);
        // Pinned scan (B2_ZEROCOPY, default 1): a copy engine moves it into the handle's buffer on the side stream WHILE find runs, a second small
        // copy behind it raises a flag, and the loop kernel -- launched programmatically behind find, no event in between -- checks the flag
        // before it unpacks the scan.  2: the loop kernel reads the caller's buffer itself over PCIe (latency-sensitive: 10-20 us slower on some
        // hosts).  Needs every pair of the sensor resident in registers / shared memory.  Pageable buffers take the staged upload below.
        const float* zc = nullptr; bool zc_dma = false;
        if (sc[k].ranges_host && nw > 0 && use_zc && nw <= (uint64_t)(B2_ICP_REG_PAIRS + S.smem_u) * S.nblk * B2_ICP_BLOCK) {
            cudaPointerAttributes pa;      // asked on every call (about a microsecond): an address can change from pinned to pageable between calls
            if (cudaPointerGetAttributes(&pa, sc[k].ranges_host) == cudaSuccess && pa.type == cudaMemoryTypeHost && pa.devicePointer) {
                if (use_zc == 2) zc = (const float*)pa.devicePointer; else { zc = h->d_ranges_in.p; zc_dma = true; }
            }
            (void)cudaGetLastError();
        }
        const bool need_upload = sc[k].ranges_host && nw > 0 && !zc;
        if (need_upload || zc_dma) {      // the side stream starts after whatever this sensor's stream had in flight BEFORE this call
            const cudaError_t idle = cudaStreamQuery(h->stream);        // (nothing in flight, the usual case of the synchronous calls: no event needed)
            if (idle != cudaSuccess) {
                (void)cudaGetLastError();
                CU(cudaEventRecord(h->ev_aux, h->stream));
                CU(cudaStreamWaitEvent(h->aux, h->ev_aux, 0));
            }
        }
        pc.sensors[k] = h; pc.Tbm[k] = body_in_map(*Tom, sc[k].Tbo);
        RES(find_on_lead(H, h, &pc.Tbm[k], nullptr, k + 1 == ns && mode == 2 && !H->timing && !need_upload && !aux_any));
        if (need_upload) {
            // the find kernel does not read the dataset: the scan is uploaded + unpacked on the side stream WHILE it runs
            CU(cudaMemcpyAsync(h->d_ranges_in.p, sc[k].ranges_host, sizeof(float) * h->n, cudaMemcpyHostToDevice, h->aux));
            k_dataset_from_ranges<<<(h->n + 255) / 256, 256, 0, h->aux>>>(h->d_ranges_in.p, h->d_dirs.p, h->d_origs.p, h->n_origs, h->n, h->range_min, h->range_max, h->d_dpts.p, h->d_dmask.p);
            LAUNCHED();
            CU(cudaEventRecord(h->ev_aux, h->aux));
            CU(cudaStreamWaitEvent(H->stream, h->ev_aux, 0));
            aux_any = true;
        }
        if (zc_dma) {
            // after the find launch, so that the GPU is busy while the host issues the two copies
            const int fs = (int)(H->slot_counter % B2_RING);
            h->pin->flag_src[fs] = ++h->zc_seq;
            CU(cudaMemcpyAsync(h->d_ranges_in.p, sc[k].ranges_host, sizeof(float) * h->n, cudaMemcpyHostToDevice, h->aux));
            CU(cudaMemcpyAsync(h->d_bar.p, &h->pin->flag_src[fs], sizeof(unsigned int), cudaMemcpyHostToDevice, h->aux));
            S.zc_flag = h->d_bar.p; S.zc_seq = h->zc_seq;
        }
        S.zc_ranges = zc; S.zc_dirs = h->d_dirs.p; S.zc_origs = h->d_origs.p; S.zc_n_origs = h->n_origs;
        S.dpts_out = h->d_dpts.p; S.dmask_out = h->d_dmask.p; S.ranges_out = h->d_ranges_in.p;
    }
    if (H->timing) CU(cudaEventRecord(H->ev[1], H->stream));
    pc.slot = (int)(H->slot_counter++ % B2_RING);
    RES(launch_loop_after_finds(H, sc, ns, L, grid, mode, !aux_any, pc.slot, &pc.smem));
    if (H->timing) { CU(cudaEventRecord(H->ev[2], H->stream)); H->timing_valid = true; }
    RES(join_streams(sc, ns, false));
    pc.seq = L.seq; pc.grid = grid; pc.barrier_used = mode == 2;
    if (use_spin) pc.kind = 1;
    else { CU(cudaMemcpyAsync(&H->pin->res[pc.slot], H->d_res.p, sizeof(IcpResult), cudaMemcpyDeviceToHost, H->stream)); pc.kind = 2; }
    guard.ok = true;
    return B2_OK;
}

static inline void cpu_relax()
{
#if defined(__x86_64__) || defined(__i386__)
    __builtin_ia32_pause();
#elif defined(__aarch64__)
    asm volatile("yield" ::: "memory");
#endif
}

// every chunk of the mapped result carries this call's sequence number?
static bool chunks_ready(const HostPin* pin, int slot, unsigned int seq)
{
    const volatile uint4* c = pin->chunks[slot];
    for (int i = 0; i < B2_ICP_RESULT_CHUNKS; i++) if (c[i].w != seq) return false;
    return true;
}
static void chunks_read(const HostPin* pin, int slot, IcpResult* out)
{
    std::atomic_thread_fence(std::memory_order_acquire);          // payload reads stay behind the sequence-number reads (aarch64 hosts)
    uint32_t w[3 * B2_ICP_RESULT_CHUNKS];
    for (int i = 0; i < B2_ICP_RESULT_CHUNKS; i++) { const volatile uint4* c = &pin->chunks[slot][i]; w[3 * i] = c->x; w[3 * i + 1] = c->y; w[3 * i + 2] = c->z; }
    memcpy(out, w, sizeof(IcpResult));
}

static int micp_collect(b2_rcc* H, b2_transform* Tom_new, b2_transform* T_onew_oold, b2_cross_stats* Cmerged)
{
    if (H->pending.empty()) return fail(B2_ERR_INVALID, "correctOnce: nothing to wait for");
    PendingCall pc = H->pending.front();
    H->pending.pop_front();
    bool have = pc.kind == 0;
    if (pc.kind == 1 && !pc.rerun) {
        // spin on the chunks the kernel writes into mapped host memory (a stream synchronise costs several microseconds more)
        const auto t_start = std::chrono::steady_clock::now();
        unsigned long long spins = 0;
        while (!chunks_ready(H->pin, pc.slot, pc.seq)) {
            cpu_relax();
            if ((++spins & 0xfffffull) == 0 && std::chrono::duration<double>(std::chrono::steady_clock::now() - t_start).count() > 5.0) break;
        }
        if (chunks_ready(H->pin, pc.slot, pc.seq)) { chunks_read(H->pin, pc.slot, &pc.res); have = true; }
    }
    if (!have) {
        const cudaError_t e = cudaStreamSynchronize(H->stream);
        if (e != cudaSuccess) { (void)cudaGetLastError(); return fail(B2_ERR_CUDA, "correctOnce: %s", cudaGetErrorString(e)); }
        if (pc.kind == 3) {
            const IcpState& st = H->pin->icp;
            pc.res.Tom_new = st.Tom_new; pc.res.T_onew_oold = st.T_onew_oold; pc.res.Cmerged_o = st.Cmerged_o;
        } else {
            if (pc.barrier_used && !pc.rerun) {
                // an abort: this call and every later call already in flight (their kernels saw the abort word and left) run again
                RES(exchange_aborted(H, &pc.rerun));
                if (pc.rerun) for (PendingCall& q : H->pending) if (q.barrier_used) q.rerun = true;
            }
            if (pc.rerun) {
                H->n_reruns++;
                for (uint32_t k = 0; k < pc.launch.n_sensors; k++) RES(find_on_lead(H, pc.sensors[k], &pc.Tbm[k], nullptr, false));
                pc.launch.seq = pc.seq = next_seq(H);
                RES(launch_icp_loop(H, pc.launch, pc.grid, pc.smem, 1, false, pc.slot));
                CU(cudaMemcpyAsync(&H->pin->res[pc.slot], H->d_res.p, sizeof(IcpResult), cudaMemcpyDeviceToHost, H->stream));
                CU(cudaStreamSynchronize(H->stream));
                memcpy(&pc.res, (const void*)&H->pin->res[pc.slot], sizeof(IcpResult));
            } else if (pc.kind == 1) {
                // spin timed out without an abort: the stream has drained meanwhile, the chunks must be there now
                if (!chunks_ready(H->pin, pc.slot, pc.seq)) return fail(B2_ERR_CUDA, "correctOnce: the result of the ICP loop never arrived");
                chunks_read(H->pin, pc.slot, &pc.res);
            } else memcpy(&pc.res, (const void*)&H->pin->res[pc.slot], sizeof(IcpResult));
        }
    }
    if (Tom_new) *Tom_new = pc.res.Tom_new;
    if (T_onew_oold) *T_onew_oold = pc.res.T_onew_oold;
    if (Cmerged) *Cmerged = pc.res.Cmerged_o;
    return B2_OK;
}

extern "C" int b2_rcc_set_exec_mode(b2_rcc* h, int mode)
{
    NOTNULL(h);
    if (mode < 0 || mode > 2) return fail(B2_ERR_INVALID, "unknown exec mode %d", mode);
    h->exec_mode = mode;
    return B2_OK;
}

extern "C" int b2_rcc_correct_once(b2_rcc* h, const b2_transform* Tom, const b2_transform* Tbo, uint32_t iterations, double cp,
                                   b2_transform* Tom_new, b2_transform* T_onew_oold, b2_cross_stats* Cmerged)
{
    NOTNULL(h); NOTNULL(Tom); NOTNULL(Tbo);
    CU(cudaSetDevice(h->map->device));
    if (!h->pending.empty()) return fail(B2_ERR_INVALID, "correctOnce: asynchronous calls are still in flight on this handle, collect them first");
    SensorCall sc{h, *Tbo, 1.0, nullptr, 0};
    RES(micp_enqueue(&sc, 1, Tom, iterations, cp));
    return micp_collect(h, Tom_new, T_onew_oold, Cmerged);
}

extern "C" int b2_rcc_correct_once_ranges(b2_rcc* h, const float* ranges, uint32_t n, const b2_transform* Tom, const b2_transform* Tbo, uint32_t iterations,
                                          double cp, b2_transform* Tom_new, b2_transform* T_onew_oold, b2_cross_stats* Cmerged)
{
    NOTNULL(h); NOTNULL(Tom); NOTNULL(Tbo);
    CU(cudaSetDevice(h->map->device));
    if (n) NOTNULL(ranges);
    if (!h->has_model) return fail(B2_ERR_INVALID, "set_ranges before setModel");
    SensorCall sc{h, *Tbo, 1.0, n ? ranges : nullptr, n};
    if (n == 0 && h->n != 0) return fail(B2_ERR_INVALID, "ranges size %u != model size %u", n, h->n);
    if (!h->pending.empty()) return fail(B2_ERR_INVALID, "correctOnce: asynchronous calls are still in flight on this handle, collect them first");
    RES(micp_enqueue(&sc, 1, Tom, iterations, cp));
    return micp_collect(h, Tom_new, T_onew_oold, Cmerged);
}

extern "C" int b2_rcc_correct_once_async(b2_rcc* h, const b2_transform* Tom, const b2_transform* Tbo, uint32_t iterations, double cp)
{
    NOTNULL(h); NOTNULL(Tom); NOTNULL(Tbo);
    CU(cudaSetDevice(h->map->device));
    SensorCall sc{h, *Tbo, 1.0, nullptr, 0};
    return micp_enqueue(&sc, 1, Tom, iterations, cp);
}

extern "C" int b2_rcc_correct_once_wait(b2_rcc* h, b2_transform* Tom_new, b2_transform* T_onew_oold, b2_cross_stats* Cmerged)
{
    NOTNULL(h);
    CU(cudaSetDevice(h->map->device));
    return micp_collect(h, Tom_new, T_onew_oold, Cmerged);
}

extern "C" int b2_micp_correct_once(b2_rcc* const* sensors, const b2_transform* Tbo, const double* merge_weights, const float* const* ranges_host, uint32_t n_sensors,
                                    const b2_transform* Tom, uint32_t iterations, double cp, b2_transform* Tom_new, b2_transform* T_onew_oold, b2_cross_stats* Cmerged)
{
    NOTNULL(sensors); NOTNULL(Tbo); NOTNULL(Tom);
    SensorCall sc[B2_MAX_SENSORS];
    RES(sensor_list(__func__, "correctOnce", sensors, Tbo, merge_weights, ranges_host, n_sensors, sc));
    RES(micp_enqueue(sc, n_sensors, Tom, iterations, cp));
    return micp_collect(sc[0].h, Tom_new, T_onew_oold, Cmerged);
}

// ---------------------------------------------------------------------------------------------------------------------
// b2_micp_correct: correctOnce after correctOnce (correct(), micp_localization.cpp:847-854) with the state between them -- Tom_, convergence_progress_
// -- in device memory (IcpChainState, icp_loop.cuh).  Per step the finds read Tom * Tbo from the state through their device-pose argument, the
// loop gates with the state's progress, and block 0 of the loop writes the next state and the step's record.  The lead handle's d_chain holds the
// state followed by the records; the host reads both once, at the end.
// ---------------------------------------------------------------------------------------------------------------------
static IcpChainState* chain_state(const b2_rcc* H) { return reinterpret_cast<IcpChainState*>(H->d_chain.p); }
static b2_micp_step* chain_records(const b2_rcc* H) { return reinterpret_cast<b2_micp_step*>(H->d_chain.p + sizeof(IcpChainState)); }

// one step: every sensor's find (the last one arms the programmatic launch, as in micp_enqueue), then the loop writing record `step`
static int chain_step(SensorCall* sc, uint32_t ns, IcpLaunch& L, int grid, int mode, uint32_t step)
{
    b2_rcc* H = sc[0].h;
    for (uint32_t k = 0; k < ns; k++) RES(find_on_lead(H, sc[k].h, nullptr, &chain_state(H)->find[k], k + 1 == ns && mode == 2));
    L.step_out = chain_records(H) + step;
    return launch_loop_after_finds(H, sc, ns, L, grid, mode, true, -1, nullptr);
}

extern "C" int b2_micp_correct(b2_rcc* const* sensors, const b2_transform* Tbo, const double* merge_weights, uint32_t n_sensors,
                               b2_transform* Tom_inout, double* cp_inout, int adaptive_max_dist, uint32_t n_corrections, uint32_t iterations, b2_micp_step* steps_out)
{
    NOTNULL(sensors); NOTNULL(Tbo); NOTNULL(Tom_inout); NOTNULL(cp_inout);
    SensorCall sc[B2_MAX_SENSORS];
    RES(sensor_list(__func__, "correct", sensors, Tbo, merge_weights, nullptr, n_sensors, sc));
    b2_rcc* H = sc[0].h;
    const uint32_t ns = n_sensors;
    if (H->fused_grid <= 0) return fail(B2_ERR_UNSUPPORTED, "correct: a chain of corrections needs a device with cooperative launch");
    const int mode = H->exec_mode == 0 ? 1 : H->exec_mode;           // exec mode 0 keeps its state on the host between reductions: the chain runs the fused loop
    uint64_t pairs = 0;
    RES(check_sensors(sc, ns, "correct", &pairs));
    const uint32_t total_meas = (uint32_t)pairs;                     // the dataset sizes: check_sensors saw n_dataset == work_n() for each
    if (n_corrections == 0) return B2_OK;
    const size_t bytes = sizeof(IcpChainState) + sizeof(b2_micp_step) * (size_t)n_corrections;
    RES(H->d_chain.reserve(bytes));
    RES(join_streams(sc, ns, true));
    {
        IcpChainState st; memset(&st, 0, sizeof(st));
        for (uint32_t k = 0; k < ns; k++) { st.find[k].Tom = *Tom_inout; st.find[k].Tbo = sc[k].Tbo; }
        st.cp = *cp_inout; st.total = total_meas;
        CU(cudaMemcpyAsync(H->d_chain.p, &st, sizeof(st), cudaMemcpyHostToDevice, H->stream));      // pageable source: staged before the call returns
        for (uint32_t k = 0; k < ns; k++) {
            const b2_rcc* h = sc[k].h;
            if (!h->n_dataset) continue;
            const int g = (int)std::min<uint32_t>((uint32_t)H->red_grid * 4u, (h->n_dataset + 255u) / 256u);
            k_mask_count<<<g, 256, 0, H->stream>>>(h->dmask(), h->n_dataset, &chain_state(H)->valid);
            LAUNCHED();
        }
    }
    std::vector<unsigned char> out(bytes);
    IcpChainState* got = reinterpret_cast<IcpChainState*>(out.data());
    b2_micp_step* rec = reinterpret_cast<b2_micp_step*>(out.data() + sizeof(IcpChainState));
    if (pairs == 0 || iterations == 0) {
        // Tom stays and the progress becomes 0 (micp_localization.cpp:974, :988-990); the finds still run (:900-908), at the same pose every step
        for (uint32_t k = 0; k < ns && pairs > 0; k++) {
            const b2_transform Tbm = body_in_map(*Tom_inout, sc[k].Tbo);
            RES(find_on_lead(H, sc[k].h, &Tbm, nullptr, false));
        }
        CU(cudaMemcpyAsync(out.data(), H->d_chain.p, sizeof(IcpChainState), cudaMemcpyDeviceToHost, H->stream));
        CU(cudaStreamSynchronize(H->stream));
        for (uint32_t s = 0; s < n_corrections; s++) {
            memset(&rec[s], 0, sizeof(b2_micp_step));
            rec[s].Tom_new = *Tom_inout; rec[s].T_onew_oold = tf_identity_pod(); rec[s].valid_measurements = got->valid; rec[s].total_measurements = total_meas;
        }
        got->find[0].Tom = *Tom_inout; got->cp = 0.0; got->done = n_corrections;
    } else {
        IcpLaunch L;
        const int grid = loop_layout(H, sc, ns, pairs, *Tom_inout, iterations, L);
        L.chain = chain_state(H); L.adaptive = adaptive_max_dist ? 1u : 0u;
        for (uint32_t k = 0; k < ns; k++) {          // the loop interpolates the gate with the progress (CorrespondencesCPU.cpp:21-23)
            L.s[k].max_dist = sc[k].h->max_dist; L.s[k].max_dist_min = sc[k].h->adaptive_max_dist_min;
        }
        for (uint32_t s = 0; s < n_corrections; s++) RES(chain_step(sc, ns, L, grid, mode, s));
        CU(cudaMemcpyAsync(out.data(), H->d_chain.p, bytes, cudaMemcpyDeviceToHost, H->stream));
        CU(cudaStreamSynchronize(H->stream));
        if (got->done < n_corrections) {
            // A mode-2 exchange gave up; the steps behind it saw the abort word and left.  The device state is the last completed step's: the
            // rest of the chain runs cooperatively.
            bool aborted = false;
            if (mode == 2) RES(exchange_aborted(H, &aborted));
            if (!aborted) return fail(B2_ERR_CUDA, "correct: step %u of %u left no record", got->done + 1, n_corrections);
            H->n_reruns++;
            for (uint32_t s = got->done; s < n_corrections; s++) RES(chain_step(sc, ns, L, grid, 1, s));
            CU(cudaMemcpyAsync(out.data(), H->d_chain.p, bytes, cudaMemcpyDeviceToHost, H->stream));
            CU(cudaStreamSynchronize(H->stream));
            if (got->done != n_corrections) return fail(B2_ERR_CUDA, "correct: the cooperative re-run left %u of %u records", got->done, n_corrections);
        }
    }
    RES(join_streams(sc, ns, false));
    *Tom_inout = got->find[0].Tom;
    *cp_inout = got->cp;
    if (steps_out) memcpy(steps_out, rec, sizeof(b2_micp_step) * (size_t)n_corrections);
    return B2_OK;
}

// ---------------------------------------------------------------------------------------------------------------------
// b2_micp_pose_covariance (SURVEY appendix I): one k_micp_information launch over the final correspondences of all sensors
// ---------------------------------------------------------------------------------------------------------------------
// row-major rotation matrix of a float quaternion, normalised in double
static void quat_to_mat_d(const b2_quat& q, double R[9])
{
    const double n = std::sqrt((double)q.x * q.x + (double)q.y * q.y + (double)q.z * q.z + (double)q.w * q.w);
    const double x = q.x / n, y = q.y / n, z = q.z / n, w = q.w / n;
    R[0] = 1.0 - 2.0 * (y * y + z * z); R[1] = 2.0 * (x * y - z * w); R[2] = 2.0 * (x * z + y * w);
    R[3] = 2.0 * (x * y + z * w); R[4] = 1.0 - 2.0 * (x * x + z * z); R[5] = 2.0 * (y * z - x * w);
    R[6] = 2.0 * (x * z - y * w); R[7] = 2.0 * (y * z + x * w); R[8] = 1.0 - 2.0 * (x * x + y * y);
}
// C = A B (transpose_a: A^T B, transpose_b: A B^T), 3x3 row-major
static void mat3_mul_d(const double* A, bool transpose_a, const double* B, bool transpose_b, double* C)
{
    for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) {
        double s = 0.0;
        for (int k = 0; k < 3; k++) s += (transpose_a ? A[k * 3 + i] : A[i * 3 + k]) * (transpose_b ? B[j * 3 + k] : B[k * 3 + j]);
        C[i * 3 + j] = s;
    }
}

extern "C" int b2_micp_pose_covariance(b2_rcc* const* sensors, const b2_transform* Tbo, const double* merge_weights, uint32_t n_sensors,
                                       const b2_transform* T_onew_oold, double cp, const b2_transform* Tbo_ref, const b2_micp_cov_config* cfg,
                                       b2_micp_covariance* out_host)
{
    NOTNULL(sensors); NOTNULL(Tbo); NOTNULL(T_onew_oold); NOTNULL(cfg); NOTNULL(out_host);
    static const char* what = "micp_pose_covariance";
    if (!(cfg->tau > 0.0 && cfg->tau < 1.0)) return fail(B2_ERR_INVALID, "%s: tau %g outside (0, 1)", what, cfg->tau);
    if (!(std::isfinite(cfg->degenerate_variance) && cfg->degenerate_variance > 0.0))
        return fail(B2_ERR_INVALID, "%s: degenerate_variance %g is not finite and > 0", what, cfg->degenerate_variance);
    SensorCall sc[B2_MAX_SENSORS];
    RES(sensor_list(__func__, what, sensors, Tbo, merge_weights, nullptr, n_sensors, sc));
    b2_rcc* H = sc[0].h;
    const uint32_t ns = n_sensors;
    const b2_transform Tref = Tbo_ref ? *Tbo_ref : Tbo[0];
    if (!all_finite(&T_onew_oold->R.x, 7) || !all_finite(&Tref.R.x, 7)) return fail(B2_ERR_INVALID, "%s: non-finite T_onew_oold or Tbo_ref", what);
    uint32_t n[B2_MAX_SENSORS]; uint64_t total = 0;
    for (uint32_t k = 0; k < ns; k++) {
        const b2_rcc* h = sc[k].h;
        if (h->map->device != H->map->device) return fail(B2_ERR_INVALID, "%s: all sensors must live on the same device", what);
        if (!h->pending.empty()) return fail(B2_ERR_INVALID, "%s: asynchronous calls are still in flight on sensor %u, collect them first", what, k);
        if (!h->found) return fail(B2_ERR_INVALID, "%s: sensor %u has no correspondences (find first)", what, k);
        if (h->n_dataset != h->n_model) return fail(B2_ERR_INVALID, "%s: sensor %u: dataset size %u != model size %u", what, k, h->n_dataset, h->n_model);
        if (!all_finite(&sc[k].Tbo.R.x, 7) || !all_finite(&h->Tsb.R.x, 7)) return fail(B2_ERR_INVALID, "%s: sensor %u: non-finite Tbo or Tsb", what, k);
        if (!(std::isfinite(sc[k].weight) && sc[k].weight >= 0.0)) return fail(B2_ERR_INVALID, "%s: sensor %u: merge weight %g is negative or not finite", what, k, sc[k].weight);
        n[k] = h->n_model; total += n[k];
    }
    MicpCovLaunch L; memset(&L, 0, sizeof(L));
    L.n_sensors = ns; L.tau = cfg->tau; L.degenerate_variance = cfg->degenerate_variance;
    uint32_t nblk[B2_MAX_SENSORS];
    const int grid = std::max(1, split_blocks(n, ns, total, H->red_grid, B2_COV_BLOCK, nblk));      // no pairs: one block writes the record
    double Rref[9]; quat_to_mat_d(Tref.R, Rref);
    uint32_t blk0 = 0;
    for (uint32_t k = 0; k < ns; k++) {
        const b2_rcc* h = sc[k].h;
        MicpCovSensor& S = L.s[k];
        S.dpts = h->dpts(); S.dmask = h->dmask(); S.mpts = h->mpts(); S.mnrm = h->mnrm(); S.mmask = h->mhits();
        S.n = n[k]; S.blk0 = blk0; S.nblk = nblk[k]; blk0 += nblk[k];
        S.max_dist = adaptive_max_dist(h, cp); S.weight = sc[k].weight;
        const Tf Tos = tf_mul(tf_from_pod(sc[k].Tbo), tf_from_pod(h->Tsb));
        const Tf Tpre = tf_mul(tf_mul(tf_inv(Tos), tf_from_pod(*T_onew_oold)), Tos);              // icp_tail_rest's pre-transform
        tf_store(&S.Tpre, Tpre);
        // U = ~Tbo_ref * Tbo * Tsb and R(U) R(Tpre)^T in double, each rounded to float once
        double Rbo[9], Rsb[9], Rpre[9], Rbs[9], RU[9], RN[9];
        quat_to_mat_d(sc[k].Tbo.R, Rbo); quat_to_mat_d(h->Tsb.R, Rsb);
        b2_quat qp; qp.x = Tpre.R.x; qp.y = Tpre.R.y; qp.z = Tpre.R.z; qp.w = Tpre.R.w;
        quat_to_mat_d(qp, Rpre);
        mat3_mul_d(Rbo, false, Rsb, false, Rbs);
        mat3_mul_d(Rref, true, Rbs, false, RU);
        mat3_mul_d(RU, false, Rpre, true, RN);
        const double tb[3] = {sc[k].Tbo.t.x, sc[k].Tbo.t.y, sc[k].Tbo.t.z}, ts[3] = {h->Tsb.t.x, h->Tsb.t.y, h->Tsb.t.z}, tr[3] = {Tref.t.x, Tref.t.y, Tref.t.z};
        double p[3];
        for (int i = 0; i < 3; i++) p[i] = Rbo[i * 3] * ts[0] + Rbo[i * 3 + 1] * ts[1] + Rbo[i * 3 + 2] * ts[2] + tb[i] - tr[i];
        for (int i = 0; i < 9; i++) { S.U[i] = (float)RU[i]; S.RN[i] = (float)RN[i]; }
        for (int i = 0; i < 3; i++) S.U[9 + i] = (float)(Rref[i] * p[0] + Rref[3 + i] * p[1] + Rref[6 + i] * p[2]);
    }
    RES(H->d_cov_part.reserve((size_t)B2_COV_NACC * std::max(H->red_grid, 1))); RES(H->d_cov_rec.reserve(1));
    if (!H->d_cov_ticket.p) { RES(H->d_cov_ticket.reserve(1)); CU(cudaMemset(H->d_cov_ticket.p, 0, sizeof(unsigned int))); }
    RES(join_streams(sc, ns, true));
    k_micp_information<<<grid, B2_COV_BLOCK, 0, H->stream>>>(L, H->d_cov_part.p, H->d_cov_ticket.p, H->d_cov_rec.p);
    LAUNCHED();
    b2_micp_covariance rec;
    CU(cudaMemcpyAsync(&rec, H->d_cov_rec.p, sizeof(rec), cudaMemcpyDeviceToHost, H->stream));
    RES(join_streams(sc, ns, false));
    CU(cudaStreamSynchronize(H->stream));
    *out_host = rec;
    return B2_OK;
}

extern "C" int b2_rcc_correct_batch(b2_rcc* h, const b2_transform* Tbm, uint32_t n_poses, int poses_on_device,
                                    b2_transform* Tdelta, uint32_t* ncorr, b2_cross_stats* stats_b, int out_on_device)
{
    NOTNULL(h);
    CU(cudaSetDevice(h->map->device));
    if (!h->has_model) return fail(B2_ERR_INVALID, "correct before setModel");
    if (n_poses == 0 || h->n == 0) return B2_OK;
    NOTNULL(Tbm);
    if (h->n_dataset != h->n) return fail(B2_ERR_INVALID, "correct before setInputData (dataset %u != model %u)", h->n_dataset, h->n);
    const b2_transform* poses_dev = Tbm;
    if (!poses_on_device) {
        RES(h->d_poses.reserve(n_poses));
        CU(cudaMemcpyAsync(h->d_poses.p, Tbm, sizeof(b2_transform) * (size_t)n_poses, cudaMemcpyHostToDevice, h->stream));
        poses_dev = h->d_poses.p;
    }
    const uint32_t rays_per_block = B2_FUSED_BLOCK * 8;
    const uint32_t bpp = (h->n + rays_per_block - 1) / rays_per_block;
    const uint64_t grid = (uint64_t)bpp * n_poses;
    if (grid > 0x7fffffffull) return fail(B2_ERR_INVALID, "too many poses");
    RES(h->d_partials.reserve((size_t)std::max<uint64_t>(grid, (uint64_t)h->red_grid) * (B2_NACC + 1)));
    k_rcc_fused_batch<<<(uint32_t)grid, B2_FUSED_BLOCK, 0, h->stream>>>(h->map->view(), poses_dev, h->Tsb, ray_model(h), h->dpts(), h->dmask(), h->max_dist,
                                                                       bpp, rays_per_block, h->d_partials.p);
    LAUNCHED();
    b2_transform* td = Tdelta; uint32_t* nc = ncorr; b2_cross_stats* sb = stats_b;
    if (!out_on_device) {
        RES(h->d_tdelta.reserve(n_poses)); RES(h->d_ncorr.reserve(n_poses)); RES(h->d_bstats.reserve(n_poses));
        td = h->d_tdelta.p; nc = h->d_ncorr.p; sb = h->d_bstats.p;
    }
    k_umeyama_from_partials<<<(n_poses + 63) / 64, 64, 0, h->stream>>>(h->d_partials.p, bpp, n_poses, h->Tsb, td, nc, sb);
    LAUNCHED();
    if (!out_on_device) {
        if (Tdelta) CU(cudaMemcpyAsync(Tdelta, td, sizeof(b2_transform) * (size_t)n_poses, cudaMemcpyDeviceToHost, h->stream));
        if (ncorr) CU(cudaMemcpyAsync(ncorr, nc, sizeof(uint32_t) * (size_t)n_poses, cudaMemcpyDeviceToHost, h->stream));
        if (stats_b) CU(cudaMemcpyAsync(stats_b, sb, sizeof(b2_cross_stats) * (size_t)n_poses, cudaMemcpyDeviceToHost, h->stream));
        CU(cudaStreamSynchronize(h->stream));
    }
    return B2_OK;
}

// v1 corrector.benchmark(Tbm, Nruns) -> {sim, red, svd} (rmcl_ros/src/benchmarks/lidar_corrector_optix_benchmark.cpp:143-155): the three stages
// of correct() run UNFUSED and timed separately with CUDA events (trace of all poses into pose-major model buffers, P2L reduction, Umeyama),
// summed over n_runs.  The production call b2_rcc_correct_batch fuses trace + reduction; this entry exists for the stage split only.
extern "C" int b2_rcc_benchmark_batch(b2_rcc* h, const b2_transform* Tbm_host, uint32_t n_poses, uint32_t n_runs, double* sim_s, double* red_s, double* svd_s)
{
    NOTNULL(h); NOTNULL(Tbm_host);
    CU(cudaSetDevice(h->map->device));
    if (!h->has_model || h->n == 0 || n_poses == 0 || n_runs == 0) return fail(B2_ERR_INVALID, "benchmark needs a model, poses and runs");
    if (h->n_dataset != h->n) return fail(B2_ERR_INVALID, "benchmark before setInputData (dataset %u != model %u)", h->n_dataset, h->n);
    const uint64_t total = (uint64_t)h->n * n_poses;
    if (total > 0x7fffffffull) return fail(B2_ERR_INVALID, "too many rays for the unfused benchmark (%llu)", (unsigned long long)total);
    DevBuf<float> pts, nrm, rng; DevBuf<uint8_t> hits; DevBuf<uint32_t> faces;
    auto cleanup = [&]() { pts.release(); nrm.release(); rng.release(); hits.release(); faces.release(); };
    int rc = B2_OK;
    if ((rc = pts.reserve(3 * total)) || (rc = nrm.reserve(3 * total)) || (rc = rng.reserve(total)) || (rc = hits.reserve(total)) || (rc = faces.reserve(total)) ||
        (rc = h->d_poses.reserve(n_poses)) || (rc = h->d_tdelta.reserve(n_poses)) || (rc = h->d_ncorr.reserve(n_poses)) || (rc = h->d_bstats.reserve(n_poses))) { cleanup(); return rc; }
    const uint32_t rays_per_block = B2_FUSED_BLOCK * 8, bpp = (h->n + rays_per_block - 1) / rays_per_block;
    if ((rc = h->d_partials.reserve((size_t)std::max<uint64_t>((uint64_t)bpp * n_poses, (uint64_t)std::max(h->red_grid, 2 * B2_ICP_MAX_GRID)) * (B2_NACC + 1)))) { cleanup(); return rc; }
    cudaEvent_t ev[4] = {nullptr, nullptr, nullptr, nullptr};
    cudaError_t e = cudaMemcpyAsync(h->d_poses.p, Tbm_host, sizeof(b2_transform) * (size_t)n_poses, cudaMemcpyHostToDevice, h->stream);
    for (int i = 0; i < 4 && e == cudaSuccess; i++) e = cudaEventCreate(&ev[i]);
    double acc[3] = {0, 0, 0};
    ModelBuffers out; out.pts = pts.p; out.nrm = nrm.p; out.hits = hits.p; out.faces = faces.p; out.ranges = rng.p;
    for (uint32_t r = 0; r < n_runs && e == cudaSuccess; r++) {
        cudaEventRecord(ev[0], h->stream);
        if ((rc = launch_rcc_find(h, total, 0, h->d_poses.p, nullptr, tf_identity_pod(), n_poses, out, 0, nullptr, nullptr)) != B2_OK) break;
        cudaEventRecord(ev[1], h->stream);
        k_p2l_batch<<<bpp * n_poses, B2_FUSED_BLOCK, 0, h->stream>>>(pts.p, nrm.p, hits.p, h->n, h->dpts(), h->dmask(), h->max_dist, bpp, rays_per_block, h->d_partials.p);
        cudaEventRecord(ev[2], h->stream);
        k_umeyama_from_partials<<<(n_poses + 63) / 64, 64, 0, h->stream>>>(h->d_partials.p, bpp, n_poses, h->Tsb, h->d_tdelta.p, h->d_ncorr.p, h->d_bstats.p);
        cudaEventRecord(ev[3], h->stream);
        g_launches.fetch_add(3);
        e = cudaEventSynchronize(ev[3]);
        for (int i = 0; i < 3 && e == cudaSuccess; i++) { float ms = 0.f; e = cudaEventElapsedTime(&ms, ev[i], ev[i + 1]); acc[i] += ms * 1e-3; }
        if (e == cudaSuccess) e = cudaGetLastError();
    }
    for (int i = 0; i < 4; i++) if (ev[i]) cudaEventDestroy(ev[i]);
    if (rc != B2_OK) CU(cudaStreamSynchronize(h->stream));
    cleanup();
    if (rc != B2_OK) return rc;
    if (e != cudaSuccess) { (void)cudaGetLastError(); return fail(B2_ERR_CUDA, "b2_rcc_benchmark_batch: %s", cudaGetErrorString(e)); }
    if (sim_s) *sim_s = acc[0]; if (red_s) *red_s = acc[1]; if (svd_s) *svd_s = acc[2];
    return B2_OK;
}

extern "C" int b2_umeyama_batch(const b2_cross_stats* stats, uint32_t n, b2_transform* out, int on_device, int device, void* stream_)
{
    if (n == 0) return B2_OK;
    NOTNULL(stats); NOTNULL(out);
    CU(cudaSetDevice(device));
    cudaStream_t stream = (cudaStream_t)stream_;
    if (on_device) {
        k_umeyama_batch<<<(n + 63) / 64, 64, 0, stream>>>(stats, n, out);
        LAUNCHED();
        return B2_OK;
    }
    DevBuf<b2_cross_stats> ds; DevBuf<b2_transform> dt;
    int rc;
    if ((rc = ds.reserve(n)) || (rc = dt.reserve(n))) { ds.release(); dt.release(); return rc; }
    cudaError_t e = cudaMemcpyAsync(ds.p, stats, sizeof(b2_cross_stats) * (size_t)n, cudaMemcpyHostToDevice, stream);
    if (e == cudaSuccess) { k_umeyama_batch<<<(n + 63) / 64, 64, 0, stream>>>(ds.p, n, dt.p); g_launches.fetch_add(1); e = cudaGetLastError(); }
    if (e == cudaSuccess) e = cudaMemcpyAsync(out, dt.p, sizeof(b2_transform) * (size_t)n, cudaMemcpyDeviceToHost, stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(stream);
    ds.release(); dt.release();
    if (e != cudaSuccess) return fail(B2_ERR_CUDA, "b2_umeyama_batch: %s", cudaGetErrorString(e));
    return B2_OK;
}

// ---------------------------------------------------------------------------------------------------------------------
// Memory-system micro-benchmark (bench.py's roofline denominators): read `bytes` with 128-bit loads from all SMs, `iters` launches timed with
// CUDA events after one warm-up pass.  A working set below the L2 capacity measures the L2 read bandwidth, a large one the HBM read bandwidth.
// ---------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(512) k_read_bw(const uint4* __restrict__ p, size_t n16, unsigned int* __restrict__ sink)
{
    unsigned int acc = 0;
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    for (; i + 3 * stride < n16; i += 4 * stride) {
        const uint4 a = __ldcg(p + i), b = __ldcg(p + i + stride), c = __ldcg(p + i + 2 * stride), d = __ldcg(p + i + 3 * stride);
        acc ^= a.x ^ a.y ^ a.z ^ a.w ^ b.x ^ b.y ^ b.z ^ b.w ^ c.x ^ c.y ^ c.z ^ c.w ^ d.x ^ d.y ^ d.z ^ d.w;
    }
    for (; i < n16; i += stride) { const uint4 a = __ldcg(p + i); acc ^= a.x ^ a.y ^ a.z ^ a.w; }
    if (acc == 0x12345678u) *sink = acc;            // never true in practice; keeps the loads alive
}
extern "C" int b2_debug_read_bandwidth(int device, uint64_t bytes, int iters, double* gbytes_per_s)
{
    NOTNULL(gbytes_per_s);
    if (bytes < 4096 || iters < 1) return fail(B2_ERR_INVALID, "b2_debug_read_bandwidth: bad arguments");
    CU(cudaSetDevice(device));
    int n_sm = 0; CU(cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, device));
    DevBuf<uint4> buf; DevBuf<unsigned int> sink;
    const size_t n16 = bytes / 16;
    int rc = buf.reserve(n16); if (rc == B2_OK) rc = sink.reserve(1);
    cudaEvent_t a = nullptr, b = nullptr;
    cudaError_t e = rc == B2_OK ? cudaMemset(buf.p, 1, n16 * 16) : cudaErrorMemoryAllocation;
    if (e == cudaSuccess) e = cudaEventCreate(&a);
    if (e == cudaSuccess) e = cudaEventCreate(&b);
    float ms = 0.f;
    if (e == cudaSuccess) {
        k_read_bw<<<n_sm * 4, 512>>>(buf.p, n16, sink.p);
        k_read_bw<<<n_sm * 4, 512>>>(buf.p, n16, sink.p);
        cudaEventRecord(a);
        for (int i = 0; i < iters; i++) k_read_bw<<<n_sm * 4, 512>>>(buf.p, n16, sink.p);
        cudaEventRecord(b);
        g_launches.fetch_add(iters + 2);
        e = cudaEventSynchronize(b);
        if (e == cudaSuccess) e = cudaEventElapsedTime(&ms, a, b);
        if (e == cudaSuccess) e = cudaGetLastError();
    }
    if (a) cudaEventDestroy(a); if (b) cudaEventDestroy(b);
    buf.release(); sink.release();
    if (rc != B2_OK) return rc;
    if (e != cudaSuccess) { (void)cudaGetLastError(); return fail(B2_ERR_CUDA, "b2_debug_read_bandwidth: %s", cudaGetErrorString(e)); }
    *gbytes_per_s = (double)(n16 * 16) * iters / (ms * 1e-3) / 1e9;
    return B2_OK;
}

// ---------------------------------------------------------------------------------------------------------------------
// particle filter
// ---------------------------------------------------------------------------------------------------------------------
// the fixed-size device records of the particle-filter entry points: one device block, zeroed at the handle's creation, and one pinned
// host mirror of the same layout that pf_fetch reads members back into
struct PfRecords {
    PfEstimateScratch est;                              // the estimate's two passes: record, Tbm, L_sum, tickets
    PfResidualState res;                                // the weight statistics (pf_weight_stats) and the residual's chunk record
    PfKldState kld;                                     // KLD's chunk record
    PfClusterState cl;                                  // the cluster labelling's record
    PfClusterHead heads[B2_CLUSTER_MAX_RECORDS];        // the recorded clusters' heads ...
    b2_particle_stats recs[B2_CLUSTER_MAX_RECORDS];     // ... and their estimates
    b2_recovery_state rec;                              // the recovery's {w_avg, w_slow, w_fast, p_inject}
    b2_recovery_result rec_res;                         // the result of an injection
    unsigned long long traffic;                         // remote bytes read by the p2p Gladiator kernel
    PfSteinState stein;                                 // the Stein step's result record and reduction tickets
};

// The scratch below (partials, records, the resamplers' and the clusters' buffers) is shared by the entry points: a handle serves one call at
// a time, and each call's work runs in h->stream order.
struct b2_pf {
    b2_mesh* map = nullptr; cudaStream_t stream = 0;
    DevBuf<PfBeam> d_beams; PfBeam* h_beams = nullptr; size_t h_beams_cap = 0;
    DevBuf<b2_transform> d_poses; DevBuf<b2_particle_attr> d_attrs;
    int n_sm = 0;
    int smem_optin = 0;
    cudaStream_t side = nullptr; cudaEvent_t ev_beams = nullptr, ev_side = nullptr;      // second stream of the chunked host variant (b2_pf_sensor_update_host)
    // ray mapping of k_pf_update (kernels.cuh): 0 lanes = beams, 1 lanes = particles, 2 lanes = particles sorted by pose, 3 (default) whichever of 0 / 2
    // was faster when last timed -- both are timed on the first updates and the loser again every 64 updates (particle sets converge and spread out)
    int map_mode = 3, map_cur = 0, map_best = 0; unsigned int map_updates = 0; float map_ms[2] = {0.f, 0.f}; bool map_timed = false;
    cudaEvent_t ev_m0 = nullptr, ev_m1 = nullptr;
    uint32_t launch_geom[12] = {};      // launch shape of the last sensor update that launched (b2_pf_debug_launch_geometry)
    DevBuf<uint32_t> d_keys, d_keys2, d_idx, d_idx2; DevBuf<unsigned char> d_sort_tmp;
    // sharded resampling over NVLink peer memory (b2_pf_p2p_*): own exchange buffers (cudaMalloc: exportable through CUDA IPC) + the peers' mappings
    b2_transform* x_poses = nullptr; b2_particle_attr* x_attrs = nullptr; uint32_t x_cap = 0;
    PfPeers peers{}; bool peers_open = false;
    // the records (PfRecords) and their pinned mirror; block partials of the grid reductions (k_pf_residual_stats and the estimate's two
    // passes): B2_EST_NV_MAX per block of at most 4 n_sm blocks
    DevBuf<PfRecords> d_recs; PfRecords* h_recs = nullptr; DevBuf<double> d_part;
    // beam sampling from a device cloud (b2_pf_sample_cloud): one record per sample, and its pinned host copy
    DevBuf<PfBeamSample> d_samples; PfBeamSample* h_samples = nullptr; uint32_t h_samples_cap = 0;
    // residual resampling (b2_pf_resample_residual), grown at its calls: per-draw parents, counts and their prefix for the largest chunk, and
    // the scan's temporary storage
    DevBuf<uint32_t> d_res_parents; DevBuf<unsigned long long> d_res_counts, d_res_prefix; DevBuf<unsigned char> d_res_tmp;
    // KLD-sampling (b2_pf_resample_kld), grown at its calls: integer weights and their prefix, the hash set (keys, first draws), per-draw
    // parents, hash slots, flags and their prefix for the largest chunk, the scan's temporary storage, and the yaw-sector table of kld_K
    // sectors with its host copy
    DevBuf<unsigned long long> d_kld_w, d_kld_W, d_kld_keys, d_kld_slots; DevBuf<unsigned int> d_kld_first; DevBuf<uint32_t> d_kld_parents, d_kld_flags, d_kld_cum;
    DevBuf<unsigned char> d_kld_tmp; DevBuf<float> d_kld_tab; std::vector<float> h_kld_tab; uint32_t kld_K = 0;
    // pose hypotheses (b2_pf_cluster_stats), grown at its calls.  It shares KLD's hash set (d_kld_keys; d_kld_first holds each slot's link
    // to its root), sector table, temporary storage and, for the cluster sort's keys, d_kld_w / d_kld_W.  Its own: per slot the weight, the
    // member count and the bin count / rank; per particle the slot, the sort key and the index, each of the latter two before and after the
    // sort (the index buffers also list the roots); and the gathered members
    DevBuf<unsigned long long> d_cl_w; DevBuf<unsigned int> d_cl_cnt, d_cl_aux; DevBuf<uint32_t> d_cl_slot, d_cl_key, d_cl_key2, d_cl_idx, d_cl_idx2;
    DevBuf<b2_transform> d_cl_poses; DevBuf<b2_particle_attr> d_cl_attrs;
    // Stein steps (b2_pf_stein_update), grown at its calls: J's snapshot, the RMSProp state of a call (3 floats per particle) and the block
    // partials of its two grid reductions (one block per 256 particles)
    DevBuf<SteinRef> d_stein_snap; DevBuf<float> d_stein_v; DevBuf<double> d_stein_part;
};

extern "C" int b2_pf_destroy(b2_pf* h);

static int pf_init(b2_pf* h)
{
    b2_mesh* map = h->map;
    CU(cudaDeviceGetAttribute(&h->smem_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, map->device));
    h->smem_optin -= 1024;              // room for the kernel's static shared memory
    CU(cudaDeviceGetAttribute(&h->n_sm, cudaDevAttrMultiProcessorCount, map->device));
    RES(h->d_part.reserve((size_t)B2_EST_NV_MAX * 4 * (size_t)h->n_sm)); RES(h->d_recs.reserve(1));
    CU(cudaMemset(h->d_recs.p, 0, sizeof(PfRecords)));
    CU(cudaMallocHost((void**)&h->h_recs, sizeof(PfRecords)));
    CU(cudaFuncSetAttribute(k_pf_update<0, 0>, cudaFuncAttributeMaxDynamicSharedMemorySize, h->smem_optin));
    CU(cudaFuncSetAttribute(k_pf_update<1, 0>, cudaFuncAttributeMaxDynamicSharedMemorySize, h->smem_optin));
    CU(cudaFuncSetAttribute(k_pf_update<0, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, h->smem_optin));
    CU(cudaFuncSetAttribute(k_pf_update<1, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, h->smem_optin));
    CU(cudaFuncSetAttribute(k_pf_update_field, cudaFuncAttributeMaxDynamicSharedMemorySize, h->smem_optin));
    CU(cudaFuncSetAttribute(k_pf_stein_score, cudaFuncAttributeMaxDynamicSharedMemorySize, h->smem_optin));
    CU(cudaEventCreate(&h->ev_m0)); CU(cudaEventCreate(&h->ev_m1));
    { const char* e = getenv("B2_PF_MAP"); if (e) h->map_mode = std::min(3, std::max(0, atoi(e))); }
    return B2_OK;
}

extern "C" int b2_pf_create(b2_mesh* map, b2_pf** out)
{
    NOTNULL(out); *out = nullptr;
    if (!map) return fail(B2_ERR_NO_MAP, "NO MAP");
    CU(cudaSetDevice(map->device));
    b2_pf* h = new (std::nothrow) b2_pf();
    if (!h) return fail(B2_ERR_OOM, "out of host memory");
    h->map = map;
    map->refs.fetch_add(1);             // released in b2_pf_destroy
    const int rc = pf_init(h);
    if (rc != B2_OK) { b2_pf_destroy(h); return rc; }
    *out = h;
    return B2_OK;
}
extern "C" int b2_pf_destroy(b2_pf* h)
{
    if (!h) return B2_OK;
    cudaSetDevice(h->map->device);
    cudaStreamSynchronize(h->stream);
    h->d_beams.release(); h->d_poses.release(); h->d_attrs.release(); h->d_part.release(); h->d_recs.release();
    if (h->h_beams) cudaFreeHost(h->h_beams);
    if (h->h_recs) cudaFreeHost(h->h_recs);
    if (h->side) { cudaStreamSynchronize(h->side); cudaStreamDestroy(h->side); }
    if (h->ev_beams) cudaEventDestroy(h->ev_beams);
    if (h->ev_side) cudaEventDestroy(h->ev_side);
    if (h->ev_m0) cudaEventDestroy(h->ev_m0);
    if (h->ev_m1) cudaEventDestroy(h->ev_m1);
    h->d_keys.release(); h->d_keys2.release(); h->d_idx.release(); h->d_idx2.release(); h->d_sort_tmp.release();
    if (h->peers_open) for (uint32_t r = 0; r < h->peers.world; r++) if (r != h->peers.rank) {
        if (h->peers.poses[r]) cudaIpcCloseMemHandle((void*)h->peers.poses[r]);
        if (h->peers.attrs[r]) cudaIpcCloseMemHandle((void*)h->peers.attrs[r]);
    }
    if (h->x_poses) cudaFree(h->x_poses);
    if (h->x_attrs) cudaFree(h->x_attrs);
    h->d_samples.release();
    if (h->h_samples) cudaFreeHost(h->h_samples);
    h->d_res_parents.release(); h->d_res_counts.release(); h->d_res_prefix.release(); h->d_res_tmp.release();
    h->d_kld_w.release(); h->d_kld_W.release(); h->d_kld_keys.release(); h->d_kld_slots.release(); h->d_kld_first.release(); h->d_kld_parents.release();
    h->d_kld_flags.release(); h->d_kld_cum.release(); h->d_kld_tmp.release(); h->d_kld_tab.release();
    h->d_cl_w.release(); h->d_cl_cnt.release(); h->d_cl_aux.release(); h->d_cl_slot.release(); h->d_cl_key.release(); h->d_cl_key2.release(); h->d_cl_idx.release();
    h->d_cl_idx2.release(); h->d_cl_poses.release(); h->d_cl_attrs.release();
    h->d_stein_snap.release(); h->d_stein_v.release(); h->d_stein_part.release();
    b2_mesh* map = h->map;
    delete h;
    (void)cudaGetLastError();
    mesh_unref(map);
    return B2_OK;
}
extern "C" int b2_pf_set_stream(b2_pf* h, void* s) { NOTNULL(h); h->stream = (cudaStream_t)s; return B2_OK; }

// read back: `count` elements starting at mirror_member (a member of h->h_recs) from the same offset of the device records, then a synchronise
template <class T> static int pf_fetch(b2_pf* h, const T& mirror_member, size_t count = 1)
{
    const size_t off = (size_t)((const char*)&mirror_member - (const char*)h->h_recs);
    CU(cudaMemcpyAsync((char*)h->h_recs + off, (const char*)h->d_recs.p + off, sizeof(T) * count, cudaMemcpyDeviceToHost, h->stream));
    CU(cudaStreamSynchronize(h->stream));
    return B2_OK;
}

// blocks of the grid reductions over n > 0 particles: 256 threads each, at most 4 per SM (grid-stride beyond)
static uint32_t pf_stats_grid(const b2_pf* h, uint32_t n) { return std::min<uint32_t>((uint32_t)h->n_sm * 4u, (n + 255) / 256); }

// The set's weight statistics S, L_min and L_max (k_pf_residual_stats) of n > 0 particles into h->d_recs.p->res, with read_back also into
// h->h_recs->res.  usable: the set can be resampled or clustered -- a NaN or infinite likelihood makes S non-finite, and all zero gives
// 0 / 0 in the reference (SURVEY D31).
static int pf_weight_stats(b2_pf* h, const b2_particle_attr* attrs_dev, uint32_t n, bool read_back, bool* usable = nullptr)
{
    k_pf_residual_stats<<<pf_stats_grid(h, n), 256, 0, h->stream>>>(attrs_dev, n, h->d_part.p, &h->d_recs.p->res);
    LAUNCHED();
    if (!read_back) return B2_OK;
    RES(pf_fetch(h, h->h_recs->res));
    const PfResidualState& r = h->h_recs->res;
    if (usable) *usable = std::isfinite(r.S) && r.S > 0.0 && r.L_min >= 0.0;
    return B2_OK;
}

static uint32_t dir_sort_key(const b2_range_meas& m)
{
    // Morton code of the direction on a 1024^3 lattice: neighbouring beams end up in the same warp (coherent traversal)
    auto q = [](float v) { int i = (int)((v * 0.5f + 0.5f) * 1023.0f); return (uint32_t)std::min(std::max(i, 0), 1023); };
    auto spread = [](uint32_t x) { x &= 0x3ff; x = (x | (x << 16)) & 0x30000ff; x = (x | (x << 8)) & 0x300f00f; x = (x | (x << 4)) & 0x30c30c3; x = (x | (x << 2)) & 0x9249249; return x; };
    return spread(q(m.dir.x)) | (spread(q(m.dir.y)) << 1) | (spread(q(m.dir.z)) << 2);
}

// beams: host -> compact, direction-sorted device table (merge order preserved through PfBeam::slot), on h->stream; particles per block
static int pf_prepare_beams(b2_pf* h, const b2_range_meas* beams, uint32_t n_beams, uint32_t* ppb_out)
{
    if (h->h_beams_cap < n_beams) {
        if (h->h_beams) cudaFreeHost(h->h_beams);
        h->h_beams = nullptr; h->h_beams_cap = 0;
        CU(cudaMallocHost((void**)&h->h_beams, sizeof(PfBeam) * (size_t)n_beams));
        h->h_beams_cap = n_beams;
    }
    RES(h->d_beams.reserve(n_beams));
    CU(cudaStreamSynchronize(h->stream));                 // previous launch may still read the staging buffer's device copy
    std::vector<std::pair<uint32_t, uint32_t>> order;
    try { order.resize(n_beams); } catch (const std::exception&) { return fail(B2_ERR_OOM, "out of host memory (%u beams)", n_beams); }
    for (uint32_t i = 0; i < n_beams; i++) order[i] = {dir_sort_key(beams[i]), i};
    std::sort(order.begin(), order.end());
    for (uint32_t j = 0; j < n_beams; j++) {
        const b2_range_meas& m = beams[order[j].second];
        PfBeam& b = h->h_beams[j];
        b.ox = m.orig.x; b.oy = m.orig.y; b.oz = m.orig.z; b.dx = m.dir.x; b.dy = m.dir.y; b.dz = m.dir.z; b.range = m.range; b.slot = order[j].second;
    }
    CU(cudaMemcpyAsync(h->d_beams.p, h->h_beams, sizeof(PfBeam) * (size_t)n_beams, cudaMemcpyHostToDevice, h->stream));
    // particles per block: as many as fit the shared-memory evaluation tile, capped so that a block still has enough rays
    const size_t bytes_per_particle = sizeof(float) * (size_t)n_beams;
    if (bytes_per_particle > (size_t)h->smem_optin) return fail(B2_ERR_UNSUPPORTED, "too many beams per update (%u)", n_beams);
    uint32_t ppb = (uint32_t)std::min<size_t>((size_t)h->smem_optin / bytes_per_particle, 64);
    const uint32_t want = std::max(1u, (B2_PF_BLOCK * 8 + n_beams - 1) / n_beams);       // ~8 rays per thread
    ppb = std::max(1u, std::min(ppb, want));
    *ppb_out = std::min(ppb, (uint32_t)B2_PF_BLOCK);
    return B2_OK;
}
// host-side record of an update's launch shape (b2_pf_debug_launch_geometry); pf_launch fills in the kernel's mapping, ppb, blocks and shared memory
static void pf_geom_begin(b2_pf* h, uint32_t n, uint32_t n_beams, int map, uint32_t n_chunks, uint32_t per)
{
    uint32_t* g = h->launch_geom;
    memset(g, 0, sizeof(h->launch_geom));
    g[0] = (uint32_t)h->smem_optin; g[1] = (uint32_t)h->map_mode; g[2] = (uint32_t)map; g[8] = n_chunks; g[9] = per; g[10] = n; g[11] = n_beams;
}
static int pf_launch(b2_pf* h, const b2_transform* poses_dev, b2_particle_attr* attrs_dev, uint32_t n, const b2_transform* Tsb, uint32_t n_beams, const b2_pf_params* prm,
                     uint32_t ppb, cudaStream_t stream, int map = 0, const uint32_t* order = nullptr)
{
    const size_t bytes_per_particle = sizeof(float) * (size_t)n_beams;
    if (map) { ppb = 32; if (bytes_per_particle * ppb > (size_t)h->smem_optin) { map = 0; order = nullptr; ppb = std::max(1u, (uint32_t)((size_t)h->smem_optin / bytes_per_particle)); } }
    const uint32_t grid = (n + ppb - 1) / ppb;
    const size_t smem = bytes_per_particle * ppb;
    const bool cp = prm->correspondence_type == 1;
    uint32_t* g = h->launch_geom;
    g[3] = (uint32_t)map; g[4] = order != nullptr; g[5] = ppb; g[6] += grid; g[7] = (uint32_t)smem;
    if (map) {
        if (cp) k_pf_update<1, 1><<<grid, B2_PF_BLOCK, smem, stream>>>(h->map->view(), poses_dev, attrs_dev, n, *Tsb, h->d_beams.p, n_beams, *prm, ppb, order);
        else    k_pf_update<0, 1><<<grid, B2_PF_BLOCK, smem, stream>>>(h->map->view(), poses_dev, attrs_dev, n, *Tsb, h->d_beams.p, n_beams, *prm, ppb, order);
    } else {
        if (cp) k_pf_update<1, 0><<<grid, B2_PF_BLOCK, smem, stream>>>(h->map->view(), poses_dev, attrs_dev, n, *Tsb, h->d_beams.p, n_beams, *prm, ppb, nullptr);
        else    k_pf_update<0, 0><<<grid, B2_PF_BLOCK, smem, stream>>>(h->map->view(), poses_dev, attrs_dev, n, *Tsb, h->d_beams.p, n_beams, *prm, ppb, nullptr);
    }
    LAUNCHED();
    return B2_OK;
}
// particles sorted by (heading bin, Morton cell) for the lanes = particles mapping: h->d_idx2 = particle at position p
static int pf_sort_particles(b2_pf* h, const b2_transform* poses_dev, uint32_t n, cudaStream_t stream)
{
    RES(h->d_keys.reserve(n)); RES(h->d_keys2.reserve(n)); RES(h->d_idx.reserve(n)); RES(h->d_idx2.reserve(n));
    const BvhView v = h->map->view();
    k_pf_sort_keys<<<(n + 255) / 256, 256, 0, stream>>>(poses_dev, n, v.bx, v.by, h->d_keys.p, h->d_idx.p);
    LAUNCHED();
    size_t tmp = 0;
    CU(cub::DeviceRadixSort::SortPairs(nullptr, tmp, h->d_keys.p, h->d_keys2.p, h->d_idx.p, h->d_idx2.p, (int)n, 0, 24, stream));
    RES(h->d_sort_tmp.reserve(tmp));
    CU(cub::DeviceRadixSort::SortPairs(h->d_sort_tmp.p, tmp, h->d_keys.p, h->d_keys2.p, h->d_idx.p, h->d_idx2.p, (int)n, 0, 24, stream));
    LAUNCHED();
    return B2_OK;
}
static int pf_update_impl(b2_pf* h, const b2_transform* poses_dev, b2_particle_attr* attrs_dev, uint32_t n, const b2_transform* Tsb,
                          const b2_range_meas* beams, uint32_t n_beams, const b2_pf_params* prm)
{
    if (n == 0 || n_beams == 0) return B2_OK;
    uint32_t ppb = 1;
    RES(pf_prepare_beams(h, beams, n_beams, &ppb));
    int map = h->map_mode;
    if (map == 3) {
        // timing of the previous update (pf_prepare_beams synchronised the stream: its events are complete)
        if (h->map_timed) {
            float ms = 0.f;
            if (cudaEventElapsedTime(&ms, h->ev_m0, h->ev_m1) == cudaSuccess) h->map_ms[h->map_cur ? 1 : 0] = ms; else (void)cudaGetLastError();
            h->map_timed = false;
        }
        const unsigned int k = h->map_updates++;
        if (n < 4096u) map = 0;                                        // too few particles for the sort to pay
        else if (k == 0) map = 0;
        else if (k == 1) map = 2;
        else {
            h->map_best = h->map_ms[1] > 0.f && h->map_ms[1] < h->map_ms[0] ? 2 : 0;
            map = (k % 64u) == 0u ? (h->map_best ? 0 : 2) : h->map_best;      // the other one gets another chance now and then
        }
        h->map_cur = map;
        CU(cudaEventRecord(h->ev_m0, h->stream));
    }
    pf_geom_begin(h, n, n_beams, map, 0, 0);
    const uint32_t* order = nullptr;
    if (map == 2) { RES(pf_sort_particles(h, poses_dev, n, h->stream)); order = h->d_idx2.p; }
    RES(pf_launch(h, poses_dev, attrs_dev, n, Tsb, n_beams, prm, ppb, h->stream, map != 0, order));
    if (h->map_mode == 3) { CU(cudaEventRecord(h->ev_m1, h->stream)); h->map_timed = true; }
    return B2_OK;
}

extern "C" int b2_pf_set_mapping(b2_pf* h, int mode)
{
    NOTNULL(h);
    if (mode < 0 || mode > 3) return fail(B2_ERR_INVALID, "unknown ray mapping %d", mode);
    h->map_mode = mode; h->map_updates = 0; h->map_timed = false; h->map_ms[0] = h->map_ms[1] = 0.f;
    return B2_OK;
}
extern "C" int b2_pf_get_mapping(b2_pf* h, int* mode, int* current)
{
    NOTNULL(h);
    if (mode) *mode = h->map_mode;
    if (current) *current = h->map_mode == 3 ? h->map_cur : h->map_mode;
    return B2_OK;
}
// test aid (not part of the public header): the launch shape of the handle's last sensor update that launched k_pf_update, so that tests can
// place beam and particle counts on its regime boundaries.  out[0] = dynamic shared memory a block may use (opt-in limit less the 1 KiB
// reserve), out[1] = requested mapping (b2_pf_set_mapping), out[2] = mapping chosen for the update (0 / 1 / 2; the host path always 0),
// out[3] = mapping of the kernel launched (0 lanes = beams, 1 lanes = particles; 0 where MAP 1 does not fit in shared memory),
// out[4] = 1 if the particles ran in sorted order, out[5] = particles per block, out[6] = blocks launched (all chunks), out[7] = dynamic
// shared memory per block in bytes, out[8] = chunks of the host path (0: device-resident call), out[9] = particles per chunk,
// out[10] = particles, out[11] = beams; 12 words
extern "C" __attribute__((visibility("default"))) int b2_pf_debug_launch_geometry(b2_pf* h, uint32_t* out)
{
    NOTNULL(h); NOTNULL(out);
    memcpy(out, h->launch_geom, sizeof(h->launch_geom));
    return B2_OK;
}

extern "C" int b2_pf_sensor_update(b2_pf* h, const b2_transform* poses_dev, b2_particle_attr* attrs_dev, uint32_t n, const b2_transform* Tsb,
                                   const b2_range_meas* beams, uint32_t n_beams, const b2_pf_params* prm)
{
    NOTNULL(h); NOTNULL(Tsb); NOTNULL(prm);
    if (n) { NOTNULL(poses_dev); NOTNULL(attrs_dev); }
    if (n_beams) NOTNULL(beams);
    CU(cudaSetDevice(h->map->device));
    return pf_update_impl(h, poses_dev, attrs_dev, n, Tsb, beams, n_beams, prm);
}

extern "C" int b2_pf_sensor_update_host(b2_pf* h, const b2_transform* poses, b2_particle_attr* attrs, uint32_t n, const b2_transform* Tsb,
                                        const b2_range_meas* beams, uint32_t n_beams, const b2_pf_params* prm)
{
    NOTNULL(h); NOTNULL(Tsb); NOTNULL(prm);
    if (n == 0) return B2_OK;
    NOTNULL(poses); NOTNULL(attrs);
    if (n_beams) NOTNULL(beams);
    CU(cudaSetDevice(h->map->device));
    RES(h->d_poses.reserve(n)); RES(h->d_attrs.reserve(n));
    if (n_beams == 0) return B2_OK;
    uint32_t ppb = 1;
    RES(pf_prepare_beams(h, beams, n_beams, &ppb));
    // Particles are independent: the set is cut into chunks that alternate between two streams, so that the upload of chunk i+1 and the
    // download of chunk i-1 (two copy engines) run under the kernel of chunk i.  With pinned host arrays the call then costs the kernel time
    // plus one chunk's transfers instead of kernel + all transfers.
    const uint32_t n_chunks = n >= 32768u ? 8u : 1u;
    const uint32_t per = ((n + n_chunks - 1) / n_chunks + ppb - 1) / ppb * ppb;          // whole blocks per chunk
    pf_geom_begin(h, n, n_beams, 0, n_chunks, per);
    if (n_chunks > 1) {
        if (!h->side) { CU(cudaStreamCreateWithFlags(&h->side, cudaStreamNonBlocking)); CU(cudaEventCreateWithFlags(&h->ev_beams, cudaEventDisableTiming)); CU(cudaEventCreateWithFlags(&h->ev_side, cudaEventDisableTiming)); }
        CU(cudaEventRecord(h->ev_beams, h->stream));                  // beam table (and whatever the caller had queued on the stream before)
        CU(cudaStreamWaitEvent(h->side, h->ev_beams, 0));
    }
    uint32_t c = 0;
    for (uint32_t first = 0; first < n; first += per, c++) {
        const uint32_t m = std::min(per, n - first);
        cudaStream_t st = (c & 1u) ? h->side : h->stream;
        CU(cudaMemcpyAsync(h->d_poses.p + first, poses + first, sizeof(b2_transform) * (size_t)m, cudaMemcpyHostToDevice, st));
        CU(cudaMemcpyAsync(h->d_attrs.p + first, attrs + first, sizeof(b2_particle_attr) * (size_t)m, cudaMemcpyHostToDevice, st));
        RES(pf_launch(h, h->d_poses.p + first, h->d_attrs.p + first, m, Tsb, n_beams, prm, ppb, st));
        CU(cudaMemcpyAsync(attrs + first, h->d_attrs.p + first, sizeof(b2_particle_attr) * (size_t)m, cudaMemcpyDeviceToHost, st));
    }
    if (n_chunks > 1) { CU(cudaEventRecord(h->ev_side, h->side)); CU(cudaStreamWaitEvent(h->stream, h->ev_side, 0)); }
    CU(cudaStreamSynchronize(h->stream));
    return B2_OK;
}

// ---------------------------------------------------------------------------------------------------------------------
// truncated distance field (kernels.cuh: FIELD, LAYOUT, LOOKUP).  A snapshot of the map at creation: it keeps a reference to the map, and a
// b2_mesh_refit afterwards leaves it as built.
// ---------------------------------------------------------------------------------------------------------------------
struct b2_dfield {
    b2_mesh* map = nullptr;
    DfieldView v{};
    uint64_t n_bricks = 0, n_alloc = 0;
    float build_ms = 0.f;
    DevBuf<uint32_t> d_index; DevBuf<float> d_bricks;
    DevBuf<float> d_qin, d_qout;                      // staging of host queries
};

extern "C" int b2_dfield_destroy(b2_dfield* f)
{
    if (!f) return B2_OK;
    cudaSetDevice(f->map->device);
    cudaDeviceSynchronize();
    f->d_index.release(); f->d_bricks.release(); f->d_qin.release(); f->d_qout.release();
    b2_mesh* map = f->map;
    delete f;
    (void)cudaGetLastError();
    mesh_unref(map);
    return B2_OK;
}

// grid-stride launches over up to 2^32 x 729 items: blocks of 256, at most 64 per SM
static unsigned dfield_grid(int n_sm, uint64_t n) { return (unsigned)std::max<uint64_t>(1u, std::min<uint64_t>((n + 255u) / 256u, (uint64_t)n_sm * 64u)); }

static int dfield_build(b2_dfield* f)
{
    b2_mesh* map = f->map;
    int n_sm = 0; CU(cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, map->device));
    const BvhView bvh = map->view();
    float ta, ta2, trunc2; df_limits(f->v, ta, ta2, trunc2);
    const uint64_t nb = f->n_bricks;
    RES(f->d_index.reserve(nb));
    DevBuf<uint32_t> offs, list; DevBuf<unsigned char> tmp;
    int rc = offs.reserve(nb);
    if (rc == B2_OK) {
        k_dfield_classify<<<dfield_grid(n_sm, nb), 256>>>(bvh, f->v, nb, ta, ta2, f->d_index.p);
        g_launches.fetch_add(1);
        size_t tmp_bytes = 0;
        cudaError_t e = cub::DeviceScan::ExclusiveSum(nullptr, tmp_bytes, f->d_index.p, offs.p, (int64_t)nb);
        if (e == cudaSuccess) rc = tmp.reserve(std::max<size_t>(tmp_bytes, 1));
        if (e == cudaSuccess && rc == B2_OK) e = cub::DeviceScan::ExclusiveSum(tmp.p, tmp_bytes, f->d_index.p, offs.p, (int64_t)nb);
        uint32_t last[2] = {0u, 0u};
        if (e == cudaSuccess && rc == B2_OK) e = cudaMemcpy(&last[0], offs.p + (nb - 1), sizeof(uint32_t), cudaMemcpyDeviceToHost);
        if (e == cudaSuccess && rc == B2_OK) e = cudaMemcpy(&last[1], f->d_index.p + (nb - 1), sizeof(uint32_t), cudaMemcpyDeviceToHost);
        if (e != cudaSuccess) rc = fail(B2_ERR_CUDA, "distance field classification failed: %s", cudaGetErrorString(e));
        f->n_alloc = (uint64_t)last[0] + last[1];
        tmp.release();
        if (rc == B2_OK && f->n_alloc) rc = list.reserve(f->n_alloc);
        if (rc == B2_OK && f->n_alloc) rc = f->d_bricks.reserve(f->n_alloc * B2_DF_NODES);
        if (rc == B2_OK) {
            k_dfield_index<<<dfield_grid(n_sm, nb), 256>>>(nb, offs.p, f->d_index.p, f->n_alloc ? list.p : nullptr);
            g_launches.fetch_add(1);
            if (f->n_alloc) {
                f->v.index = f->d_index.p; f->v.bricks = f->d_bricks.p;
                k_dfield_fill<<<dfield_grid(n_sm, f->n_alloc * B2_DF_NODES), 256>>>(bvh, f->v, list.p, f->n_alloc * B2_DF_NODES, trunc2, f->d_bricks.p);
                g_launches.fetch_add(1);
            }
            e = cudaDeviceSynchronize();
            if (e == cudaSuccess) e = cudaGetLastError();
            if (e != cudaSuccess) rc = fail(B2_ERR_CUDA, "distance field build failed: %s", cudaGetErrorString(e));
        }
    }
    offs.release(); list.release();
    f->v.index = f->d_index.p; f->v.bricks = f->d_bricks.p;
    return rc;
}

extern "C" int b2_dfield_create(b2_mesh* map, const b2_dfield_params* prm, b2_dfield** out)
{
    NOTNULL(out); *out = nullptr;
    NOTNULL(map); NOTNULL(prm);
    if ((prm->bb_min == nullptr) != (prm->bb_max == nullptr)) return fail(B2_ERR_INVALID, "dfield_create: give both bb_min and bb_max or neither");
    const float h = prm->resolution, trunc = prm->truncation;
    if (!(std::isfinite(h) && h > 0.0f && std::isfinite(trunc) && trunc > 0.0f))
        return fail(B2_ERR_INVALID, "dfield_create: resolution %g and truncation %g must be finite and > 0", (double)h, (double)trunc);
    if (map->n_faces == 0) return fail(B2_ERR_NO_MAP, "EMPTY MAP");
    float lo[3], hi[3];
    CU(cudaSetDevice(map->device));
    if (prm->bb_min) { for (int k = 0; k < 3; k++) { lo[k] = prm->bb_min[k]; hi[k] = prm->bb_max[k]; } }
    else {
        // the map's AABB: the union of the root's child boxes (exact float AABBs of the triangles; empty slots are +inf / -inf), grown by trunc
        B2Node8 root;
        CU(cudaMemcpy(&root, map->d_nodes, sizeof(B2Node8), cudaMemcpyDeviceToHost));
        for (int k = 0; k < 3; k++) {
            float a = INFINITY, b = -INFINITY;
            for (int s = 0; s < 8; s++) { a = std::min(a, root.lo[k][s]); b = std::max(b, root.hi[k][s]); }
            lo[k] = a - trunc; hi[k] = b + trunc;
        }
    }
    DfieldView v; uint64_t nb = 0;
    if (const char* why = df_grid(lo, hi, h, trunc, &v, &nb)) return fail(B2_ERR_INVALID, "dfield_create: %s", why);
    b2_dfield* f = new (std::nothrow) b2_dfield();
    if (!f) return fail(B2_ERR_OOM, "out of host memory");
    f->map = map; f->v = v; f->n_bricks = nb;
    map->refs.fetch_add(1);             // released in b2_dfield_destroy
    const auto t0 = std::chrono::steady_clock::now();
    const int rc = dfield_build(f);
    if (rc != B2_OK) { b2_dfield_destroy(f); return rc; }
    f->build_ms = std::chrono::duration<float, std::milli>(std::chrono::steady_clock::now() - t0).count();
    *out = f;
    return B2_OK;
}

extern "C" int b2_dfield_get_info(const b2_dfield* f, b2_dfield_info* info)
{
    NOTNULL(f); NOTNULL(info);
    b2_dfield_info r{};
    r.dims[0] = f->v.dx; r.dims[1] = f->v.dy; r.dims[2] = f->v.dz;
    r.brick_dims[0] = f->v.bx; r.brick_dims[1] = f->v.by; r.brick_dims[2] = f->v.bz;
    r.origin[0] = f->v.ox; r.origin[1] = f->v.oy; r.origin[2] = f->v.oz;
    r.resolution = f->v.h; r.inv_resolution = f->v.inv_h; r.truncation = f->v.trunc;
    r.bricks_total = f->n_bricks; r.bricks_allocated = f->n_alloc;
    r.bytes = sizeof(uint32_t) * f->n_bricks + sizeof(float) * B2_DF_NODES * f->n_alloc;
    r.build_ms = f->build_ms; r.device = f->map->device;
    *info = r;
    return B2_OK;
}

extern "C" int b2_dfield_download(const b2_dfield* f, uint32_t* index_host, float* bricks_host)
{
    NOTNULL(f);
    CU(cudaSetDevice(f->map->device));
    if (index_host) CU(cudaMemcpy(index_host, f->d_index.p, sizeof(uint32_t) * f->n_bricks, cudaMemcpyDeviceToHost));
    if (bricks_host && f->n_alloc) CU(cudaMemcpy(bricks_host, f->d_bricks.p, sizeof(float) * B2_DF_NODES * f->n_alloc, cudaMemcpyDeviceToHost));
    return B2_OK;
}

extern "C" int b2_dfield_query(b2_dfield* f, const float* points_xyz, uint32_t n, float* dist_out, int src_is_device)
{
    NOTNULL(f);
    if (n == 0) return B2_OK;
    NOTNULL(points_xyz); NOTNULL(dist_out);
    CU(cudaSetDevice(f->map->device));
    const float* pin = points_xyz; float* pout = dist_out;
    if (!src_is_device) {
        RES(f->d_qin.reserve(3 * (size_t)n)); RES(f->d_qout.reserve(n));
        CU(cudaMemcpy(f->d_qin.p, points_xyz, sizeof(float) * 3 * (size_t)n, cudaMemcpyHostToDevice));
        pin = f->d_qin.p; pout = f->d_qout.p;
    }
    k_dfield_query<<<(n + 255) / 256, 256>>>(f->v, pin, n, pout);
    LAUNCHED();
    if (!src_is_device) CU(cudaMemcpy(dist_out, pout, sizeof(float) * (size_t)n, cudaMemcpyDeviceToHost));
    else CU(cudaDeviceSynchronize());
    return B2_OK;
}

extern "C" int b2_pf_sensor_update_field(b2_pf* h, const b2_dfield* f, const b2_transform* poses_dev, b2_particle_attr* attrs_dev, uint32_t n,
                                         const b2_transform* Tsb, const b2_range_meas* beams, uint32_t n_beams, const b2_pf_params* prm)
{
    NOTNULL(h); NOTNULL(f); NOTNULL(Tsb); NOTNULL(prm);
    if (n) { NOTNULL(poses_dev); NOTNULL(attrs_dev); }
    if (n_beams) NOTNULL(beams);
    if (f->map->device != h->map->device) return fail(B2_ERR_INVALID, "pf_sensor_update_field: the field is on device %d, the handle on device %d", f->map->device, h->map->device);
    CU(cudaSetDevice(h->map->device));
    if (n == 0 || n_beams == 0) return B2_OK;
    uint32_t ppb = 1;
    RES(pf_prepare_beams(h, beams, n_beams, &ppb));
    const uint32_t grid = (n + ppb - 1) / ppb;
    k_pf_update_field<<<grid, B2_PF_BLOCK, sizeof(float) * (size_t)n_beams * ppb, h->stream>>>(f->v, poses_dev, attrs_dev, n, *Tsb, h->d_beams.p, n_beams, *prm, ppb);
    LAUNCHED();
    return B2_OK;
}

// Stein variational steps (kernels.cuh, SURVEY appendix L): per iteration the score of J, the bandwidth and the move, all on h->stream
extern "C" int b2_pf_stein_update(b2_pf* h, const b2_dfield* f, b2_transform* poses_dev, uint32_t n, const b2_transform* Tsb, const b2_range_meas* beams,
                                  uint32_t n_beams, const b2_pf_params* prm, const b2_stein_config* cfg, uint64_t seed, uint32_t step, b2_stein_result* out_host)
{
    NOTNULL(h); NOTNULL(f); NOTNULL(Tsb); NOTNULL(prm); NOTNULL(cfg);
    if (n) NOTNULL(poses_dev);
    if (n_beams) NOTNULL(beams);
    if (f->map->device != h->map->device) return fail(B2_ERR_INVALID, "pf_stein_update: the field is on device %d, the handle on device %d", f->map->device, h->map->device);
    const b2_stein_config c = *cfg;
    auto pos = [](float v) { return std::isfinite(v) && v > 0.0f; };
    if (!(pos(c.step_t) && pos(c.step_r) && pos(c.min_bandwidth_t) && pos(c.min_bandwidth_r)))
        return fail(B2_ERR_INVALID, "pf_stein_update: steps (%g, %g) and bandwidth floors (%g, %g) must be finite and > 0", (double)c.step_t, (double)c.step_r,
                    (double)c.min_bandwidth_t, (double)c.min_bandwidth_r);
    if (!(c.w_rand >= 0.0f && c.w_rand < 1.0f)) return fail(B2_ERR_INVALID, "pf_stein_update: w_rand = %g outside [0, 1)", (double)c.w_rand);
    if (!pos(prm->dist_sigma)) return fail(B2_ERR_INVALID, "pf_stein_update: dist_sigma = %g must be finite and > 0", (double)prm->dist_sigma);
    if (out_host) memset(out_host, 0, sizeof(*out_host));
    CU(cudaSetDevice(h->map->device));
    if (n == 0 || c.iterations == 0) return B2_OK;
    const uint32_t m = (c.n_ref == 0 || c.n_ref >= n) ? n : c.n_ref;
    uint32_t ppb = B2_PF_BLOCK;
    if (n_beams) {
        if (sizeof(float) * 3 * (size_t)n_beams > (size_t)h->smem_optin) return fail(B2_ERR_UNSUPPORTED, "pf_stein_update: too many beams (%u)", n_beams);
        RES(pf_prepare_beams(h, beams, n_beams, &ppb));
        ppb = std::max<uint32_t>(1u, std::min<uint32_t>(ppb, (uint32_t)((size_t)h->smem_optin / (sizeof(float) * 3 * (size_t)n_beams))));
    }
    const uint32_t grid = (n + B2_STEIN_BLOCK - 1) / B2_STEIN_BLOCK;
    RES(h->d_stein_snap.reserve(m)); RES(h->d_stein_v.reserve(3 * (size_t)n));
    RES(h->d_stein_part.reserve((size_t)std::max(B2_STEIN_NBW, B2_STEIN_NMV) * grid));
    PfSteinState* st = &h->d_recs.p->stein;
    CU(cudaMemsetAsync(&st->rec, 0, sizeof(b2_stein_result), h->stream));
    CU(cudaMemsetAsync(h->d_stein_v.p, 0, sizeof(float) * 3 * (size_t)n, h->stream));
    const BvhView bvh = h->map->view();
    const double fac = std::pow((double)m, -1.0 / 7.0);                    // Scott's rule in 3 dimensions
    const float sigma2 = prm->dist_sigma * prm->dist_sigma;
    for (uint32_t it = 0; it < c.iterations; it++) {
        k_pf_stein_score<<<(m + ppb - 1) / ppb, B2_PF_BLOCK, sizeof(float) * 3 * (size_t)n_beams * ppb, h->stream>>>(f->v, poses_dev, n, m, c.n_ref, seed, step, it, *Tsb,
                                                                                                                 h->d_beams.p, n_beams, sigma2, c.w_rand, ppb, h->d_stein_snap.p);
        LAUNCHED();
        k_pf_stein_bandwidth<<<grid, B2_STEIN_BLOCK, 0, h->stream>>>(poses_dev, n, m, fac, c.min_bandwidth_t, c.min_bandwidth_r, h->d_stein_part.p, st);
        LAUNCHED();
        k_pf_stein_move<<<grid, B2_STEIN_BLOCK, 0, h->stream>>>(bvh, poses_dev, n, h->d_stein_snap.p, m, it, c.step_t, c.step_r, h->d_stein_v.p, h->d_stein_part.p, st);
        LAUNCHED();
    }
    if (out_host) {
        RES(pf_fetch(h, h->h_recs->stein.rec));
        *out_host = h->h_recs->stein.rec;
    }
    return B2_OK;
}

// PCDSensorUpdaterOptix::update's beam sampling (PCDSensorUpdaterOptix.cpp:227-311).  pf_sample_beam (kernels.cuh) runs where the cloud
// lives: a device cloud by k_pf_sample_cloud on the handle's stream, after which 68 B per sample come back; a host cloud by the same
// function in a host loop that reads only the points it draws, so the cloud is never uploaded (scripts/bench_pf_cloud.py measures both).
// The give-up rule then runs over the samples in order.
extern "C" int b2_pf_sample_cloud(b2_pf* h, const void* data, uint64_t bytes, const b2_cloud_layout* L, int src_is_device, uint32_t n_samples,
                                  uint64_t seed, uint32_t step, b2_range_meas* beams, uint32_t* n_beams)
{
    NOTNULL(L); NOTNULL(n_beams);                   // the arguments are checked before the handle: the checks need no device
    const uint64_t n_points = (uint64_t)L->width * L->height;
    if (n_points) NOTNULL(data);
    if (n_samples) NOTNULL(beams);
    if (n_points > 0xffffffffull) return fail(B2_ERR_INVALID, "pf_sample_cloud: %llu points, at most 2^32 - 1 are read", (unsigned long long)n_points);
    uint64_t need = 0;
    RES(check_cloud_layout(L, bytes, n_points != 0, n_points ? L->height - 1 : 0, n_points ? L->width - 1 : 0, "pf_sample_cloud", "", "", &need));
    NOTNULL(h);
    *n_beams = 0;
    if (n_points == 0 || n_samples == 0) return B2_OK;
    CloudBeams c;
    c.width = L->width; c.n_points = (uint32_t)n_points; c.row_step = L->row_step; c.point_step = L->point_step;
    c.off[0] = L->offset_x; c.off[1] = L->offset_y; c.off[2] = L->offset_z;
    c.f64 = L->datatype == 8 ? 1u : 0u;
    c.seed = seed; c.step = step;
    const uint8_t* src = static_cast<const uint8_t*>(data);
    if (src_is_device) {
        CU(cudaSetDevice(h->map->device));
        RES(h->d_samples.reserve(n_samples));
        if (h->h_samples_cap < n_samples) {
            if (h->h_samples) cudaFreeHost(h->h_samples);
            h->h_samples = nullptr; h->h_samples_cap = 0;
            CU(cudaMallocHost((void**)&h->h_samples, sizeof(PfBeamSample) * (size_t)n_samples));
            h->h_samples_cap = n_samples;
        }
        k_pf_sample_cloud<<<(n_samples + 127) / 128, 128, 0, h->stream>>>(src, c, n_samples, h->d_samples.p);
        LAUNCHED();
        CU(cudaMemcpyAsync(h->h_samples, h->d_samples.p, sizeof(PfBeamSample) * (size_t)n_samples, cudaMemcpyDeviceToHost, h->stream));
        CU(cudaStreamSynchronize(h->stream));
    }
    uint32_t n_out = 0, invalids = 0;
    for (uint32_t k = 0; k < n_samples && invalids < B2_PF_BEAM_MAX_INVALIDS; k++) {       // :264-287: stop at the 10th sample that found no point
        b2_range_meas m;
        const bool valid = src_is_device ? (m = h->h_samples[k].m, h->h_samples[k].valid != 0u) : pf_sample_beam(src, c, k, &m);
        if (valid) beams[n_out++] = m;
        else invalids++;
    }
    *n_beams = n_out;
    return B2_OK;
}

extern "C" int b2_pf_motion_update(b2_pf* h, b2_transform* poses_dev, b2_particle_attr* attrs_dev, uint32_t n, const b2_transform* T, double forget_rate, int check_collision)
{
    NOTNULL(h); NOTNULL(T);
    if (n == 0) return B2_OK;
    NOTNULL(poses_dev); NOTNULL(attrs_dev);
    CU(cudaSetDevice(h->map->device));
    if (check_collision) k_pf_motion<true><<<(n + 127) / 128, 128, 0, h->stream>>>(h->map->view(), poses_dev, attrs_dev, n, *T, forget_rate);
    else                 k_pf_motion<false><<<(n + 127) / 128, 128, 0, h->stream>>>(h->map->view(), poses_dev, attrs_dev, n, *T, forget_rate);
    LAUNCHED();
    return B2_OK;
}

// the checks of a surface config (`what` names the caller in the message), and the constants the rule takes from it
static int surface_config_check(const b2_surface_config& c, const char* what, float* cos_max, float* tfar)
{
    const float f[4] = {c.probe_above, c.probe_below, c.base_height, c.max_slope};
    if (!all_finite(f, 4)) return fail(B2_ERR_INVALID, "%s: a config field is not finite (%g, %g, %g, %g)", what, f[0], f[1], f[2], f[3]);
    *tfar = c.probe_above + c.probe_below;
    if (c.probe_above < 0.0f || c.probe_below < 0.0f || !(*tfar > 0.0f))
        return fail(B2_ERR_INVALID, "%s: probe_above %g and probe_below %g must be >= 0 with a positive sum", what, f[0], f[1]);
    if (c.base_height < 0.0f) return fail(B2_ERR_INVALID, "%s: base_height %g < 0", what, f[2]);
    if (!(c.max_slope >= 0.0f && c.max_slope <= (float)1.5707963267948966))           // pi/2 rounded to float, as a caller passes it
        return fail(B2_ERR_INVALID, "%s: max_slope %g outside [0, pi/2]", what, f[3]);
    if (c.align != 0 && c.align != 1) return fail(B2_ERR_INVALID, "%s: align is 0 or 1, not %d", what, (int)c.align);
    *cos_max = (float)std::cos((double)c.max_slope);
    return B2_OK;
}

// the motion stage's surface constraint (docs/RMCL.md:72; SURVEY appendix F): one downward ray per particle, in place
extern "C" int b2_pf_project_to_surface(b2_pf* h, b2_transform* poses_dev, b2_particle_attr* attrs_dev, uint32_t n, const b2_surface_config* cfg)
{
    NOTNULL(h); NOTNULL(cfg);
    if (n > 0) { NOTNULL(poses_dev); NOTNULL(attrs_dev); }
    const b2_surface_config c = *cfg;
    float cos_max, tfar;
    RES(surface_config_check(c, "project to surface", &cos_max, &tfar));
    if (n == 0) return B2_OK;
    CU(cudaSetDevice(h->map->device));
    k_pf_surface<<<(n + 127) / 128, 128, 0, h->stream>>>(h->map->view(), poses_dev, attrs_dev, n, c, cos_max, tfar);
    LAUNCHED();
    return B2_OK;
}

extern "C" int b2_pf_resample_gladiator(b2_pf* h, const b2_transform* poses_dev, const b2_particle_attr* attrs_dev, uint32_t n_all, uint32_t first, uint32_t n_local,
                                        b2_transform* poses_new_dev, b2_particle_attr* attrs_new_dev, const b2_gladiator_config* cfg, uint64_t seed, uint32_t step,
                                        const uint32_t* raw_dev, const float* normals_dev)
{
    NOTNULL(h); NOTNULL(cfg);
    if ((uint64_t)first + n_local > n_all) return fail(B2_ERR_INVALID, "champion range %u+%u exceeds the %u particles", first, n_local, n_all);
    if ((raw_dev == nullptr) != (normals_dev == nullptr)) return fail(B2_ERR_INVALID, "raw_dev and normals_dev must be given together");
    if (n_local == 0) return B2_OK;
    NOTNULL(poses_dev); NOTNULL(attrs_dev); NOTNULL(poses_new_dev); NOTNULL(attrs_new_dev);
    if ((const void*)poses_dev == (const void*)poses_new_dev || (const void*)attrs_dev == (const void*)attrs_new_dev)
        return fail(B2_ERR_INVALID, "resampling is not in place: outputs must not alias the inputs (resampling.cu:112-117 double-buffers)");
    CU(cudaSetDevice(h->map->device));
    k_pf_gladiator<<<(n_local + 255) / 256, 256, 0, h->stream>>>(poses_dev, attrs_dev, n_all, first, n_local, poses_new_dev, attrs_new_dev, *cfg, seed, step, raw_dev, normals_dev);
    LAUNCHED();
    return B2_OK;
}

// ---- sharded Gladiator resampling over NVLink peer memory ------------------------------------------------------------------------------------
// Life cycle (one process per GPU):  init -> exchange the 128-byte handles of all ranks (any transport: torch.distributed all_gather) -> connect;
// then per resampling step: publish (device-to-device copy of the local particles into the exported buffers), a cross-rank barrier, resample_p2p,
// a second barrier before the next publish.
extern "C" int b2_pf_p2p_init(b2_pf* h, uint32_t n_per_rank, void* handles_out_128)
{
    NOTNULL(h); NOTNULL(handles_out_128);
    if (n_per_rank == 0) return fail(B2_ERR_INVALID, "p2p: empty shard");
    CU(cudaSetDevice(h->map->device));
    if (h->peers_open) return fail(B2_ERR_INVALID, "p2p: already connected");
    if (h->x_cap < n_per_rank) {
        if (h->x_poses) cudaFree(h->x_poses); if (h->x_attrs) cudaFree(h->x_attrs);
        h->x_poses = nullptr; h->x_attrs = nullptr; h->x_cap = 0;
        CU(cudaMalloc((void**)&h->x_poses, sizeof(b2_transform) * (size_t)n_per_rank));
        CU(cudaMalloc((void**)&h->x_attrs, sizeof(b2_particle_attr) * (size_t)n_per_rank));
        h->x_cap = n_per_rank;
    }
    cudaIpcMemHandle_t hp, ha;
    CU(cudaIpcGetMemHandle(&hp, h->x_poses)); CU(cudaIpcGetMemHandle(&ha, h->x_attrs));
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "CUDA IPC handle size");
    memcpy(handles_out_128, &hp, 64); memcpy(static_cast<char*>(handles_out_128) + 64, &ha, 64);
    return B2_OK;
}
extern "C" int b2_pf_p2p_connect(b2_pf* h, const void* all_handles, uint32_t world, uint32_t rank, uint32_t n_per_rank)
{
    NOTNULL(h); NOTNULL(all_handles);
    if (world == 0 || world > B2_MAX_PEERS || rank >= world) return fail(B2_ERR_INVALID, "p2p: world %u / rank %u (at most %d ranks)", world, rank, B2_MAX_PEERS);
    if (!h->x_poses || n_per_rank > h->x_cap) return fail(B2_ERR_INVALID, "p2p: connect before init");
    if (h->peers_open) return fail(B2_ERR_INVALID, "p2p: already connected");
    CU(cudaSetDevice(h->map->device));
    PfPeers P{}; P.world = world; P.rank = rank; P.n_per_rank = n_per_rank;
    for (uint32_t r = 0; r < world; r++) {
        if (r == rank) { P.poses[r] = h->x_poses; P.attrs[r] = h->x_attrs; continue; }
        cudaIpcMemHandle_t hp, ha;
        memcpy(&hp, static_cast<const char*>(all_handles) + 128 * (size_t)r, 64); memcpy(&ha, static_cast<const char*>(all_handles) + 128 * (size_t)r + 64, 64);
        void *pp = nullptr, *pa = nullptr;
        cudaError_t e = cudaIpcOpenMemHandle(&pp, hp, cudaIpcMemLazyEnablePeerAccess);
        if (e == cudaSuccess) e = cudaIpcOpenMemHandle(&pa, ha, cudaIpcMemLazyEnablePeerAccess);
        if (e != cudaSuccess) {
            (void)cudaGetLastError();
            for (uint32_t q = 0; q < r; q++) if (q != rank) { cudaIpcCloseMemHandle((void*)P.poses[q]); cudaIpcCloseMemHandle((void*)P.attrs[q]); }
            if (pp) cudaIpcCloseMemHandle(pp);
            return fail(B2_ERR_CUDA, "p2p: cannot map the particle buffers of rank %u (%s): no peer access between the GPUs or CUDA IPC unavailable", r, cudaGetErrorString(e));
        }
        P.poses[r] = (const b2_transform*)pp; P.attrs[r] = (const b2_particle_attr*)pa;
    }
    h->peers = P; h->peers_open = true;
    return B2_OK;
}
extern "C" int b2_pf_p2p_publish(b2_pf* h, const b2_transform* poses_dev, const b2_particle_attr* attrs_dev, uint32_t n_local)
{
    NOTNULL(h); NOTNULL(poses_dev); NOTNULL(attrs_dev);
    if (!h->peers_open || n_local != h->peers.n_per_rank) return fail(B2_ERR_INVALID, "p2p: publish needs a connected handle and exactly n_per_rank particles");
    CU(cudaSetDevice(h->map->device));
    CU(cudaMemcpyAsync(h->x_poses, poses_dev, sizeof(b2_transform) * (size_t)n_local, cudaMemcpyDeviceToDevice, h->stream));
    CU(cudaMemcpyAsync(h->x_attrs, attrs_dev, sizeof(b2_particle_attr) * (size_t)n_local, cudaMemcpyDeviceToDevice, h->stream));
    CU(cudaStreamSynchronize(h->stream));            // the caller's cross-rank barrier follows: peers may read as soon as it is passed
    return B2_OK;
}
extern "C" int b2_pf_resample_gladiator_p2p(b2_pf* h, b2_transform* poses_new_dev, b2_particle_attr* attrs_new_dev, const b2_gladiator_config* cfg, uint64_t seed, uint32_t step,
                                            uint64_t* remote_bytes_out)
{
    NOTNULL(h); NOTNULL(cfg); NOTNULL(poses_new_dev); NOTNULL(attrs_new_dev);
    if (!h->peers_open && h->peers.pad != 1u) return fail(B2_ERR_INVALID, "p2p: resample before connect");
    CU(cudaSetDevice(h->map->device));
    unsigned long long* traffic = &h->d_recs.p->traffic;
    CU(cudaMemsetAsync(traffic, 0, sizeof(unsigned long long), h->stream));
    k_pf_gladiator_p2p<<<(h->peers.n_per_rank + 255) / 256, 256, 0, h->stream>>>(h->peers, poses_new_dev, attrs_new_dev, *cfg, seed, step, traffic);
    LAUNCHED();
    if (remote_bytes_out) {
        RES(pf_fetch(h, h->h_recs->traffic));
        *remote_bytes_out = h->h_recs->traffic;
    }
    return B2_OK;
}
// test hook: a "world" of several shards on ONE device (the peers are plain device buffers of this process), so that the indexing of the
// p2p kernel can be checked on a single GPU; poses_all / attrs_all hold world * n_per_rank particles, this handle plays `rank`
extern "C" int b2_pf_p2p_connect_local(b2_pf* h, const b2_transform* poses_all_dev, const b2_particle_attr* attrs_all_dev, uint32_t world, uint32_t rank, uint32_t n_per_rank)
{
    NOTNULL(h); NOTNULL(poses_all_dev); NOTNULL(attrs_all_dev);
    if (world == 0 || world > B2_MAX_PEERS || rank >= world || n_per_rank == 0) return fail(B2_ERR_INVALID, "p2p: bad local world");
    if (h->peers_open) return fail(B2_ERR_INVALID, "p2p: already connected");
    CU(cudaSetDevice(h->map->device));
    PfPeers P{}; P.world = world; P.rank = rank; P.n_per_rank = n_per_rank;
    for (uint32_t r = 0; r < world; r++) { P.poses[r] = poses_all_dev + (size_t)r * n_per_rank; P.attrs[r] = attrs_all_dev + (size_t)r * n_per_rank; }
    h->peers = P;                 // peers_open stays false: nothing to unmap, and publish is not needed
    h->peers.pad = 1u;
    return B2_OK;
}

extern "C" int b2_pf_gladiator_randoms(b2_pf* h, uint64_t seed, uint32_t step, uint32_t first, uint32_t n, uint32_t* raw_dev, float* normals_dev)
{
    NOTNULL(h);
    if (n == 0) return B2_OK;
    NOTNULL(raw_dev); NOTNULL(normals_dev);
    CU(cudaSetDevice(h->map->device));
    k_pf_gladiator_randoms<<<(n + 255) / 256, 256, 0, h->stream>>>(seed, step, first, n, raw_dev, normals_dev);
    LAUNCHED();
    return B2_OK;
}

// ---- particle set initialisation ------------------------------------------------------------------------------------------------------------
static int pf_init_range(uint32_t first, uint32_t n)
{
    if ((uint64_t)first + n > (1ull << 32)) return fail(B2_ERR_INVALID, "particle range %u+%u exceeds 2^32 global indices", first, n);
    return B2_OK;
}

// the box of the uniform initialiser and of the recovery's candidates, narrowed to float and checked (`what` names the caller)
static int pf_box_check(const double* bb_min, const double* bb_max, const char* what, PfInitBox* box)
{
    static const char* dim[6] = {"x", "y", "z", "roll", "pitch", "yaw"};
    for (int k = 0; k < 6; k++) {
        box->lo[k] = (float)bb_min[k]; box->hi[k] = (float)bb_max[k];         // uniform_real_distribution<float> of the double parameters
        if (!std::isfinite(box->lo[k]) || !std::isfinite(box->hi[k]))
            return fail(B2_ERR_INVALID, "%s: %s bounds [%g, %g] are not finite in float", what, dim[k], bb_min[k], bb_max[k]);
        if (box->lo[k] > box->hi[k]) return fail(B2_ERR_INVALID, "%s: %s bounds [%g, %g] have min > max", what, dim[k], bb_min[k], bb_max[k]);
        if (!std::isfinite(box->hi[k] - box->lo[k])) return fail(B2_ERR_INVALID, "%s: the %s extent %g overflows float", what, dim[k], bb_max[k] - bb_min[k]);
    }
    return B2_OK;
}

extern "C" int b2_pf_init_uniform(b2_pf* h, b2_transform* poses_dev, b2_particle_attr* attrs_dev, uint32_t first, uint32_t n, const double* bb_min, const double* bb_max,
                                  uint64_t seed)
{
    NOTNULL(h); NOTNULL(bb_min); NOTNULL(bb_max);
    PfInitBox box;
    RES(pf_box_check(bb_min, bb_max, "init uniform", &box));
    RES(pf_init_range(first, n));
    if (n == 0) return B2_OK;
    NOTNULL(poses_dev); NOTNULL(attrs_dev);
    CU(cudaSetDevice(h->map->device));
    k_pf_init_uniform<<<(n + 255) / 256, 256, 0, h->stream>>>(poses_dev, attrs_dev, first, n, box, seed);
    LAUNCHED();
    return B2_OK;
}

// rm::chol (Cholesky-Banachiewicz in float, sums over k in order) of the covariance narrowed to float (convert, rmcl_localization.cpp:154-163),
// lower triangle only.  A zero pivot whose column numerators are all exactly zero gives a zero column (a component without noise, as in rviz's
// /initialpose and any 2-D robot's covariance) where the reference divides 0 by 0 (SURVEY quirk D14); any other non-positive pivot is refused.
static int pf_chol6(const double* cov, float L[36])
{
    float A[36];
    for (int i = 0; i < 36; i++) { A[i] = (float)cov[i]; L[i] = 0.0f; }
    for (int i = 0; i < 6; i++)
        for (int j = 0; j <= i; j++)
            if (!std::isfinite(A[6 * i + j])) return fail(B2_ERR_INVALID, "init gaussian: covariance entry (%d,%d) = %g is not finite in float", i, j, cov[6 * i + j]);
    for (int i = 0; i < 6; i++)                                                    // row by row; column j's pivot is row j's diagonal
        for (int j = 0; j <= i; j++) {
            float s = 0.0f;
            for (int k = 0; k < j; k++) s += L[6 * i + k] * L[6 * j + k];
            const float num = A[6 * i + j] - s;
            if (i == j) {
                if (!(num >= 0.0f) || !std::isfinite(num))
                    return fail(B2_ERR_INVALID, "init gaussian: covariance is not positive semi-definite at column %d (pivot %g)", j, (double)num);
                L[6 * i + i] = std::sqrt(num);
            } else if (L[6 * j + j] == 0.0f) {
                if (num != 0.0f) return fail(B2_ERR_INVALID, "init gaussian: column %d has zero variance but a non-zero covariance at (%d,%d)", j, i, j);
                // zero column: no noise on this component
            } else {
                L[6 * i + j] = num / L[6 * j + j];
                if (!std::isfinite(L[6 * i + j])) return fail(B2_ERR_INVALID, "init gaussian: Cholesky factor (%d,%d) of column %d overflows float", i, j, j);
            }
        }
    return B2_OK;
}

extern "C" int b2_pf_init_gaussian(b2_pf* h, b2_transform* poses_dev, b2_particle_attr* attrs_dev, uint32_t first, uint32_t n, const b2_transform* pose,
                                   const double* cov_rowmajor, uint64_t seed)
{
    NOTNULL(h); NOTNULL(pose); NOTNULL(cov_rowmajor);
    PfInitGauss g;
    RES(pf_chol6(cov_rowmajor, g.L));
    g.Tlm = *pose;                                                                 // Tpm = Identity (:222-225), so Tlm = Tlp
    RES(pf_init_range(first, n));
    if (n == 0) return B2_OK;
    NOTNULL(poses_dev); NOTNULL(attrs_dev);
    CU(cudaSetDevice(h->map->device));
    k_pf_init_gaussian<<<(n + 255) / 256, 256, 0, h->stream>>>(poses_dev, attrs_dev, first, n, g, seed);
    LAUNCHED();
    return B2_OK;
}

// ---- recovery from a kidnapping (Augmented MCL; SURVEY appendix J) ---------------------------------------------------------------------------
extern "C" int b2_pf_recovery_reset(b2_pf* h)
{
    NOTNULL(h);
    CU(cudaSetDevice(h->map->device));
    CU(cudaMemsetAsync(&h->d_recs.p->rec, 0, sizeof(b2_recovery_state), h->stream));
    return B2_OK;
}

extern "C" int b2_pf_recovery_observe(b2_pf* h, const b2_particle_attr* attrs_dev, uint32_t n, const b2_recovery_config* cfg, b2_recovery_state* state_host)
{
    NOTNULL(h); NOTNULL(attrs_dev); NOTNULL(cfg);
    if (n == 0) return fail(B2_ERR_INVALID, "recovery observe: no particles (n = 0)");
    const double as = cfg->alpha_slow, af = cfg->alpha_fast;
    if (!(std::isfinite(as) && as >= 0.0 && as <= 1.0) || !(std::isfinite(af) && af >= 0.0 && af <= 1.0))
        return fail(B2_ERR_INVALID, "recovery observe: alpha_slow = %g and alpha_fast = %g must lie in [0, 1]", as, af);
    if (as > af) return fail(B2_ERR_INVALID, "recovery observe: alpha_slow = %g > alpha_fast = %g", as, af);
    CU(cudaSetDevice(h->map->device));
    RES(pf_weight_stats(h, attrs_dev, n, false));
    k_pf_recovery_filter<<<1, 1, 0, h->stream>>>(&h->d_recs.p->res.S, n, as, af, &h->d_recs.p->rec);
    LAUNCHED();
    if (state_host) {
        RES(pf_fetch(h, h->h_recs->rec));
        *state_host = h->h_recs->rec;
    }
    return B2_OK;
}

extern "C" int b2_pf_recovery_inject(b2_pf* h, b2_transform* poses_dev, b2_particle_attr* attrs_dev, uint32_t first, uint32_t n_local, const double* bb_min,
                                     const double* bb_max, const b2_surface_config* surface, uint32_t max_tries, uint64_t seed, uint32_t step,
                                     b2_recovery_result* out_host)
{
    NOTNULL(h); NOTNULL(bb_min); NOTNULL(bb_max);
    PfInitBox box;
    RES(pf_box_check(bb_min, bb_max, "recovery inject", &box));
    b2_surface_config sc{};
    float cos_max = 0.0f, tfar = 0.0f;
    if (surface) { sc = *surface; RES(surface_config_check(sc, "recovery inject", &cos_max, &tfar)); }
    if (max_tries < 1 || max_tries > B2_RECOVERY_MAX_TRIES) return fail(B2_ERR_INVALID, "recovery inject: max_tries = %u outside [1, %u]", max_tries, B2_RECOVERY_MAX_TRIES);
    if (n_local > 0) { NOTNULL(poses_dev); NOTNULL(attrs_dev); }
    RES(pf_init_range(first, n_local));
    CU(cudaSetDevice(h->map->device));
    if (n_local == 0) {
        if (out_host) {                                   // nothing to replace: the p a slice would have used
            RES(pf_fetch(h, h->h_recs->rec.p_inject));
            *out_host = b2_recovery_result{h->h_recs->rec.p_inject, 0, 0};
        }
        return B2_OK;
    }
    b2_recovery_state* rec = &h->d_recs.p->rec;
    b2_recovery_result* res = out_host ? &h->d_recs.p->rec_res : nullptr;
    if (res) CU(cudaMemsetAsync(res, 0, sizeof(b2_recovery_result), h->stream));
    const uint32_t grid = (n_local + 127) / 128;
    if (surface) k_pf_recovery_inject<true><<<grid, 128, 0, h->stream>>>(h->map->view(), poses_dev, attrs_dev, first, n_local, box, sc, cos_max, tfar, max_tries, seed, step, rec, res);
    else         k_pf_recovery_inject<false><<<grid, 128, 0, h->stream>>>(h->map->view(), poses_dev, attrs_dev, first, n_local, box, sc, cos_max, tfar, max_tries, seed, step, rec, res);
    LAUNCHED();
    k_pf_recovery_clear<<<1, 1, 0, h->stream>>>(rec);
    LAUNCHED();
    if (out_host) {
        RES(pf_fetch(h, h->h_recs->rec_res));
        *out_host = h->h_recs->rec_res;
    }
    return B2_OK;
}

extern "C" int b2_pf_likelihood_stats(b2_pf* h, const b2_particle_attr* attrs_dev, uint32_t n, float* sum_out, float* max_out)
{
    NOTNULL(h);
    CU(cudaSetDevice(h->map->device));
    float s = 0.f, m = 0.f;
    if (n > 0) {
        NOTNULL(attrs_dev);
        RES(pf_weight_stats(h, attrs_dev, n, true));
        s = (float)h->h_recs->res.S; m = (float)h->h_recs->res.L_max;
    }
    if (sum_out) *sum_out = s;
    if (max_out) *max_out = m;
    return B2_OK;
}

// RmclNode::estimateStats (rmcl_localization.cpp:642-731): two read passes, Tbm handed from the first to the second in device memory
// both passes over n > 0 particles; the record is left in h->d_recs.p->est.rec
static int estimate_launch(b2_pf* h, const b2_transform* poses_dev, const b2_particle_attr* attrs_dev, uint32_t n)
{
    const uint32_t grid = pf_stats_grid(h, n);
    k_pf_estimate_moments<<<grid, 256, 0, h->stream>>>(poses_dev, attrs_dev, n, h->d_part.p, &h->d_recs.p->est);
    LAUNCHED();
    k_pf_estimate_cov<<<grid, 256, 0, h->stream>>>(poses_dev, attrs_dev, n, h->d_part.p, &h->d_recs.p->est);
    LAUNCHED();
    return B2_OK;
}
extern "C" int b2_pf_estimate_stats(b2_pf* h, const b2_transform* poses_dev, const b2_particle_attr* attrs_dev, uint32_t n, b2_particle_stats* out_host)
{
    NOTNULL(h); NOTNULL(poses_dev); NOTNULL(attrs_dev); NOTNULL(out_host);
    if (n == 0) return fail(B2_ERR_INVALID, "estimate stats: no particles (n = 0)");
    CU(cudaSetDevice(h->map->device));
    RES(estimate_launch(h, poses_dev, attrs_dev, n));
    RES(pf_fetch(h, h->h_recs->est.rec));
    *out_host = h->h_recs->est.rec;
    return B2_OK;
}

// the resamplers' outputs: slots first .. first + n_local - 1 of n_out, in ranges that overlap neither an input nor each other
static bool ranges_overlap(const void* a, size_t a_bytes, const void* b, size_t b_bytes)
{
    const uintptr_t pa = (uintptr_t)a, pb = (uintptr_t)b;
    return a_bytes && b_bytes && pa < pb + b_bytes && pb < pa + a_bytes;
}
static int check_resample_outputs(const char* what, const b2_transform* poses_dev, const b2_particle_attr* attrs_dev, uint32_t n, uint32_t n_out, uint32_t first,
                                  uint32_t n_local, const b2_transform* poses_new_dev, const b2_particle_attr* attrs_new_dev)
{
    if ((uint64_t)first + n_local > n_out) return fail(B2_ERR_INVALID, "%s: slots %u+%u exceed the %u output slots", what, first, n_local, n_out);
    const size_t in_p = sizeof(b2_transform) * (size_t)n, in_a = sizeof(b2_particle_attr) * (size_t)n;
    const size_t out_p = sizeof(b2_transform) * (size_t)n_local, out_a = sizeof(b2_particle_attr) * (size_t)n_local;
    if (ranges_overlap(poses_new_dev, out_p, poses_dev, in_p) || ranges_overlap(poses_new_dev, out_p, attrs_dev, in_a) ||
        ranges_overlap(attrs_new_dev, out_a, poses_dev, in_p) || ranges_overlap(attrs_new_dev, out_a, attrs_dev, in_a) ||
        ranges_overlap(poses_new_dev, out_p, attrs_new_dev, out_a))
        return fail(B2_ERR_INVALID, "%s: an output range overlaps an input range or the other output (the node double-buffers)", what);
    return B2_OK;
}

// ResidualResamplerCPU::update (ResidualResamplerCPU.cpp:55-202): a statistics pass, then the draws in chunks of doubling size, each counted,
// scanned and searched for the draw that fills the last slot, with one read-back per chunk; the slots a chunk filled are built right after it
extern "C" int b2_pf_resample_residual(b2_pf* h, const b2_transform* poses_dev, const b2_particle_attr* attrs_dev, uint32_t n, uint32_t n_new,
                                       uint32_t first, uint32_t n_local, b2_transform* poses_new_dev, b2_particle_attr* attrs_new_dev,
                                       const b2_gladiator_config* cfg, uint64_t seed, uint32_t step, b2_residual_result* out_host)
{
    NOTNULL(h); NOTNULL(poses_dev); NOTNULL(attrs_dev); NOTNULL(poses_new_dev); NOTNULL(attrs_new_dev); NOTNULL(cfg); NOTNULL(out_host);
    if (n == 0 || n_new == 0) return fail(B2_ERR_INVALID, "resample residual: %u particles into %u slots (both must be > 0)", n, n_new);
    RES(check_resample_outputs("resample residual", poses_dev, attrs_dev, n, n_new, first, n_local, poses_new_dev, attrs_new_dev));
    CU(cudaSetDevice(h->map->device));
    const uint64_t M = n_new, nm = std::max<uint64_t>(n, M), d_max = 16 * nm;
    // draws are keyed by their index: the chunk size changes no result.  2^30 keeps a chunk within the scan's int item count.
    const uint64_t cap = std::min<uint64_t>(2 * nm, 1ull << 30);
    uint64_t chunk = std::min<uint64_t>(std::max<uint64_t>(2 * (uint64_t)n, 1ull << 16), cap);
    bool usable = false;
    RES(pf_weight_stats(h, attrs_dev, n, true, &usable));
    const double S = h->h_recs->res.S, L_max = h->h_recs->res.L_max;
    b2_residual_result res = {0, 0, S, L_max};
    if (!usable) { *out_host = res; return B2_OK; }
    size_t tmp_bytes = 0;
    CU(cub::DeviceScan::InclusiveSum(nullptr, tmp_bytes, h->d_res_counts.p, h->d_res_prefix.p, (int)cap, h->stream));
    RES(h->d_res_parents.reserve(cap)); RES(h->d_res_counts.reserve(cap)); RES(h->d_res_prefix.reserve(cap)); RES(h->d_res_tmp.reserve(std::max<size_t>(tmp_bytes, 16)));
    uint64_t fill = 0, draws = 0;
    while (fill < M && draws < d_max) {
        const uint32_t len = (uint32_t)std::min<uint64_t>(chunk, d_max - draws);
        k_pf_residual_counts<<<(len + 255) / 256, 256, 0, h->stream>>>(attrs_dev, n, M, S, seed, step, draws, len, h->d_res_parents.p, h->d_res_counts.p);
        LAUNCHED();
        size_t bytes = h->d_res_tmp.cap;
        CU(cub::DeviceScan::InclusiveSum(h->d_res_tmp.p, bytes, h->d_res_counts.p, h->d_res_prefix.p, (int)len, h->stream));
        LAUNCHED();
        k_pf_residual_find<<<1, 1, 0, h->stream>>>(h->d_res_prefix.p, len, M - fill, &h->d_recs.p->res);
        LAUNCHED();
        RES(pf_fetch(h, h->h_recs->res));
        const uint64_t filled = h->h_recs->res.filled, used = h->h_recs->res.used;
        const uint64_t lo = std::max<uint64_t>(fill, first), hi = std::min<uint64_t>(fill + filled, (uint64_t)first + n_local);
        if (lo < hi) {
            const uint32_t n_k = (uint32_t)(hi - lo);
            k_pf_residual_expand<<<(n_k + 255) / 256, 256, 0, h->stream>>>(poses_dev, attrs_dev, h->d_res_parents.p, h->d_res_prefix.p, len, fill, (uint32_t)lo, n_k, first,
                                                                          L_max, *cfg, seed, step, poses_new_dev, attrs_new_dev);
            LAUNCHED();
        }
        fill += filled; draws += used;
        chunk = std::min(2 * chunk, cap);
    }
    CU(cudaStreamSynchronize(h->stream));
    res.n_particles = fill; res.draws = draws;
    *out_host = res;
    return B2_OK;
}

// K = ceil(2 pi / res_yaw) of the ratio shrunk by 2^-20: a float res_yaw is 2 pi / K rounded (10 deg in float is a hair under 10 deg), and
// a plain ceil would then give K + 1 sectors; with the shrink every float within 2^-21 of 2 pi / K gives K (SURVEY G3)
static const double kKldPi = 3.14159265358979323846;
static double kld_sector_count(float res_yaw) { return std::ceil(2.0 * kKldPi / (double)res_yaw * (1.0 - 0x1p-20)); }
// the handle's table of the K sector boundaries theta_k = -pi + 2 pi k / K, as (float)cos, (float)sin of the double angle
static int kld_sector_table(b2_pf* h, uint32_t K)
{
    if (h->kld_K == K) return B2_OK;
    h->h_kld_tab.resize(2 * (size_t)K);
    for (uint32_t k = 0; k < K; k++) {
        const double th = -kKldPi + 2.0 * kKldPi * (double)k / (double)K;
        h->h_kld_tab[2 * k] = (float)std::cos(th); h->h_kld_tab[2 * k + 1] = (float)std::sin(th);
    }
    RES(h->d_kld_tab.reserve(2 * (size_t)K));
    CU(cudaMemcpyAsync(h->d_kld_tab.p, h->h_kld_tab.data(), sizeof(float) * 2 * K, cudaMemcpyHostToDevice, h->stream));
    h->kld_K = K;
    return B2_OK;
}
// KLD-sampling (Fox 2003; rmcl/docs/RMCL.md:80-83): the weight statistics, the integer weights and their scan, then the draws in chunks of
// doubling size, each drawn into the hash set, flagged, scanned and searched for the first draw that meets the stop rule, with one read-back
// per chunk; the slots a chunk filled are built right after it
extern "C" int b2_pf_resample_kld(b2_pf* h, const b2_transform* poses_dev, const b2_particle_attr* attrs_dev, uint32_t n, uint32_t n_max, uint32_t first,
                                  uint32_t n_local, b2_transform* poses_new_dev, b2_particle_attr* attrs_new_dev, const b2_gladiator_config* cfg,
                                  const b2_kld_config* kld, uint64_t seed, uint32_t step, b2_kld_result* out_host)
{
    NOTNULL(h); NOTNULL(poses_dev); NOTNULL(attrs_dev); NOTNULL(poses_new_dev); NOTNULL(attrs_new_dev); NOTNULL(cfg); NOTNULL(kld); NOTNULL(out_host);
    if (n == 0 || n_max == 0) return fail(B2_ERR_INVALID, "resample kld: %u particles into %u slots (both must be > 0)", n, n_max);
    if (kld->n_min == 0 || kld->n_min > n_max) return fail(B2_ERR_INVALID, "resample kld: n_min = %u must lie in [1, n_max = %u]", kld->n_min, n_max);
    RES(check_resample_outputs("resample kld", poses_dev, attrs_dev, n, n_max, first, n_local, poses_new_dev, attrs_new_dev));
    if (!(std::isfinite(kld->res_xy) && kld->res_xy > 0.0f) || !(std::isfinite(kld->epsilon) && kld->epsilon > 0.0))
        return fail(B2_ERR_INVALID, "resample kld: res_xy = %g and epsilon = %g must be finite and > 0", (double)kld->res_xy, kld->epsilon);
    if (!(std::isfinite(kld->res_z) && kld->res_z >= 0.0f)) return fail(B2_ERR_INVALID, "resample kld: res_z = %g must be finite and >= 0", (double)kld->res_z);
    if (!std::isfinite(kld->z)) return fail(B2_ERR_INVALID, "resample kld: z = %g must be finite", kld->z);
    const double Kd = kld_sector_count(kld->res_yaw);
    if (!(Kd >= 1.0 && Kd <= (double)B2_KLD_MAX_SECTORS))
        return fail(B2_ERR_INVALID, "resample kld: res_yaw = %g gives %g yaw sectors (1 .. %u)", (double)kld->res_yaw, Kd, B2_KLD_MAX_SECTORS);
    const uint32_t K = (uint32_t)Kd;
    CU(cudaSetDevice(h->map->device));
    bool usable = false;
    RES(pf_weight_stats(h, attrs_dev, n, true, &usable));
    const double S = h->h_recs->res.S, L_max = h->h_recs->res.L_max;
    b2_kld_result res = {0, 0, S, L_max};
    if (!usable) { *out_host = res; return B2_OK; }
    // the chunk schedule: sizes double from max(n_min, 2^16) up to n_max draws in all; 2^30 keeps a chunk within the scan's int item count
    const uint64_t c0 = std::min<uint64_t>(std::max<uint64_t>(kld->n_min, 1ull << 16), n_max);
    uint64_t max_len = 0;
    for (uint64_t c = c0, d = 0; d < n_max; d += std::min<uint64_t>(c, n_max - d), c = std::min<uint64_t>(2 * c, 1ull << 30))
        max_len = std::max<uint64_t>(max_len, std::min<uint64_t>(c, n_max - d));
    uint64_t T = 1;                                      // the hash set: a power of two >= 2 n_max slots (load <= 1/2)
    while (T < 2 * (uint64_t)n_max) T <<= 1;
    size_t scan_w = 0, scan_f = 0;
    CU(cub::DeviceScan::InclusiveSum(nullptr, scan_w, h->d_kld_w.p, h->d_kld_W.p, (int)n, h->stream));
    CU(cub::DeviceScan::InclusiveSum(nullptr, scan_f, h->d_kld_flags.p, h->d_kld_cum.p, (int)max_len, h->stream));
    RES(h->d_kld_w.reserve(n)); RES(h->d_kld_W.reserve(n)); RES(h->d_kld_keys.reserve(T)); RES(h->d_kld_first.reserve(T));
    RES(h->d_kld_parents.reserve(max_len)); RES(h->d_kld_slots.reserve(max_len)); RES(h->d_kld_flags.reserve(max_len)); RES(h->d_kld_cum.reserve(max_len));
    RES(h->d_kld_tmp.reserve(std::max<size_t>(std::max(scan_w, scan_f), 16)));
    RES(kld_sector_table(h, K));
    // the hash set is cleared by memset on the stream: at 12 B per slot it costs less than one chunk's draws, and unlike epoch tags it keeps
    // every stored key a plain 64-bit word that one atomicCAS claims
    CU(cudaMemsetAsync(h->d_kld_keys.p, 0, sizeof(unsigned long long) * T, h->stream));
    CU(cudaMemsetAsync(h->d_kld_first.p, 0xff, sizeof(unsigned int) * T, h->stream));
    k_pf_kld_weights<<<(n + 255) / 256, 256, 0, h->stream>>>(attrs_dev, n, L_max, h->d_kld_w.p);
    LAUNCHED();
    size_t bytes = h->d_kld_tmp.cap;
    CU(cub::DeviceScan::InclusiveSum(h->d_kld_tmp.p, bytes, h->d_kld_w.p, h->d_kld_W.p, (int)n, h->stream));
    LAUNCHED();
    const KldBins bins{kld->res_xy, kld->res_z, K, h->d_kld_tab.p};
    uint64_t d0 = 0, n_bins = 0, chunk = c0;
    PfKldState* st = &h->d_recs.p->kld;
    bool done = false;
    while (!done && d0 < n_max) {
        const uint32_t len = (uint32_t)std::min<uint64_t>(chunk, n_max - d0), grid = (len + 255) / 256;
        k_pf_kld_draw<<<grid, 256, 0, h->stream>>>(h->d_kld_W.p, n, poses_dev, bins, seed, step, d0, len, h->d_kld_keys.p, h->d_kld_first.p, T - 1,
                                                   h->d_kld_parents.p, h->d_kld_slots.p, st);
        LAUNCHED();
        k_pf_kld_flags<<<grid, 256, 0, h->stream>>>(h->d_kld_first.p, h->d_kld_slots.p, d0, len, h->d_kld_flags.p);
        LAUNCHED();
        bytes = h->d_kld_tmp.cap;
        CU(cub::DeviceScan::InclusiveSum(h->d_kld_tmp.p, bytes, h->d_kld_flags.p, h->d_kld_cum.p, (int)len, h->stream));
        LAUNCHED();
        k_pf_kld_stop<<<grid, 256, 0, h->stream>>>(h->d_kld_cum.p, d0, len, n_bins, kld->n_min, n_max, kld->epsilon, kld->z, st);
        LAUNCHED();
        RES(pf_fetch(h, h->h_recs->kld));
        const unsigned long long stop = h->h_recs->kld.stop;
        done = stop != ~0ull;
        const uint64_t used = done ? (stop >> 32) + 1 : len, chunk_bins = done ? (stop & 0xffffffffull) : h->h_recs->kld.bins;
        const uint64_t lo = std::max<uint64_t>(d0, first), hi = std::min<uint64_t>(d0 + used, (uint64_t)first + n_local);
        if (lo < hi) {
            const uint32_t n_k = (uint32_t)(hi - lo);
            k_pf_kld_expand<<<(n_k + 255) / 256, 256, 0, h->stream>>>(poses_dev, attrs_dev, h->d_kld_parents.p, d0, (uint32_t)lo, n_k, first, L_max, *cfg, seed, step,
                                                                      poses_new_dev, attrs_new_dev);
            LAUNCHED();
        }
        d0 += used; n_bins += chunk_bins;
        chunk = std::min<uint64_t>(2 * chunk, 1ull << 30);
    }
    CU(cudaStreamSynchronize(h->stream));
    res.n_particles = d0; res.bins = n_bins;
    *out_host = res;
    return B2_OK;
}

// The filter's pose hypotheses (SURVEY appendix H): the statistics pass, the members' bins into the hash set, the union-find labelling, the
// ranking of the clusters, every particle's label, a stable sort that lines the recorded clusters' members up, and the two estimate passes
// on each of them
extern "C" int b2_pf_cluster_stats(b2_pf* h, const b2_transform* poses_dev, const b2_particle_attr* attrs_dev, uint32_t n, const b2_cluster_config* cfg,
                                   b2_cluster_record* records_host, uint32_t* labels_dev, b2_cluster_result* out_host)
{
    NOTNULL(h); NOTNULL(poses_dev); NOTNULL(attrs_dev); NOTNULL(cfg); NOTNULL(records_host); NOTNULL(out_host);
    if (n == 0 || n > (1u << 30)) return fail(B2_ERR_INVALID, "cluster stats: %u particles (1 .. 2^30)", n);
    if (!(std::isfinite(cfg->res_xy) && cfg->res_xy > 0.0f)) return fail(B2_ERR_INVALID, "cluster stats: res_xy = %g must be finite and > 0", (double)cfg->res_xy);
    if (!(std::isfinite(cfg->res_z) && cfg->res_z >= 0.0f)) return fail(B2_ERR_INVALID, "cluster stats: res_z = %g must be finite and >= 0", (double)cfg->res_z);
    const double Kd = kld_sector_count(cfg->res_yaw);
    if (!(Kd >= 1.0 && Kd <= (double)B2_KLD_MAX_SECTORS))
        return fail(B2_ERR_INVALID, "cluster stats: res_yaw = %g gives %g yaw sectors (1 .. %u)", (double)cfg->res_yaw, Kd, B2_KLD_MAX_SECTORS);
    if (cfg->max_records < 1 || cfg->max_records > B2_CLUSTER_MAX_RECORDS)
        return fail(B2_ERR_INVALID, "cluster stats: max_records = %u must lie in [1, %u]", cfg->max_records, B2_CLUSTER_MAX_RECORDS);
    const uint32_t K = (uint32_t)Kd;
    CU(cudaSetDevice(h->map->device));
    bool usable = false;
    RES(pf_weight_stats(h, attrs_dev, n, true, &usable));
    const double S = h->h_recs->res.S, L_max = h->h_recs->res.L_max;
    b2_cluster_result res = {0, 0, 0, 0, 0, 0, S, L_max};
    if (!usable) { *out_host = res; return B2_OK; }       // as KLD (SURVEY G1)
    uint64_t T = 1;                                      // the hash set: a power of two >= 2 n slots (load <= 1/2)
    while (T < 2 * (uint64_t)n) T <<= 1;
    size_t sort_c = 0, sort_p = 0;
    CU(cub::DeviceRadixSort::SortPairs(nullptr, sort_c, h->d_kld_w.p, h->d_kld_W.p, h->d_cl_idx.p, h->d_cl_idx2.p, (int)n, 0, 64, h->stream));
    CU(cub::DeviceRadixSort::SortPairs(nullptr, sort_p, h->d_cl_key.p, h->d_cl_key2.p, h->d_cl_idx.p, h->d_cl_idx2.p, (int)n, 0, 5, h->stream));
    RES(h->d_kld_keys.reserve(T)); RES(h->d_kld_first.reserve(T)); RES(h->d_cl_w.reserve(T)); RES(h->d_cl_cnt.reserve(T)); RES(h->d_cl_aux.reserve(T));
    RES(h->d_kld_w.reserve(n)); RES(h->d_kld_W.reserve(n)); RES(h->d_cl_slot.reserve(n)); RES(h->d_cl_key.reserve(n)); RES(h->d_cl_key2.reserve(n));
    RES(h->d_cl_idx.reserve(n)); RES(h->d_cl_idx2.reserve(n)); RES(h->d_kld_tmp.reserve(std::max<size_t>(std::max(sort_c, sort_p), 16)));
    PfRecords* d = h->d_recs.p;
    const PfRecords& hr = *h->h_recs;
    RES(kld_sector_table(h, K));
    CU(cudaMemsetAsync(h->d_kld_keys.p, 0, sizeof(unsigned long long) * T, h->stream));
    CU(cudaMemsetAsync(h->d_cl_w.p, 0, sizeof(unsigned long long) * T, h->stream));
    CU(cudaMemsetAsync(h->d_cl_cnt.p, 0, sizeof(unsigned int) * T, h->stream));
    CU(cudaMemsetAsync(&d->cl, 0, sizeof(PfClusterState), h->stream));
    const KldBins bins{cfg->res_xy, cfg->res_z, K, h->d_kld_tab.p};
    const uint32_t grid_n = (n + 255) / 256, grid_T = (uint32_t)((T + 255) / 256);
    k_pf_cluster_insert<<<grid_n, 256, 0, h->stream>>>(poses_dev, attrs_dev, n, L_max, bins, h->d_kld_keys.p, T - 1, h->d_kld_first.p, h->d_cl_w.p, h->d_cl_cnt.p,
                                                       h->d_cl_slot.p, &d->cl);
    LAUNCHED();
    // A round joins every pair of touching bins and ends in the fixed point unless one of its bounded loops ran out, which the bounds (the
    // table's size, above any path or retry count) do not allow; the cap keeps the call finite even so.
    uint32_t rounds = 0;
    for (;;) {
        if (rounds == B2_CLUSTER_MAX_ROUNDS) return fail(B2_ERR_CUDA, "cluster stats: the labelling did not settle within %u rounds", B2_CLUSTER_MAX_ROUNDS);
        rounds++;
        CU(cudaMemsetAsync(&d->cl.retry, 0, sizeof(unsigned int), h->stream));
        k_pf_cluster_hook<<<grid_T, 256, 0, h->stream>>>(h->d_kld_keys.p, T - 1, K, cfg->res_z > 0.0f ? 1 : 0, h->d_kld_first.p, h->d_cl_aux.p, &d->cl);
        LAUNCHED();
        k_pf_cluster_flatten<<<grid_T, 256, 0, h->stream>>>(h->d_kld_keys.p, T - 1, h->d_kld_first.p, h->d_cl_w.p, h->d_cl_cnt.p, h->d_cl_aux.p, h->d_cl_idx.p,
                                                            h->d_kld_w.p, &d->cl);
        LAUNCHED();
        RES(pf_fetch(h, hr.cl));
        if (hr.cl.fault) return fail(B2_ERR_CUDA, "cluster stats: the hash set of %llu slots had no room for %u particles", (unsigned long long)T, n);
        if (!hr.cl.retry) break;
    }
    const uint32_t m = hr.cl.n_clusters, n_records = std::min<uint32_t>(m, cfg->max_records);
    res.n_clusters = m; res.n_records = n_records; res.bins = hr.cl.bins; res.n_clustered = hr.cl.n_clustered; res.weight_total = hr.cl.weight_total; res.rounds = rounds;
    if (m == 0) {                                        // weights > 0, but no finite pose among them
        if (labels_dev) CU(cudaMemsetAsync(labels_dev, 0xff, sizeof(uint32_t) * (size_t)n, h->stream));
        CU(cudaStreamSynchronize(h->stream));
        *out_host = res;
        return B2_OK;
    }
    // rank: by key, then stably by the weight's complement; d_cl_idx lists the roots in rank order afterwards
    size_t bytes = h->d_kld_tmp.cap;
    if (m > 1) {
        CU(cub::DeviceRadixSort::SortPairs(h->d_kld_tmp.p, bytes, h->d_kld_w.p, h->d_kld_W.p, h->d_cl_idx.p, h->d_cl_idx2.p, (int)m, 0, 64, h->stream));
        LAUNCHED();
        k_pf_cluster_weight_keys<<<(m + 255) / 256, 256, 0, h->stream>>>(h->d_cl_idx2.p, h->d_cl_w.p, m, h->d_kld_w.p);
        LAUNCHED();
        bytes = h->d_kld_tmp.cap;
        CU(cub::DeviceRadixSort::SortPairs(h->d_kld_tmp.p, bytes, h->d_kld_w.p, h->d_kld_W.p, h->d_cl_idx2.p, h->d_cl_idx.p, (int)m, 0, 64, h->stream));
        LAUNCHED();
    }
    k_pf_cluster_rank<<<(m + 255) / 256, 256, 0, h->stream>>>(h->d_cl_idx.p, m, n_records, h->d_kld_keys.p, h->d_cl_w.p, h->d_cl_cnt.p, h->d_cl_aux.p, d->heads);
    LAUNCHED();
    k_pf_cluster_labels<<<grid_n, 256, 0, h->stream>>>(h->d_cl_slot.p, n, h->d_kld_first.p, h->d_cl_aux.p, n_records, labels_dev, h->d_cl_key.p, h->d_cl_idx.p);
    LAUNCHED();
    int bits = 1;                                        // sort keys 0 .. n_records
    while ((1u << bits) <= n_records) bits++;
    bytes = h->d_kld_tmp.cap;
    CU(cub::DeviceRadixSort::SortPairs(h->d_kld_tmp.p, bytes, h->d_cl_key.p, h->d_cl_key2.p, h->d_cl_idx.p, h->d_cl_idx2.p, (int)n, 0, bits, h->stream));
    LAUNCHED();
    RES(pf_fetch(h, hr.heads[0], n_records));
    uint64_t total = 0;
    for (uint32_t r = 0; r < n_records; r++) total += hr.heads[r].members;
    RES(h->d_cl_poses.reserve(total)); RES(h->d_cl_attrs.reserve(total));
    k_pf_cluster_gather<<<(uint32_t)((total + 255) / 256), 256, 0, h->stream>>>(h->d_cl_idx2.p, (uint32_t)total, poses_dev, attrs_dev, h->d_cl_poses.p, h->d_cl_attrs.p);
    LAUNCHED();
    uint64_t at = 0;
    for (uint32_t r = 0; r < n_records; r++) {
        RES(estimate_launch(h, h->d_cl_poses.p + at, h->d_cl_attrs.p + at, hr.heads[r].members));
        CU(cudaMemcpyAsync(&d->recs[r], &d->est.rec, sizeof(b2_particle_stats), cudaMemcpyDeviceToDevice, h->stream));
        at += hr.heads[r].members;
    }
    RES(pf_fetch(h, hr.recs[0], n_records));
    for (uint32_t r = 0; r < n_records; r++) {
        const PfClusterHead& hd = hr.heads[r];
        b2_cluster_record& o = records_host[r];
        memset(&o, 0, sizeof(o));
        o.stats = hr.recs[r];
        o.weight = (double)hd.weight_int / (double)res.weight_total;
        o.weight_int = hd.weight_int; o.bins = hd.bins; o.key = hd.key;
    }
    *out_host = res;
    return B2_OK;
}
