// api.cu -- C ABI (include/rmcl_b200.h) over the sm_90a kernels.  No CPU fallback anywhere: every entry point either runs
// the CUDA path or fails with B2_ERR_CUDA.
#include "kernels.cuh"
#include "lbvh.cuh"

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
        for (size_t i = 0; i < 3 * (size_t)nv; i++) if (!std::isfinite(verts[i])) return fail(B2_ERR_INVALID, "BVH build failed: non-finite vertex");
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
    if (!src_is_device) for (size_t i = 0; i < 3 * (size_t)nv; i++) if (!std::isfinite(verts[i])) return fail(B2_ERR_INVALID, "refit: non-finite vertex");
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

// ---- BVH blob: build once, ship to the other ranks / to disk (SURVEY.md 8b: b2_mesh_bvh_blob for broadcast) ---------------------------
struct B2BlobHeader {
    char     magic[8];                 // "B2BVH8F\0"
    uint32_t version, node_bytes, tri_bytes, n_nodes, n_tris, n_faces, n_verts, max_depth;
    int32_t  build_mode;
    float    abs_max[3], sah;
    uint32_t pad;                      // 64 bytes: the node array that follows stays 16-byte aligned inside an aligned buffer
};
static_assert(sizeof(B2BlobHeader) == 64, "blob header must be 64 bytes");
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
    DevBuf<uint32_t> d_tile_cost; DevBuf<uint16_t> d_tile_perm; uint32_t perm_tiles = 0, cost_tiles = 0;    // tile schedule of k_rcc_find: warp durations of the last launch (cost_tiles of them if it recorded any), order for the next (always a permutation of perm_tiles tiles)
    unsigned long long n_reruns = 0;                            // calls that were run again through the cooperative launch (exchange abort: co-residency or range)
    uint32_t loop_geom[2 + 4 * B2_MAX_SENSORS] = {};            // last fused call: sensors, grid, per sensor {n, blk0, nblk, smem_u} (b2_rcc_debug_loop_geometry)
    DevBuf<unsigned int> d_bar; unsigned int zc_seq = 0;        // [0] = "scan copy complete" flag (value: zc_seq of the call), [1] = abort word of the ICP loop
    DevBuf<unsigned long long> d_slots; unsigned int tag_base = 0; // exchange buffers of the ICP loop (icp_loop.cuh: accumulators, base, FP64 slots); round number of the next launch
    unsigned int seq = 0;               // sequence number of the last k_icp_loop launch (carried by every result chunk)
    std::deque<PendingCall> pending;    // enqueued, not yet collected (oldest first), at most B2_RING
    unsigned int slot_counter = 0;
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
    CU(cudaMemset(h->d_ticket.p, 0, sizeof(unsigned int)));
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
    h->d_partials.release(); h->d_ticket.release(); h->d_stats.release(); h->d_icp.release(); h->d_bar.release(); h->d_res.release(); h->d_dbg.release(); h->d_slots.release(); h->d_tile_cost.release(); h->d_tile_perm.release();
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
// make PROFILE=1 only: per block {ns at publish, ns at collect, cycles since the block reduce at publish, at collect} of iteration 1
extern "C" __attribute__((visibility("default"))) int b2_rcc_debug_blocks(b2_rcc* h, unsigned long long* out /* 4 * B2_ICP_MAX_GRID */)
{
    NOTNULL(h); NOTNULL(out);
    CU(cudaSetDevice(h->map->device));
    CU(cudaStreamSynchronize(h->stream));
    CU(cudaMemcpy(out, h->d_dbg.p + 16, 4 * B2_ICP_MAX_GRID * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
    return B2_OK;
}

// profiling aid (not part of the public header): per-warp {start, end} %globaltimer stamps of the NEXT k_rcc_find launches.
// buf_dev: device buffer of 2 x ceil(n_rays / 32) u64, or nullptr to switch the stamps off again.
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
    if (n == 0) { h->has_model = true; h->n = 0; h->width = w; h->height = hgt; return B2_OK; }   // zero-size model: find() silently returns (RCCOptix.cpp:30-34)
    if (n > 0xffffffffu / 4) return fail(B2_ERR_INVALID, "model too large");
    RES(h->d_dirs.reserve(3 * n)); RES(h->d_origs.reserve(3 * (size_t)n_origs));
    CU(cudaStreamSynchronize(h->stream));
    CU(cudaMemcpy(h->d_dirs.p, dirs, sizeof(float) * 3 * n, cudaMemcpyHostToDevice));
    CU(cudaMemcpy(h->d_origs.p, origs, sizeof(float) * 3 * (size_t)n_origs, cudaMemcpyHostToDevice));
    h->has_model = true; h->n = (uint32_t)n; h->width = w; h->height = hgt; h->n_origs = n_origs; h->range_min = rmin; h->range_max = rmax;
    h->perm_tiles = 0;                                             // the tile schedule belongs to the previous model
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
    return set_model_tables(h, m->theta_size, m->phi_size, o, 1, dirs.data(), m->range_min, m->range_max);
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
    const uint32_t grid = (h->n + B2_FIND_BLOCK - 1) / B2_FIND_BLOCK;
    // no L2 prefetch by default: on an H100 (50 MB L2) prefetching the 37 MB node array of a 1M-triangle map slowed the C2 step from
    // 80 to 86 us (nodes + triangles, mode 2: 91 us)
    static const int prefetch_mode = [] { const char* e = getenv("B2_FIND_PREFETCH"); return e ? atoi(e) : 0; }();
    // early_dependents: only when every block of this grid is resident in the first wave (14 blocks per SM), so that an early-resident
    // dependent block can never take an SM slot a find block is still waiting for
    const int early = (h->pdl_next && grid <= 14u * (uint32_t)h->red_grid) ? 1 : 0;
    h->pdl_armed = early != 0;
    // tile schedule (kernels.cuh): whole tiles only, as many as the ICP loop's idle warps sort in the time they have (icp_loop.cuh)
    static const int use_sched = [] { const char* e = getenv("B2_FIND_SCHED"); return e ? atoi(e) : 1; }();
    const uint32_t n_tiles = h->n / 32u;
    const bool sched = use_sched && (h->n % 32u) == 0u && n_tiles >= 2u && n_tiles <= (uint32_t)B2_PERM_MAX_TILES && grid * (B2_FIND_BLOCK / 32u) == n_tiles;
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
    k_rcc_find<<<grid, B2_FIND_BLOCK, 0, h->stream>>>(h->map->view(), h->map->n_nodes, h->map->n_tris, prefetch_mode, nullptr, icp_dev, Tbm_host ? *Tbm_host : tf_identity_pod(), h->Tsb, ray_model(h), 1u, model_buffers(h), early,
                                                      perm, cost);
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

static void fill_sensor_frames(IcpSensor& S, const b2_transform& Tbo, const b2_transform& Tsb)
{
    const Tf Tos = tf_mul(tf_from_pod(Tbo), tf_from_pod(Tsb));
    memset(&S.Tos, 0, sizeof(S.Tos)); memset(&S.Tso, 0, sizeof(S.Tso));
    tf_store(&S.Tos, Tos); tf_store(&S.Tso, tf_inv(Tos)); quat_to_mat(Tos.R, S.Ros);
}

static int launch_icp_loop(b2_rcc* H, const IcpLaunch& L, int grid, size_t smem, int mode, bool pdl, int slot)
{
    unsigned long long* parts = H->d_slots.p; IcpResult* res_dev = H->d_res.p; uint4* host_out = H->pin_chunks_dev + (size_t)slot * (B2_ICP_RESULT_CHUNKS + 1);
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

static int micp_enqueue(SensorCall* sc, uint32_t ns, const b2_transform* Tom, uint32_t iterations, double cp)
{
    b2_rcc* H = sc[0].h;
    if (H->pending.size() >= B2_RING) return fail(B2_ERR_INVALID, "correctOnce: %d asynchronous calls are in flight already, collect one first (b2_rcc_correct_once_wait)", B2_RING);
    static const int use_zc = [] { const char* e = getenv("B2_ZEROCOPY"); return e ? atoi(e) : 1; }();
    static const int use_spin = [] { const char* e = getenv("B2_SPIN"); return e ? atoi(e) : 1; }();
    static const int use_pdl = [] { const char* e = getenv("B2_PDL"); return e ? atoi(e) : 1; }();
    int mode = H->exec_mode;
    if (H->fused_grid <= 0) mode = 0;
    if (ns > 1 && mode == 0) mode = H->fused_grid > 0 ? 1 : 0;
    if (ns > 1 && mode == 0) return fail(B2_ERR_UNSUPPORTED, "multi-sensor correctOnce needs a device with cooperative launch");
    uint64_t total = 0;
    for (uint32_t k = 0; k < ns; k++) {
        b2_rcc* h = sc[k].h;
        if (h->map->device != H->map->device) return fail(B2_ERR_INVALID, "correctOnce: all sensors must live on the same device");
        const bool cpc = h->corr_type == B2_CORR_CPC;
        if (sc[k].ranges_host && cpc) return fail(B2_ERR_INVALID, "correctOnce(ranges) needs ray-casting correspondences (the handle is in closest-point mode)");
        if (!cpc && !h->has_model) return fail(B2_ERR_INVALID, "correctOnce before setModel");
        if (sc[k].ranges_host) {
            if (sc[k].n_ranges != h->n) return fail(B2_ERR_INVALID, "ranges size %u != model size %u", sc[k].n_ranges, h->n);
            h->n_dataset = h->n; h->n_ranges_in = h->n; h->b_dpts = nullptr; h->b_dmask = nullptr;
            if (h->n > 0) { RES(h->d_dpts.reserve(3 * (size_t)h->n)); RES(h->d_dmask.reserve(h->n)); RES(h->d_ranges_in.reserve(h->n)); }
        }
        if (h->n_dataset != h->work_n()) return fail(B2_ERR_INVALID, "dataset size %u != model size %u", h->n_dataset, h->n);
        total += h->work_n();
    }
    if (mode == 0 && !H->pending.empty()) return fail(B2_ERR_INVALID, "correctOnce: exec mode 0 keeps its state in one staging block: collect the pending call first");
    for (const PendingCall& q : H->pending) if (q.kind == 3) return fail(B2_ERR_INVALID, "correctOnce: an exec-mode-0 call is pending: collect it first");
    H->pending.emplace_back();
    PendingCall& pc = H->pending.back();
    struct Guard { b2_rcc* H; bool ok = false; ~Guard() { if (!ok) H->pending.pop_back(); } } guard{H};
    // ---- nothing to do on the device: identity update (micp_localization.cpp:974: Tom stays when n_meas == 0) ----
    if (total == 0 || iterations == 0) {
        memset(&pc.res, 0, sizeof(pc.res));
        pc.res.Tom_new = *Tom; pc.res.T_onew_oold = tf_identity_pod();
        if (total > 0) for (uint32_t k = 0; k < ns; k++) {          // iterations == 0: the reference still runs findCorrespondences (:900-908)
            b2_transform Tbm; memset(&Tbm, 0, sizeof(Tbm)); tf_store(&Tbm, tf_mul(tf_from_pod(*Tom), tf_from_pod(sc[k].Tbo)));
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
        st.Tom = *Tom; st.Tbo = sc[0].Tbo; st.Tsb = h->Tsb; st.max_dist = (float)(h->max_dist * (1.0 - cp) + h->adaptive_max_dist_min * cp);
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
    memset(&L, 0, sizeof(L));
    L.Tom = *Tom; L.n_sensors = ns; L.iterations = iterations;
    uint32_t ns_busy = 0;
    for (uint32_t k = 0; k < ns; k++) if (sc[k].h->work_n() > 0) ns_busy++;
    int grid = std::min<int>(H->fused_grid, (int)std::max<uint64_t>((total + B2_ICP_BLOCK - 1) / B2_ICP_BLOCK, ns_busy));
    // blocks per sensor in proportion to the pairs, at least one for each sensor with pairs.  A sensor without pairs gets none, so the
    // other sensors' pairs are summed by exactly the blocks a call without it would use: its presence cannot change a bit of the result.
    uint32_t nblk[B2_MAX_SENSORS]; int assigned = 0;
    for (uint32_t k = 0; k < ns; k++) {
        const uint32_t nw = sc[k].h->work_n();
        nblk[k] = nw ? std::max<uint32_t>(1u, (uint32_t)((uint64_t)grid * nw / total)) : 0u; assigned += (int)nblk[k];
    }
    while (assigned > grid) { uint32_t big = 0; for (uint32_t k = 1; k < ns; k++) if (nblk[k] > nblk[big]) big = k; nblk[big]--; assigned--; }
    while (assigned < grid) {
        uint32_t best = 0; double load = -1.0;
        for (uint32_t k = 0; k < ns; k++) { if (!nblk[k]) continue; const double l = (double)sc[k].h->work_n() / nblk[k]; if (l > load) { load = l; best = k; } }
        nblk[best]++; assigned++;
    }
    bool aux_any = false;
    uint32_t blk0 = 0, smem_u_max = 0, sort_tiles_max = 0;
    if (H->timing) CU(cudaEventRecord(H->ev[0], H->stream));
    for (uint32_t k = 0; k < ns; k++) {
        b2_rcc* h = sc[k].h;
        IcpSensor& S = L.s[k];
        const uint32_t nw = h->work_n();
        S.n = nw; S.blk0 = blk0; S.nblk = nblk[k]; blk0 += nblk[k];
        const uint32_t stride = S.nblk * B2_ICP_BLOCK;
        const uint32_t per_thread = stride ? (nw + stride - 1) / stride : 0u;
        S.smem_u = per_thread > B2_ICP_REG_PAIRS ? std::min<uint32_t>(per_thread - B2_ICP_REG_PAIRS, (uint32_t)H->smem_u_cap) : 0u;
        smem_u_max = std::max(smem_u_max, S.smem_u);
        S.max_dist = (float)(h->max_dist * (1.0 - cp) + h->adaptive_max_dist_min * cp);       // CorrespondencesCPU.cpp:21-23
        S.merge_weight = sc[k].weight; S.range_min = h->range_min; S.range_max = h->range_max;
        fill_sensor_frames(S, sc[k].Tbo, h->Tsb);
        // Pinned scan (B2_ZEROCOPY, default 1): a copy engine moves it into the handle's buffer on the side stream WHILE find runs, a second small
        // copy behind it raises a flag, and the loop kernel -- launched programmatically behind find, no event in between -- checks the flag
        // before it unpacks the scan.  2: the loop kernel reads the caller's buffer itself over PCIe (latency-sensitive: 10-20 us slower on some
        // hosts).  Needs every pair of the sensor resident in registers / shared memory.  Pageable buffers take the staged upload below.
        const float* zc = nullptr; bool zc_dma = false;
        if (sc[k].ranges_host && nw > 0 && use_zc && per_thread <= B2_ICP_REG_PAIRS + S.smem_u) {
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
        if (h != H) {           // order the lead stream behind this sensor's own stream (pending set_ranges / set_dataset copies)
            CU(cudaEventRecord(h->ev_join, h->stream));
            CU(cudaStreamWaitEvent(H->stream, h->ev_join, 0));
        }
        b2_transform Tbm_host; memset(&Tbm_host, 0, sizeof(Tbm_host));
        tf_store(&Tbm_host, tf_mul(tf_from_pod(*Tom), tf_from_pod(sc[k].Tbo)));          // MICPSensor.hpp:148, same inline ops as the kernels
        pc.sensors[k] = h; pc.Tbm[k] = Tbm_host;
        // the loop kernel may start early behind the LAST find only (event records / other kernels in between would serialise them anyway)
        const cudaStream_t own = h->stream;
        h->stream = H->stream;                                                        // all launches of this call ride the lead stream
        h->pdl_next = (k + 1 == ns) && mode == 2 && use_pdl && !H->timing && h->corr_type == B2_CORR_RCC && !need_upload && !aux_any;
        const int rc_find = launch_find(h, &Tbm_host, nullptr);
        h->pdl_next = false; h->stream = own;
        RES(rc_find);
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
        if (h->corr_type == B2_CORR_RCC && h->cost_tiles && iterations >= 3u) {
            S.tile_cost = h->d_tile_cost.p; S.tile_perm = h->d_tile_perm.p; S.n_tiles = h->cost_tiles;
            sort_tiles_max = std::max(sort_tiles_max, h->cost_tiles);
        }
        S.dpts = h->dpts(); S.dmask = h->dmask(); S.mpts = h->mpts(); S.mnrm = h->mnrm(); S.mmask = h->mhits();
        S.zc_ranges = zc; S.zc_dirs = h->d_dirs.p; S.zc_origs = h->d_origs.p; S.zc_n_origs = h->n_origs;
        S.dpts_out = h->d_dpts.p; S.dmask_out = h->d_dmask.p; S.ranges_out = h->d_ranges_in.p;
    }
    if (H->timing) CU(cudaEventRecord(H->ev[1], H->stream));
    L.smem_u_max = smem_u_max;
    unsigned int seq = ++H->seq; if (seq == 0) seq = ++H->seq;
    L.seq = seq;
    size_t smem = (size_t)smem_u_max * 9 * B2_ICP_BLOCK * sizeof(float);
    if (sort_tiles_max) {
        // the tile sort stages the durations behind the pair cache (2 bytes per tile); no room (very large scans): no sort, the order stays as it is
        const size_t want = smem + 2 * (size_t)sort_tiles_max;
        if (want <= (size_t)H->smem_u_cap * 9 * B2_ICP_BLOCK * sizeof(float)) smem = want;
        else for (uint32_t k = 0; k < ns; k++) { L.s[k].tile_cost = nullptr; L.s[k].tile_perm = nullptr; L.s[k].n_tiles = 0; }
    }
    const bool pdl = mode == 2 && sc[ns - 1].h->pdl_armed && !aux_any;
    sc[ns - 1].h->pdl_armed = false;
    pc.slot = (int)(H->slot_counter++ % B2_RING);
    RES(launch_icp_loop(H, L, grid, smem, mode, pdl, pc.slot));
    H->loop_geom[0] = ns; H->loop_geom[1] = (uint32_t)grid;
    for (uint32_t k = 0; k < B2_MAX_SENSORS; k++) {
        uint32_t* g = H->loop_geom + 2 + 4 * k;
        if (k < ns) { g[0] = L.s[k].n; g[1] = L.s[k].blk0; g[2] = L.s[k].nblk; g[3] = L.s[k].smem_u; } else g[0] = g[1] = g[2] = g[3] = 0u;
    }
    if (H->timing) { CU(cudaEventRecord(H->ev[2], H->stream)); H->timing_valid = true; }
    for (uint32_t k = 1; k < ns; k++) {        // later work on the other sensors' own streams sees the model buffers this call wrote
        CU(cudaEventRecord(sc[k].h->ev_join, H->stream));
        CU(cudaStreamWaitEvent(sc[k].h->stream, sc[k].h->ev_join, 0));
    }
    pc.seq = seq; pc.grid = grid; pc.smem = smem; pc.barrier_used = mode == 2;
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
                unsigned int bar_state[2] = {0u, 0u};
                CU(cudaMemcpy(bar_state, H->d_bar.p, sizeof(bar_state), cudaMemcpyDeviceToHost));
                if (bar_state[1] != 0u) {
                    // The loop's grid-wide exchange gave up (its blocks were not co-resident: SMs held by something that itself waits).  That is a
                    // scheduling condition, not an error: reset the abort word; this call and every later call already in flight (their kernels
                    // saw the abort word and left) run again through the cooperative launch, whose co-residency the driver guarantees.
                    // (code 2: a block's partial sum left the fixed-point range of the atomic exchange; the cooperative variant exchanges FP64)
                    CU(cudaMemset(H->d_bar.p + 1, 0, sizeof(unsigned int)));
                    CU(cudaMemset(H->d_slots.p, 0, ((size_t)B2_ICP_ACC_WORDS + B2_ICP_BASE_WORDS) * sizeof(unsigned long long)));      // the aborted rounds left them inconsistent
                    pc.rerun = true;
                    for (PendingCall& q : H->pending) if (q.barrier_used) q.rerun = true;
                }
            }
            if (pc.rerun) {
                H->n_reruns++;
                for (uint32_t k = 0; k < pc.launch.n_sensors; k++) {
                    b2_rcc* h = pc.sensors[k];
                    const cudaStream_t own = h->stream; h->stream = H->stream; h->pdl_next = false;
                    const int rc = launch_find(h, &pc.Tbm[k], nullptr);
                    h->stream = own;
                    RES(rc);
                }
                unsigned int seq = ++H->seq; if (seq == 0) seq = ++H->seq;
                pc.launch.seq = seq; pc.seq = seq;
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
    if (n_sensors == 0 || n_sensors > B2_MAX_SENSORS) return fail(B2_ERR_INVALID, "correctOnce: %u sensors (1..%d supported per call)", n_sensors, B2_MAX_SENSORS);
    SensorCall sc[B2_MAX_SENSORS];
    for (uint32_t k = 0; k < n_sensors; k++) {
        NOTNULL(sensors[k]);
        for (uint32_t j = 0; j < k; j++) if (sensors[j] == sensors[k]) return fail(B2_ERR_INVALID, "correctOnce: sensor %u given twice", k);
        sc[k].h = sensors[k]; sc[k].Tbo = Tbo[k]; sc[k].weight = merge_weights ? merge_weights[k] : 1.0;
        sc[k].ranges_host = ranges_host ? ranges_host[k] : nullptr; sc[k].n_ranges = sc[k].ranges_host ? sensors[k]->n : 0;
    }
    CU(cudaSetDevice(sc[0].h->map->device));
    if (!sc[0].h->pending.empty()) return fail(B2_ERR_INVALID, "correctOnce: asynchronous calls are still in flight on the lead handle, collect them first");
    RES(micp_enqueue(sc, n_sensors, Tom, iterations, cp));
    return micp_collect(sc[0].h, Tom_new, T_onew_oold, Cmerged);
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
        k_rcc_find<<<(uint32_t)((total + B2_FIND_BLOCK - 1) / B2_FIND_BLOCK), B2_FIND_BLOCK, 0, h->stream>>>(h->map->view(), h->map->n_nodes, h->map->n_tris, 0, h->d_poses.p, nullptr,
                                                                                                        tf_identity_pod(), h->Tsb, ray_model(h), n_poses, out, 0, nullptr, nullptr);
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
    cleanup();
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
struct b2_pf {
    b2_mesh* map = nullptr; cudaStream_t stream = 0;
    DevBuf<PfBeam> d_beams; PfBeam* h_beams = nullptr; size_t h_beams_cap = 0;
    DevBuf<b2_transform> d_poses; DevBuf<b2_particle_attr> d_attrs;
    DevBuf<double> d_part; DevBuf<unsigned int> d_ticket; DevBuf<float> d_out; float* h_out = nullptr; int n_sm = 0;
    int smem_optin = 0;
    cudaStream_t side = nullptr; cudaEvent_t ev_beams = nullptr, ev_side = nullptr;      // second stream of the chunked host variant (b2_pf_sensor_update_host)
    // ray mapping of k_pf_update (kernels.cuh): 0 lanes = beams, 1 lanes = particles, 2 lanes = particles sorted by pose, 3 (default) whichever of 0 / 2
    // was faster when last timed -- both are timed on the first updates and the loser again every 64 updates (particle sets converge and spread out)
    int map_mode = 3, map_cur = 0, map_best = 0; unsigned int map_updates = 0; float map_ms[2] = {0.f, 0.f}; bool map_timed = false;
    cudaEvent_t ev_m0 = nullptr, ev_m1 = nullptr;
    DevBuf<uint32_t> d_keys, d_keys2, d_idx, d_idx2; DevBuf<unsigned char> d_sort_tmp;
    // sharded resampling over NVLink peer memory (b2_pf_p2p_*): own exchange buffers (cudaMalloc: exportable through CUDA IPC) + the peers' mappings
    b2_transform* x_poses = nullptr; b2_particle_attr* x_attrs = nullptr; uint32_t x_cap = 0;
    PfPeers peers{}; bool peers_open = false; DevBuf<unsigned long long> d_traffic;
};

extern "C" int b2_pf_destroy(b2_pf* h);

static int pf_init(b2_pf* h)
{
    b2_mesh* map = h->map;
    CU(cudaDeviceGetAttribute(&h->smem_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, map->device));
    h->smem_optin -= 1024;              // room for the kernel's static shared memory
    CU(cudaDeviceGetAttribute(&h->n_sm, cudaDevAttrMultiProcessorCount, map->device));
    RES(h->d_part.reserve(2 * (size_t)h->n_sm * 4)); RES(h->d_ticket.reserve(1)); RES(h->d_out.reserve(2));
    CU(cudaMemset(h->d_ticket.p, 0, sizeof(unsigned int)));
    CU(cudaMallocHost((void**)&h->h_out, 2 * sizeof(float)));
    CU(cudaFuncSetAttribute(k_pf_update<0, 0>, cudaFuncAttributeMaxDynamicSharedMemorySize, h->smem_optin));
    CU(cudaFuncSetAttribute(k_pf_update<1, 0>, cudaFuncAttributeMaxDynamicSharedMemorySize, h->smem_optin));
    CU(cudaFuncSetAttribute(k_pf_update<0, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, h->smem_optin));
    CU(cudaFuncSetAttribute(k_pf_update<1, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, h->smem_optin));
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
    h->d_beams.release(); h->d_poses.release(); h->d_attrs.release(); h->d_part.release(); h->d_ticket.release(); h->d_out.release();
    if (h->h_beams) cudaFreeHost(h->h_beams);
    if (h->h_out) cudaFreeHost(h->h_out);
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
    h->d_traffic.release();
    b2_mesh* map = h->map;
    delete h;
    (void)cudaGetLastError();
    mesh_unref(map);
    return B2_OK;
}
extern "C" int b2_pf_set_stream(b2_pf* h, void* s) { NOTNULL(h); h->stream = (cudaStream_t)s; return B2_OK; }

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
static int pf_launch(b2_pf* h, const b2_transform* poses_dev, b2_particle_attr* attrs_dev, uint32_t n, const b2_transform* Tsb, uint32_t n_beams, const b2_pf_params* prm,
                     uint32_t ppb, cudaStream_t stream, int map = 0, const uint32_t* order = nullptr)
{
    const size_t bytes_per_particle = sizeof(float) * (size_t)n_beams;
    if (map) { ppb = 32; if (bytes_per_particle * ppb > (size_t)h->smem_optin) { map = 0; order = nullptr; ppb = std::max(1u, (uint32_t)((size_t)h->smem_optin / bytes_per_particle)); } }
    const uint32_t grid = (n + ppb - 1) / ppb;
    const size_t smem = bytes_per_particle * ppb;
    const bool cp = prm->correspondence_type == 1;
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
    RES(h->d_traffic.reserve(1));
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
    CU(cudaMemsetAsync(h->d_traffic.p, 0, sizeof(unsigned long long), h->stream));
    k_pf_gladiator_p2p<<<(h->peers.n_per_rank + 255) / 256, 256, 0, h->stream>>>(h->peers, poses_new_dev, attrs_new_dev, *cfg, seed, step, h->d_traffic.p);
    LAUNCHED();
    if (remote_bytes_out) {
        unsigned long long t = 0;
        CU(cudaMemcpyAsync(&t, h->d_traffic.p, sizeof(t), cudaMemcpyDeviceToHost, h->stream));
        CU(cudaStreamSynchronize(h->stream));
        *remote_bytes_out = t;
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
    RES(h->d_traffic.reserve(1));
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

extern "C" int b2_pf_likelihood_stats(b2_pf* h, const b2_particle_attr* attrs_dev, uint32_t n, float* sum_out, float* max_out)
{
    NOTNULL(h);
    CU(cudaSetDevice(h->map->device));
    float s = 0.f, m = 0.f;
    if (n > 0) {
        NOTNULL(attrs_dev);
        const uint32_t grid = std::min<uint32_t>((uint32_t)h->n_sm * 4u, (n + 255) / 256);
        k_pf_stats<<<grid, 256, 0, h->stream>>>(attrs_dev, n, h->d_part.p, h->d_ticket.p, h->d_out.p);
        LAUNCHED();
        CU(cudaMemcpyAsync(h->h_out, h->d_out.p, 2 * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
        CU(cudaStreamSynchronize(h->stream));
        s = h->h_out[0]; m = h->h_out[1];
    }
    if (sum_out) *sum_out = s;
    if (max_out) *max_out = m;
    return B2_OK;
}
