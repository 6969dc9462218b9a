// bvh8.h -- in-HBM layout of the map: 8-wide BVH with FLOAT child boxes (224-byte nodes) + 48-byte leaf triangle records.
// Shared by the host builder and the traversal kernels.
//
// Why uncompressed: the traversal is bound by instruction issue and latency more than by bytes, and every byte saved per node costs
// decode instructions on every visit.
// Round 1 started with 80-byte nodes with 8-bit quantised planes (the published "compressed wide BVH" idea, Ylitie et al. 2017): every
// visit paid ~70 instructions of per-node frame math and 48 byte->float conversions.  Float planes need neither: a child plane is one
// FMA with per-RAY constants.  The wide-node organisation kept from that design: 8 children in octant-ordered slots (traversal order =
// slot ^ ray octant, no sorting at run time), one contiguous run of inner children and of leaf triangles per node, <= 3 triangles per
// leaf child encoded in a meta byte.
//
// Node (224 B = 14 x 16 B), planes SoA so that a ray picks "near" and "far" arrays by its direction signs with an address offset:
//   +0    float lo_x[8]   +32  float lo_y[8]   +64  float lo_z[8]
//   +96   float hi_x[8]   +128 float hi_y[8]   +160 float hi_z[8]
//   +192  u32 child_base (index of first inner child), u32 tri_base (index of first leaf triangle record),
//         u32 masks = imask (bits 0..7, bit s: slot s is an inner node) | trimask << 8 (bit 3s+j: triangle j of leaf child s exists), u32 pad
//         -- everything the RAY traversal needs sits in quads 0..12 (13 loads per visit); its hit mask is built from the 8 box-test
//         bits with a handful of bit operations (trace.cuh:node_test) instead of decoding one meta byte per child
//   +208  u8 meta[8], 8 B pad -- per-child records for the closest-point traversal, the refit and the blob validation:
//   meta[s]: 0 = empty; inner: 0x20 | (24 + s); leaf: (unary triangle count 1|3|7) << 5 | offset of its first triangle from tri_base
//   The records of a node's leaf children are contiguous in slot order, so the record of slot-space bit b is tri_base + popc(trimask & ((1<<b)-1)).
//   empty slots have lo = +inf, hi = -inf (never hit).  Child boxes are the exact float AABBs (min/max of vertices) of the triangles below.
//   Slot s "points" along D_s = (s&1 ? + : -, s&2 ? + : -, s&4 ? + : -); a ray with octant code r (bit k set iff d_k >= 0) visits inner
//   children in order of descending (s ^ r).
//
// Leaf triangle record (48 B = 3 x 16 B): (v0.xyz, face_id as bits), (v1.xyz, 0), (v2.xyz, 0); records of one node are contiguous,
// in slot order; at most 3 triangles per leaf child, at most 24 per node.
#pragma once
#include <stddef.h>
#include <stdint.h>

struct alignas(16) B2Node8 {
    float    lo[3][8];
    float    hi[3][8];
    uint32_t child_base;
    uint32_t tri_base;
    uint32_t masks;                 // imask | trimask << 8
    uint32_t pad0;
    uint8_t  meta[8];
    uint32_t pad[2];                // 224 B measured faster than padding to 256 B (smaller footprint: 79.9 vs 82.5 us cold, 63.5 vs 67.6 us warm on C2)
#if defined(__CUDACC__)
    __host__ __device__
#endif
    uint32_t imask() const { return masks & 0xffu; }
};
// masks word of a node from its meta bytes (both builders): imask from the inner markers, trimask from the unary leaf counts
#if defined(__CUDACC__)
__host__ __device__
#endif
inline uint32_t b2_masks_from_meta(const uint8_t meta[8])
{
    uint32_t m = 0;
    for (int s = 0; s < 8; s++) {
        const uint32_t v = meta[s];
        if (!v) continue;
        if ((v & 0x18u) == 0x18u && (v >> 5) == 1u) m |= 1u << s;                 // inner marker 0x20 | (24 + s)
        else m |= (v >> 5) << (8 + 3 * s);                                        // unary count 1 | 3 | 7 at slot-space bits 3s..3s+2
    }
    return m;
}
static_assert(sizeof(B2Node8) == 224, "node must be 224 bytes");
#define B2_NODE_BYTES 224
#define B2_NODE_QUADS 14

struct alignas(16) B2Tri {
    float    v0[3]; uint32_t face_id;
    float    v1[3]; uint32_t pad1;
    float    v2[3]; uint32_t pad2;
};
static_assert(sizeof(B2Tri) == 48, "triangle record must be 48 bytes");

#define B2_TRAVERSAL_STACK 40          // uint2 entries per ray; builder refuses trees deeper than B2_TRAVERSAL_STACK - 4
#define B2_MAX_LEAF_TRIS 3

// Largest |vertex coordinate| a map accepts: 2^62.  Box extents then stay below 2^63, so every box half-area the builders form
// (dx dy + dy dz + dz dx <= 3 * 2^126 < FLT_MAX), every box centre 0.5 (lo + hi) and every slot cost (a sum of three centre differences)
// is finite; larger coordinates would turn them into inf / NaN and the SAH and octant decisions with them.
#define B2_MAX_ABS_COORD 4611686018427387904.0f
// vertices a map can be built or refitted from: finite and within B2_MAX_ABS_COORD
inline bool b2_vertices_ok(const float* v, size_t n_floats)
{
    for (size_t i = 0; i < n_floats; i++) if (!(v[i] >= -B2_MAX_ABS_COORD && v[i] <= B2_MAX_ABS_COORD)) return false;
    return true;
}

// BVH blob (b2_mesh_export_blob / b2_mesh_create_from_blob): this header, then n_nodes B2Node8, then n_tris B2Tri
struct B2BlobHeader {
    char     magic[8];                 // "B2BVH8F\0"
    uint32_t version, node_bytes, tri_bytes, n_nodes, n_tris, n_faces, n_verts, max_depth;
    int32_t  build_mode;
    float    abs_max[3], sah;
    uint32_t pad;                      // 64 bytes: the node array that follows stays 16-byte aligned inside an aligned buffer
};
static_assert(sizeof(B2BlobHeader) == 64, "blob header must be 64 bytes");

// host-side result of a build
struct B2BvhHost {
    B2Node8* nodes = nullptr; uint32_t n_nodes = 0;
    B2Tri*   tris = nullptr;  uint32_t n_tris = 0;
    uint32_t max_depth = 0;
    float    sah_cost = 0.f;
    float    abs_max[3] = {0, 0, 0};   // max |coordinate| per axis over all vertices (slack constant of the box test)
};

// host SAH builder (bvh_build.cpp). Returns 0 on success, negative on failure (message via *err).
int b2_build_bvh8_host(const float* verts, uint32_t nv, const uint32_t* faces, uint32_t nf, B2BvhHost* out, const char** err);
void b2_free_bvh8_host(B2BvhHost* b);
