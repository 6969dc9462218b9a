// bvh_build.cpp -- host builder of the in-HBM map: binned-SAH binary BVH -> cost-optimal 8-wide collapse -> octant slot
// assignment -> float child boxes (layout: bvh8.h).  Runs once per map at b2_mesh_create (replaces the Embree scene commit
// behind rm::import_embree_map, rmcl_ros/src/nodes/micp_localization.cpp:188); it is NOT on the per-scan path.
#include "bvh8.h"

#include <algorithm>
#include <atomic>
#include <cfloat>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <vector>

namespace {

struct Box {
    float lo[3], hi[3];
    void reset() { for (int k = 0; k < 3; k++) { lo[k] = FLT_MAX; hi[k] = -FLT_MAX; } }
    void grow(const Box& b) { for (int k = 0; k < 3; k++) { lo[k] = std::min(lo[k], b.lo[k]); hi[k] = std::max(hi[k], b.hi[k]); } }
    float half_area() const {
        float dx = hi[0] - lo[0], dy = hi[1] - lo[1], dz = hi[2] - lo[2];
        if (dx < 0) return 0.f;
        return dx * dy + dy * dz + dz * dx;
    }
};

struct Node2 {
    Box box;
    uint32_t left;      // inner: index of left child (right = left + 1); leaf: primitive id
    uint32_t count;     // number of triangles below
    bool leaf;
};

struct Prim { Box box; float c[3]; };

constexpr int   kBins = 32;
constexpr float kCNode = 1.0f;      // cost of visiting one wide node
static float kCPrim = 0.35f;        // cost of testing one triangle relative to visiting one wide node (B2_SAH_CPRIM overrides)
constexpr float kInf = INFINITY;    // "no candidate yet": every finite cost beats it

struct Builder {
    const Prim* prims;
    uint32_t* order;                 // permutation of primitive ids
    Node2* nodes;
    std::atomic<uint32_t> n_nodes{0};

    void build(uint32_t node_idx, uint32_t first, uint32_t count)
    {
        Node2& nd = nodes[node_idx];
        Box cb; cb.reset(); nd.box.reset();
        for (uint32_t i = first; i < first + count; i++) {
            const Prim& p = prims[order[i]];
            nd.box.grow(p.box);
            for (int k = 0; k < 3; k++) { cb.lo[k] = std::min(cb.lo[k], p.c[k]); cb.hi[k] = std::max(cb.hi[k], p.c[k]); }
        }
        nd.count = count;
        if (count == 1) { nd.leaf = true; nd.left = order[first]; return; }
        nd.leaf = false;

        float best = kInf; int best_axis = -1, best_split = 0;
        for (int ax = 0; ax < 3; ax++) {
            const float ext = cb.hi[ax] - cb.lo[ax];
            if (!(ext > 0.f)) continue;
            Box bb[kBins]; uint32_t bc[kBins];
            for (int b = 0; b < kBins; b++) { bb[b].reset(); bc[b] = 0; }
            const float scale = (float)kBins / ext;
            for (uint32_t i = first; i < first + count; i++) {
                const Prim& p = prims[order[i]];
                int b = (int)((p.c[ax] - cb.lo[ax]) * scale); b = std::min(std::max(b, 0), kBins - 1);
                bb[b].grow(p.box); bc[b]++;
            }
            float ra[kBins]; uint32_t rc[kBins];
            Box acc; acc.reset(); uint32_t c = 0;
            for (int b = kBins - 1; b > 0; b--) { acc.grow(bb[b]); c += bc[b]; ra[b] = acc.half_area(); rc[b] = c; }
            acc.reset(); c = 0;
            for (int b = 0; b < kBins - 1; b++) {
                acc.grow(bb[b]); c += bc[b];
                if (c == 0 || rc[b + 1] == 0) continue;
                const float cost = acc.half_area() * (float)c + ra[b + 1] * (float)rc[b + 1];
                if (cost < best) { best = cost; best_axis = ax; best_split = b + 1; }
            }
        }
        uint32_t mid;
        if (best_axis < 0) {
            mid = first + count / 2;
        } else {
            const float ext = cb.hi[best_axis] - cb.lo[best_axis];
            const float scale = (float)kBins / ext;
            uint32_t* lo = order + first; uint32_t* hi = order + first + count;
            uint32_t* m = std::partition(lo, hi, [&](uint32_t id) {
                int b = (int)((prims[id].c[best_axis] - cb.lo[best_axis]) * scale); b = std::min(std::max(b, 0), kBins - 1);
                return b < best_split;
            });
            mid = (uint32_t)(m - order);
            if (mid == first || mid == first + count) mid = first + count / 2;
        }
        const uint32_t left = n_nodes.fetch_add(2);
        nd.left = left;
        const uint32_t lc = mid - first, rc2 = count - lc;
        if (count > 8192) {
            #pragma omp task
            build(left, first, lc);
            #pragma omp task
            build(left + 1, mid, rc2);
            #pragma omp taskwait
        } else {
            build(left, first, lc);
            build(left + 1, mid, rc2);
        }
    }
};

// ---- wide collapse (dynamic programme over the binary tree) ----
struct Dp {
    float c[8];          // c[i], i = 1..7: cheapest representation of the subtree as <= i wide-BVH children
    uint8_t dist[9];     // dist[j], j = 2..8: how many of the j roots go to the left child in the best split
    uint8_t use_dist[8]; // use_dist[i], i = 2..7: 1 if c[i] comes from distributing i roots, 0 if from c[i-1]
    uint8_t kind1;       // representation behind c[1]: 0 = leaf (<= 3 triangles), 1 = inner wide node
};

struct ChildRef { uint32_t node2; bool leaf; };

void gather(const Node2* n2, const Dp* dp, uint32_t n, int j, std::vector<ChildRef>& out)
{
    // represent subtree n with at most j roots, following the recorded decisions
    const Node2& nd = n2[n];
    if (nd.leaf) { out.push_back({n, true}); return; }
    while (j >= 2 && j <= 7 && !dp[n].use_dist[j]) j--;
    if (j == 1) { out.push_back({n, dp[n].kind1 == 0}); return; }
    const int k = dp[n].dist[j];
    gather(n2, dp, nd.left, k, out);
    gather(n2, dp, nd.left + 1, j - k, out);
}

void collect_tris(const Node2* n2, uint32_t n, std::vector<uint32_t>& out)
{
    if (n2[n].leaf) { out.push_back(n2[n].left); return; }
    collect_tris(n2, n2[n].left, out);
    collect_tris(n2, n2[n].left + 1, out);
}

} // namespace

void b2_free_bvh8_host(B2BvhHost* b)
{
    if (!b) return;
    free(b->nodes); free(b->tris);
    b->nodes = nullptr; b->tris = nullptr; b->n_nodes = b->n_tris = 0;
}

int b2_build_bvh8_host(const float* verts, uint32_t nv, const uint32_t* faces, uint32_t nf, B2BvhHost* out, const char** err)
{
    static const char* e_empty = "empty mesh";
    static const char* e_index = "face index out of range";
    static const char* e_nan = "a vertex coordinate is not finite or exceeds 2^62 in magnitude";
    static const char* e_depth = "BVH too deep for the traversal stack";
    static const char* e_oom = "out of host memory";
    *out = B2BvhHost();
    if (const char* e = getenv("B2_SAH_CPRIM")) kCPrim = (float)atof(e);
    if (nf == 0 || nv == 0) { *err = e_empty; return -3; }
    for (uint32_t i = 0; i < 3 * nf; i++) if (faces[i] >= nv) { *err = e_index; return -1; }
    if (!b2_vertices_ok(verts, 3 * (size_t)nv)) { *err = e_nan; return -1; }

    std::vector<Prim> prims(nf);
    std::vector<uint32_t> order(nf);
    #pragma omp parallel for schedule(static)
    for (int64_t f = 0; f < (int64_t)nf; f++) {
        Prim& p = prims[f]; p.box.reset();
        for (int j = 0; j < 3; j++) {
            const float* v = verts + 3 * (size_t)faces[3 * f + j];
            for (int k = 0; k < 3; k++) { p.box.lo[k] = std::min(p.box.lo[k], v[k]); p.box.hi[k] = std::max(p.box.hi[k], v[k]); }
        }
        for (int k = 0; k < 3; k++) p.c[k] = 0.5f * (p.box.lo[k] + p.box.hi[k]);
        order[f] = (uint32_t)f;
    }

    const size_t max_nodes2 = 2 * (size_t)nf;
    Node2* n2 = (Node2*)malloc(sizeof(Node2) * max_nodes2);
    if (!n2) { *err = e_oom; return -4; }
    Builder bld; bld.prims = prims.data(); bld.order = order.data(); bld.nodes = n2; bld.n_nodes = 1;
    #pragma omp parallel
    {
        #pragma omp single
        bld.build(0, 0, nf);
    }
    const uint32_t nn2 = bld.n_nodes.load();

    // ---- DP, children always have larger indices than their parent -> descending order is bottom-up ----
    std::vector<Dp> dp(nn2);
    for (int64_t n = (int64_t)nn2 - 1; n >= 0; n--) {
        const Node2& nd = n2[n]; Dp& d = dp[n];
        const float A = nd.box.half_area();
        memset(&d, 0, sizeof(Dp));
        if (nd.leaf) { for (int i = 1; i <= 7; i++) d.c[i] = A * kCPrim; d.kind1 = 0; continue; }
        const Dp& L = dp[nd.left]; const Dp& R = dp[nd.left + 1];
        float cd[9];
        for (int j = 2; j <= 8; j++) {
            float best = kInf; int bk = 1;
            for (int k = 1; k < j; k++) {
                if (k > 7 || j - k > 7) continue;
                const float c = L.c[k] + R.c[j - k];
                if (c < best) { best = c; bk = k; }
            }
            cd[j] = best; d.dist[j] = (uint8_t)bk;
        }
        // a sub-tree with more triangles than a leaf child holds is an inner node whatever the costs say (they may be inf)
        const float c_leaf = A * (float)nd.count * kCPrim;
        const float c_inner = cd[8] + A * kCNode;
        if (nd.count <= B2_MAX_LEAF_TRIS && c_leaf <= c_inner) { d.c[1] = c_leaf; d.kind1 = 0; } else { d.c[1] = c_inner; d.kind1 = 1; }
        for (int i = 2; i <= 7; i++) {
            if (cd[i] < d.c[i - 1]) { d.c[i] = cd[i]; d.use_dist[i] = 1; } else { d.c[i] = d.c[i - 1]; d.use_dist[i] = 0; }
        }
    }

    // ---- emit wide nodes breadth-first ----
    struct Pending { uint32_t node2; uint32_t depth; };
    std::vector<Pending> queue; queue.reserve(nf / 2 + 16);
    std::vector<B2Node8> nodes8; nodes8.reserve(nf / 2 + 16);
    std::vector<B2Tri> tris8; tris8.reserve(nf);
    queue.push_back({0, 1}); nodes8.emplace_back();
    uint32_t max_depth = 1; double sah = 0.0;
    const float rootA = std::max(n2[0].box.half_area(), 1e-30f);

    std::vector<ChildRef> ch; std::vector<uint32_t> tl;
    for (size_t qi = 0; qi < queue.size(); qi++) {
        const Pending pe = queue[qi];
        const Node2& nd = n2[pe.node2];
        max_depth = std::max(max_depth, pe.depth);
        ch.clear();
        if (nd.leaf) ch.push_back({pe.node2, true});
        else {
            const int k = dp[pe.node2].dist[8];
            gather(n2, dp.data(), nd.left, k, ch);
            gather(n2, dp.data(), nd.left + 1, 8 - k, ch);
        }
        const int nc = (int)ch.size();
        sah += (double)nd.box.half_area() / rootA * kCNode;

        // slot assignment: greedy on cost[c][s] = (centroid_c - centroid_node) . D_s
        float cen[3]; for (int k = 0; k < 3; k++) cen[k] = 0.5f * (nd.box.lo[k] + nd.box.hi[k]);
        float cost[8][8];
        for (int c = 0; c < nc; c++) {
            const Box& b = n2[ch[c].node2].box;
            float d[3]; for (int k = 0; k < 3; k++) d[k] = 0.5f * (b.lo[k] + b.hi[k]) - cen[k];
            for (int s = 0; s < 8; s++)
                cost[c][s] = ((s & 1) ? d[0] : -d[0]) + ((s & 2) ? d[1] : -d[1]) + ((s & 4) ? d[2] : -d[2]);
        }
        int slot_of[8]; int child_in_slot[8];
        for (int i = 0; i < 8; i++) { slot_of[i] = -1; child_in_slot[i] = -1; }
        for (int it = 0; it < nc; it++) {
            float bv = -kInf; int bc = -1, bs = -1;
            for (int c = 0; c < nc; c++) if (slot_of[c] < 0)
                for (int s = 0; s < 8; s++) if (child_in_slot[s] < 0 && cost[c][s] > bv) { bv = cost[c][s]; bc = c; bs = s; }
            if (bc < 0) {                                 // every remaining cost is NaN or -inf: first free child into the first free slot
                for (bc = 0; slot_of[bc] >= 0; bc++) {}
                for (bs = 0; child_in_slot[bs] >= 0; bs++) {}
            }
            slot_of[bc] = bs; child_in_slot[bs] = bc;
        }

        B2Node8 nd8; memset(&nd8, 0, sizeof(nd8));
        for (int k = 0; k < 3; k++) for (int s8 = 0; s8 < 8; s8++) { nd8.lo[k][s8] = INFINITY; nd8.hi[k][s8] = -INFINITY; }
        nd8.child_base = (uint32_t)nodes8.size();
        nd8.tri_base = (uint32_t)tris8.size();
        uint32_t tri_off = 0;
        for (int s = 0; s < 8; s++) {
            const int c = child_in_slot[s];
            if (c < 0) continue;                      // empty slot: meta 0, box (+inf, -inf)
            const Node2& cn = n2[ch[c].node2];
            for (int k = 0; k < 3; k++) { nd8.lo[k][s] = cn.box.lo[k]; nd8.hi[k][s] = cn.box.hi[k]; }
            if (ch[c].leaf) {
                tl.clear(); collect_tris(n2, ch[c].node2, tl);
                std::sort(tl.begin(), tl.end());
                const uint32_t cnt = (uint32_t)tl.size();                 // 1..3
                const uint32_t unary = cnt == 1 ? 1u : (cnt == 2 ? 3u : 7u);
                nd8.meta[s] = (uint8_t)((unary << 5) | tri_off);
                for (uint32_t t = 0; t < cnt; t++) {
                    B2Tri tr; memset(&tr, 0, sizeof(tr));
                    const uint32_t f = tl[t];
                    const float* a = verts + 3 * (size_t)faces[3 * (size_t)f + 0];
                    const float* b = verts + 3 * (size_t)faces[3 * (size_t)f + 1];
                    const float* c3 = verts + 3 * (size_t)faces[3 * (size_t)f + 2];
                    for (int k = 0; k < 3; k++) { tr.v0[k] = a[k]; tr.v1[k] = b[k]; tr.v2[k] = c3[k]; }
                    tr.face_id = f;
                    tris8.push_back(tr);
                }
                tri_off += cnt;
                sah += (double)cn.box.half_area() / rootA * kCPrim * cnt;
            } else {
                nd8.meta[s] = (uint8_t)(0x20 | (24 + s));
                queue.push_back({ch[c].node2, pe.depth + 1});
                nodes8.emplace_back();
            }
        }
        nd8.masks = b2_masks_from_meta(nd8.meta);
        nodes8[qi] = nd8;
    }
    free(n2);

    if (max_depth > B2_TRAVERSAL_STACK - 4) { *err = e_depth; return -5; }

    out->n_nodes = (uint32_t)nodes8.size();
    out->n_tris = (uint32_t)tris8.size();
    out->nodes = (B2Node8*)malloc(sizeof(B2Node8) * nodes8.size());
    out->tris = (B2Tri*)malloc(sizeof(B2Tri) * std::max<size_t>(tris8.size(), 1));
    if (!out->nodes || !out->tris) { b2_free_bvh8_host(out); *err = e_oom; return -4; }
    memcpy(out->nodes, nodes8.data(), sizeof(B2Node8) * nodes8.size());
    memcpy(out->tris, tris8.data(), sizeof(B2Tri) * tris8.size());
    out->max_depth = max_depth;
    out->sah_cost = (float)sah;
    for (int k = 0; k < 3; k++) out->abs_max[k] = 0.f;
    for (size_t i = 0; i < (size_t)nv; i++) for (int k = 0; k < 3; k++) out->abs_max[k] = std::max(out->abs_max[k], std::fabs(verts[3 * i + k]));
    return 0;
}
