// emul.cu -- TEST HARNESS ONLY: runs the product's host+device traversal / math functions (rmcl_b200/csrc/*.cuh) on the CPU so
// that the BVH builder, the traversal logic and the op-for-op parity with the oracle can be checked in a container without a GPU.
// Not part of librmcl_b200.so and never shipped.  One translation unit with every feature's *_emul.cu (included at the end), built
// with the host BVH build into one library by tests/native.py (emulator).
// Host code is compiled with -ffp-contract=off -mfma, so plain float ops are individually rounded exactly like the device's
// __fmul_rn/__fadd_rn and fmaf() is a true FMA.
#include "../../rmcl_b200/csrc/kernels.cuh"

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#define EMUL_API extern "C" __attribute__((visibility("default")))

// the product's host-built BVH of a mesh: the scene handle of every emul_* function that takes one
EMUL_API void* emul_scene_create(const float* verts, uint32_t nv, const uint32_t* faces, uint32_t nf, const char** err)
{
    B2BvhHost* b = new B2BvhHost();
    *err = "";
    if (b2_build_bvh8_host(verts, nv, faces, nf, b, err) != 0) { delete b; return nullptr; }
    return b;
}
EMUL_API void emul_scene_destroy(void* p) { if (p) { b2_free_bvh8_host((B2BvhHost*)p); delete (B2BvhHost*)p; } }
static BvhView view_of(const void* p)
{
    const B2BvhHost* b = (const B2BvhHost*)p;
    BvhView v; v.nodes = (const float4*)b->nodes; v.tris = (const float4*)b->tris;
    v.bx = b->abs_max[0]; v.by = b->abs_max[1]; v.bz = b->abs_max[2];
    return v;
}
// a distance field's view over host arrays, its grid as df_grid makes it
static DfieldView field_of(const float* lo, const float* hi, float h, float trunc, const uint32_t* index, const float* bricks)
{
    DfieldView f; uint64_t nb = 0;
    df_grid(lo, hi, h, trunc, &f, &nb);
    f.index = index; f.bricks = bricks;
    return f;
}

extern "C" {

__attribute__((visibility("default"))) void emul_scene_info(void* p, uint32_t* n_nodes, uint32_t* n_tris, uint32_t* depth, float* sah)
{
    const B2BvhHost* b = (const B2BvhHost*)p; *n_nodes = b->n_nodes; *n_tris = b->n_tris; *depth = b->max_depth; *sah = b->sah_cost;
}
// the host-built tree in the layout of b2_mesh_export_blob (header as b2_mesh_create leaves it for a host build: build mode 0, n_verts nv),
// so that one checker reads both; dst holds sizeof(B2BlobHeader) + n_nodes * 224 + n_tris * 48 bytes
__attribute__((visibility("default"))) void emul_export(void* p, uint32_t n_faces, uint32_t n_verts, uint8_t* dst)
{
    const B2BvhHost& b = *(const B2BvhHost*)p;
    B2BlobHeader hd; memset(&hd, 0, sizeof(hd));
    memcpy(hd.magic, "B2BVH8F", 8);
    hd.version = 2; hd.node_bytes = sizeof(B2Node8); hd.tri_bytes = sizeof(B2Tri); hd.n_nodes = b.n_nodes; hd.n_tris = b.n_tris; hd.n_faces = n_faces;
    hd.n_verts = n_verts; hd.max_depth = b.max_depth; hd.build_mode = 0; hd.sah = b.sah_cost;
    for (int k = 0; k < 3; k++) hd.abs_max[k] = b.abs_max[k];
    memcpy(dst, &hd, sizeof(hd));
    memcpy(dst + sizeof(hd), b.nodes, sizeof(B2Node8) * (size_t)b.n_nodes);
    memcpy(dst + sizeof(hd) + sizeof(B2Node8) * (size_t)b.n_nodes, b.tris, sizeof(B2Tri) * (size_t)b.n_tris);
}

__attribute__((visibility("default"))) void emul_intersect(void* sc, const float* origs, const float* dirs, uint32_t n, float tfar,
                                                           float* t_out, uint32_t* face_out, float* ng_out, uint8_t* hit_out, double* mean_nodes, double* mean_tris, uint32_t* per_ray_nodes, uint32_t* per_ray_tris)
{
    const BvhView bvh = view_of(sc);
    unsigned long long tn = 0, tt = 0;
    #pragma omp parallel for schedule(dynamic, 256) reduction(+ : tn, tt)
    for (int64_t i = 0; i < (int64_t)n; i++) {
        const RaySetup r = ray_setup(mk3(origs[3 * i], origs[3 * i + 1], origs[3 * i + 2]), mk3(dirs[3 * i], dirs[3 * i + 1], dirs[3 * i + 2]), bvh);
        HitRec h = trace_init(tfar);
        uint32_t nn = 0, nt = 0;
        trace_closest<true>(bvh, r, h, nn, nt);
        tn += nn; tt += nt;
        if (per_ray_nodes) per_ray_nodes[i] = nn;
        if (per_ray_tris) per_ray_tris[i] = nt;
        const bool hit = h.face != B2_NOFACE;
        if (t_out) t_out[i] = hit ? h.t : u2f(0x7f800000u);
        if (face_out) face_out[i] = h.face;
        if (hit_out) hit_out[i] = hit;
        if (ng_out) { V3 ng = mk3(0, 0, 0); if (hit) ng = tri_ng(bvh, h.tri); ng_out[3 * i] = ng.x; ng_out[3 * i + 1] = ng.y; ng_out[3 * i + 2] = ng.z; }
    }
    if (mean_nodes) *mean_nodes = (double)tn / (double)(n ? n : 1);
    if (mean_tris) *mean_tris = (double)tt / (double)(n ? n : 1);
}

__attribute__((visibility("default"))) void emul_find_opt(void* sc, const b2_transform* Tbm, const b2_transform* Tsb, uint32_t n, const float* origs, uint32_t n_origs,
                                                          const float* dirs, float range_min, float range_max, uint32_t sim_opts, float* pts, float* nrm, uint8_t* hits, uint32_t* faces, float* ranges);
__attribute__((visibility("default"))) void emul_find(void* sc, const b2_transform* Tbm, const b2_transform* Tsb, uint32_t n, const float* origs, uint32_t n_origs,
                                                      const float* dirs, float range_max, float* pts, float* nrm, uint8_t* hits, uint32_t* faces, float* ranges)
{
    emul_find_opt(sc, Tbm, Tsb, n, origs, n_origs, dirs, 0.f, range_max, 0u, pts, nrm, hits, faces, ranges);
}
__attribute__((visibility("default"))) void emul_find_opt(void* sc, const b2_transform* Tbm, const b2_transform* Tsb, uint32_t n, const float* origs, uint32_t n_origs,
                                                          const float* dirs, float range_min, float range_max, uint32_t sim_opts, float* pts, float* nrm, uint8_t* hits, uint32_t* faces, float* ranges)
{
    const BvhView bvh = view_of(sc);
    RayModel m; m.dirs = dirs; m.origs = origs; m.n_origs = n_origs; m.n = n; m.range_min = range_min; m.range_max = range_max; m.sim_opts = sim_opts;
    ModelBuffers out; out.pts = pts; out.nrm = nrm; out.hits = hits; out.faces = faces; out.ranges = ranges;
    const Tf Tsm = tf_mul(tf_from_pod(*Tbm), tf_from_pod(*Tsb));
    #pragma omp parallel for schedule(dynamic, 256)
    for (int64_t i = 0; i < (int64_t)n; i++) find_one(bvh, Tsm, m, (uint32_t)i, (uint64_t)i, out);
}

__attribute__((visibility("default"))) void emul_cpc_find(void* sc, const b2_transform* Tbm, const b2_transform* Tsb, uint32_t n, const float* dpts, float max_dist,
                                                          float* pts, float* nrm, uint8_t* hits, uint32_t* faces, float* dists, double* mean_nodes, double* mean_tris, uint32_t* per_nodes, uint32_t* per_tris)
{
    const BvhView bvh = view_of(sc);
    ModelBuffers out; out.pts = pts; out.nrm = nrm; out.hits = hits; out.faces = faces; out.ranges = dists;
    const Tf Tsm = tf_mul(tf_from_pod(*Tbm), tf_from_pod(*Tsb));
    const Tf Tms = tf_inv(Tsm);
    #pragma omp parallel for schedule(dynamic, 256)
    for (int64_t i = 0; i < (int64_t)n; i++) cpc_find_one(bvh, Tsm, Tms, dpts, max_dist, (uint32_t)i, out);
    if (mean_nodes || mean_tris) {
        unsigned long long tn = 0, tt = 0;
        #pragma omp parallel for schedule(dynamic, 256) reduction(+ : tn, tt)
        for (int64_t i = 0; i < (int64_t)n; i++) {
            CpBest b; uint32_t nn = 0, nt = 0;
            closest_point<true>(bvh, tf_apply(Tsm, mk3(dpts[3 * i], dpts[3 * i + 1], dpts[3 * i + 2])), b, nn, nt);
            tn += nn; tt += nt;
            if (per_nodes) per_nodes[i] = nn;
            if (per_tris) per_tris[i] = nt;
        }
        if (mean_nodes) *mean_nodes = (double)tn / (double)(n ? n : 1);
        if (mean_tris) *mean_tris = (double)tt / (double)(n ? n : 1);
    }
}

__attribute__((visibility("default"))) void emul_gladiator(uint32_t n_all, const b2_transform* poses, const b2_particle_attr* attrs, uint32_t first, uint32_t n_local,
                                                           const b2_gladiator_config* cfg, uint64_t seed, uint32_t step, b2_transform* poses_new, b2_particle_attr* attrs_new,
                                                           uint32_t* raw_out, float* normals_out)
{
    for (uint32_t i = 0; i < n_local; i++) {
        uint32_t raw; float N[6];
        gladiator_draws(seed, step, first + i, raw, N);
        if (raw_out) raw_out[i] = raw;
        if (normals_out) for (int k = 0; k < 6; k++) normals_out[6 * (size_t)i + k] = N[k];
        gladiator_one(poses, attrs, n_all, first + i, raw, N, *cfg, poses_new + i, attrs_new + i);
    }
}

__attribute__((visibility("default"))) void emul_segment(uint32_t n, const float* origs, uint32_t n_origs, const float* dirs, float range_min, float range_max, const float* rr,
                                                         const float* rs, const float* nsim, float min_scan, float min_map, float* out_scan, uint32_t* n_scan, float* out_map,
                                                         uint32_t* n_map, uint8_t* labels)
{
    RayModel m; m.dirs = dirs; m.origs = origs; m.n_origs = n_origs; m.n = n; m.range_min = range_min; m.range_max = range_max; m.width = n; m.height = 1; m.sim_opts = 0;
    uint32_t a = 0, b = 0;
    for (uint32_t i = 0; i < n; i++) {
        V3 p;
        const uint32_t l = segment_classify(m, i, rr[i], rs[i], mk3(nsim[3 * i], nsim[3 * i + 1], nsim[3 * i + 2]), min_scan, min_map, p);
        labels[i] = (uint8_t)l;
        if (l == 1u) { out_scan[3 * a] = p.x; out_scan[3 * a + 1] = p.y; out_scan[3 * a + 2] = p.z; a++; }
        if (l == 2u) { out_map[3 * b] = p.x; out_map[3 * b + 1] = p.y; out_map[3 * b + 2] = p.z; b++; }
    }
    *n_scan = a; *n_map = b;
}

__attribute__((visibility("default"))) void emul_pf_motion(void* sc, uint32_t n, b2_transform* poses, b2_particle_attr* attrs, const b2_transform* T, double forget_rate, int collide)
{
    const BvhView bvh = view_of(sc);
    for (uint32_t i = 0; i < n; i++) pf_motion_one(collide ? &bvh : nullptr, poses + i, attrs + i, tf_from_pod(*T), forget_rate);
}

// refit of the whole host-built tree with the product's per-node function: nodes in decreasing index order (children of a node have
// larger indices in both builders' layouts; returns -1 if that does not hold)
__attribute__((visibility("default"))) int emul_refit(void* p, const float* verts, uint32_t nv, const uint32_t* faces)
{
    B2BvhHost& b = *(B2BvhHost*)p;
    for (uint32_t t = 0; t < b.n_nodes; t++) if (b.nodes[t].imask() && b.nodes[t].child_base <= t) return -1;
    for (uint32_t t = b.n_nodes; t-- > 0;) bvh8_refit_node(t, b.nodes, b.tris, verts, faces);
    for (int k = 0; k < 3; k++) { float m = 0.f; for (uint32_t i = 0; i < nv; i++) m = fmaxf(m, fabsf(verts[3 * (size_t)i + k])); b.abs_max[k] = m; }
    return 0;
}

// sequential stand-in for k_p2l_reduce (same per-element math, FP64 sum form)
__attribute__((visibility("default"))) void emul_cross_statistics(const b2_transform* Tpre, uint32_t n, const float* dpts, const uint8_t* dmask, const float* mpts,
                                                                  const float* mnrm, const uint8_t* mmask, float max_dist, b2_cross_stats* out)
{
    P2LAcc acc; acc_zero(acc);
    const Tf T = tf_from_pod(*Tpre);
    for (uint32_t i = 0; i < n; i++) {
        if (!(dmask[i] > 0) || !(mmask[i] > 0)) continue;
        V3 D, M;
        if (p2l_pair(T, mk3(dpts[3 * i], dpts[3 * i + 1], dpts[3 * i + 2]), mk3(mpts[3 * i], mpts[3 * i + 1], mpts[3 * i + 2]),
                     mk3(mnrm[3 * i], mnrm[3 * i + 1], mnrm[3 * i + 2]), max_dist, D, M)) acc_add_pair(acc, D, M);
    }
    cs_store(out, acc_finalize(acc.v, acc.n));
}

__attribute__((visibility("default"))) void emul_umeyama(const b2_cross_stats* s, b2_transform* out) { memset(out, 0, sizeof(*out)); tf_store(out, umeyama_dev(cs_load(s))); }
__attribute__((visibility("default"))) void emul_cs_merge(const b2_cross_stats* a, const b2_cross_stats* b, b2_cross_stats* out) { cs_store(out, cs_merge(cs_load(a), cs_load(b))); }
__attribute__((visibility("default"))) void emul_cs_transform(const b2_transform* T, const b2_cross_stats* s, b2_cross_stats* out) { cs_store(out, cs_transform(tf_from_pod(*T), cs_load(s))); }

// The fused loop of the product (icp_loop.cuh: icp_tail with pre-composed frames, weighted multi-sensor merge) run sequentially on the CPU.
struct EmulSensor {
    uint32_t n, n_origs; const float* origs; const float* dirs; const float* dpts; const uint8_t* dmask;
    b2_transform Tbo, Tsb; float range_max, max_dist, pad0, pad1; double merge_weight;
};
__attribute__((visibility("default"))) void emul_micp_multi(void* sc, uint32_t ns, const EmulSensor* sen, const b2_transform* Tom, uint32_t iterations,
                                                            b2_transform* Tom_new, b2_transform* T_onew_oold, b2_cross_stats* Cmerged)
{
    IcpLaunch L; memset(&L, 0, sizeof(L));
    L.Tom = *Tom; L.n_sensors = ns; L.iterations = iterations;
    std::vector<std::vector<float>> mp(ns), mn(ns), mr(ns); std::vector<std::vector<uint8_t>> mh(ns); std::vector<std::vector<uint32_t>> mf(ns);
    for (uint32_t k = 0; k < ns; k++) {
        const EmulSensor& E = sen[k];
        IcpSensor& S = L.s[k];
        S.n = E.n; S.max_dist = E.max_dist; S.merge_weight = E.merge_weight;
        const Tf Tos = tf_mul(tf_from_pod(E.Tbo), tf_from_pod(E.Tsb));
        tf_store(&S.Tos, Tos); tf_store(&S.Tso, tf_inv(Tos)); quat_to_mat(Tos.R, S.Ros);
        mp[k].resize(3 * (size_t)E.n); mn[k].resize(3 * (size_t)E.n); mr[k].resize(E.n); mh[k].resize(E.n); mf[k].resize(E.n);
        b2_transform Tbm; memset(&Tbm, 0, sizeof(Tbm)); tf_store(&Tbm, tf_mul(tf_from_pod(*Tom), tf_from_pod(E.Tbo)));
        emul_find(sc, &Tbm, &E.Tsb, E.n, E.origs, E.n_origs, E.dirs, E.range_max, mp[k].data(), mn[k].data(), mh[k].data(), mf[k].data(), mr[k].data());
    }
    Tf T = tf_identity(); Tf Tpre[B2_MAX_SENSORS];
    for (uint32_t k = 0; k < ns; k++) Tpre[k] = tf_mul(tf_mul(tf_from_pod(L.s[k].Tso), tf_identity()), tf_from_pod(L.s[k].Tos));
    IcpResult res; memset(&res, 0, sizeof(res));
    res.Tom_new = *Tom; tf_store(&res.T_onew_oold, tf_identity());
    for (uint32_t it = 0; it < iterations; it++) {
        double sums[B2_MAX_SENSORS][B2_NACC + 1];
        for (uint32_t k = 0; k < ns; k++) {
            const EmulSensor& E = sen[k];
            P2LAcc acc; acc_zero(acc);
            for (uint32_t i = 0; i < E.n; i++) {
                if (!(E.dmask[i] > 0) || !(mh[k][i] > 0)) continue;
                V3 D, M;
                if (p2l_pair(Tpre[k], mk3(E.dpts[3 * i], E.dpts[3 * i + 1], E.dpts[3 * i + 2]), mk3(mp[k][3 * i], mp[k][3 * i + 1], mp[k][3 * i + 2]),
                             mk3(mn[k][3 * i], mn[k][3 * i + 1], mn[k][3 * i + 2]), E.max_dist, D, M)) acc_add_pair(acc, D, M);
            }
            for (int i = 0; i < B2_NACC; i++) sums[k][i] = acc.v[i];
            sums[k][B2_NACC] = (double)acc.n;
        }
        icp_tail(L, sums, T, Tpre, it + 1 == iterations, &res);
    }
    *Tom_new = res.Tom_new; *T_onew_oold = res.T_onew_oold; *Cmerged = res.Cmerged_o;
}

// whole correctOnce with the device functions: find_one + sequential reduce + icp_step (the reference's frame-algebra order, exec mode 0), or
// -- fast_tail -- the fused loop's icp_tail
__attribute__((visibility("default"))) void emul_correct_once(void* sc, uint32_t n, const float* origs, uint32_t n_origs, const float* dirs, float range_max,
                                                              const float* dpts, const uint8_t* dmask, const b2_transform* Tom, const b2_transform* Tbo, const b2_transform* Tsb,
                                                              uint32_t iterations, float max_dist, b2_transform* Tom_new, b2_transform* T_onew_oold, b2_cross_stats* Cmerged, int fast_tail)
{
    if (fast_tail) {
        EmulSensor E; memset(&E, 0, sizeof(E));
        E.n = n; E.n_origs = n_origs; E.origs = origs; E.dirs = dirs; E.dpts = dpts; E.dmask = dmask; E.Tbo = *Tbo; E.Tsb = *Tsb; E.range_max = range_max; E.max_dist = max_dist; E.merge_weight = 1.0;
        emul_micp_multi(sc, 1, &E, Tom, iterations, Tom_new, T_onew_oold, Cmerged);
        return;
    }
    std::vector<float> mp(3 * (size_t)n), mn(3 * (size_t)n), mr(n); std::vector<uint8_t> mh(n); std::vector<uint32_t> mf(n);
    IcpState st; memset(&st, 0, sizeof(st));
    st.Tom = *Tom; st.Tbo = *Tbo; st.Tsb = *Tsb; st.max_dist = max_dist;
    const Tf I = tf_identity();
    tf_store(&st.T_onew_oold, I);
    tf_store(&st.T_snew_sold, icp_pretransform(tf_load(&st.Tbo), tf_load(&st.Tsb), I));
    tf_store(&st.Tom_new, tf_load(&st.Tom));
    b2_transform Tbm; memset(&Tbm, 0, sizeof(Tbm)); tf_store(&Tbm, tf_mul(tf_load(&st.Tom), tf_load(&st.Tbo)));
    emul_find(sc, &Tbm, Tsb, n, origs, n_origs, dirs, range_max, mp.data(), mn.data(), mh.data(), mf.data(), mr.data());
    for (uint32_t it = 0; it < iterations; it++) {
        b2_cross_stats ss;
        emul_cross_statistics(&st.T_snew_sold, n, dpts, dmask, mp.data(), mn.data(), mh.data(), max_dist, &ss);
        icp_step(&st, cs_load(&ss));
    }
    *Tom_new = st.Tom_new; *T_onew_oold = st.T_onew_oold; *Cmerged = st.Cmerged_o;
}

__attribute__((visibility("default"))) void emul_pf_update(void* sc, uint32_t n_particles, const b2_transform* poses, b2_particle_attr* attrs, const b2_transform* Tsb,
                                                           uint32_t n_beams, const b2_range_meas* beams, const b2_pf_params* prm)
{
    const BvhView bvh = view_of(sc);
    float sigma_quad; double denom; pf_constants(*prm, sigma_quad, denom);
    std::vector<PfBeam> pb(n_beams);
    for (uint32_t j = 0; j < n_beams; j++) {
        const b2_range_meas& m = beams[j];
        pb[j].ox = m.orig.x; pb[j].oy = m.orig.y; pb[j].oz = m.orig.z; pb[j].dx = m.dir.x; pb[j].dy = m.dir.y; pb[j].dz = m.dir.z; pb[j].range = m.range; pb[j].slot = j;
    }
    #pragma omp parallel for schedule(dynamic, 64)
    for (int64_t p = 0; p < (int64_t)n_particles; p++) {
        std::vector<float> e(n_beams);
        const Tf Tsm = tf_mul(tf_load(poses + p), tf_from_pod(*Tsb));
        for (uint32_t j = 0; j < n_beams; j++) e[pb[j].slot] = prm->correspondence_type == 1 ? pf_eval_one<1>(bvh, Tsm, pb[j], *prm, sigma_quad, denom) : pf_eval_one<0>(bvh, Tsm, pb[j], *prm, sigma_quad, denom);
        b2_gaussian1d lk = attrs[p].likelihood;
        pf_merge(lk, e.data(), n_beams);
        attrs[p].likelihood = lk;
    }
}

}  // extern "C"

// the features' functions
#include "../chain_ref/progress_emul.cu"
#include "../dfield_ref/dfield_emul.cu"
#include "../micp_cov_ref/cov_emul.cu"
#include "../pc2_ref/pc2_emul.cu"
#include "../pc2_scan_ref/scan_emul.cu"
#include "../pf_cloud_ref/cloud_emul.cu"
#include "../pf_cluster_ref/cluster_emul.cu"
#include "../pf_estimate_ref/estimate_emul.cu"
#include "../pf_kld_ref/kld_emul.cu"
#include "../pf_recovery_ref/recovery_emul.cu"
#include "../pf_residual_ref/residual_emul.cu"
#include "../pf_stein_ref/stein_emul.cu"
#include "../pf_surface_ref/surface_emul.cu"
