// stein_emul.cu -- TEST HARNESS ONLY: the product's Stein-step functions (rmcl_b200/csrc/kernels.cuh: df_lookup_grad, stein_ref_index,
// stein_beam_term, stein_ref_entry, stein_bw_terms, stein_bandwidth, stein_pair, stein_move_one; b2_math.cuh: exp_f, atan2_d, sin_d, cos_d)
// compiled for the CPU over the product's host-built BVH.  The three kernels of an iteration run as host loops; the two grid reductions
// are restated in est_grid_reduce's order (one value per thread, blocks of 256: warp butterflies, the block's 8 warps in order, then in the
// last block lane l adds the partials of blocks l, l + 32, ... and a butterfly), so the results are the device's bits.  Built by
// tests/pf_stein_ref.py with the flags of tests/chain_ref (host code with -ffp-contract=off: plain ops rounded like __fmul_rn etc.).
#include "../../rmcl_b200/csrc/kernels.cuh"

#include <vector>

#define EMUL_API extern "C" __attribute__((visibility("default")))

static BvhView view_of(const void* p)
{
    const B2BvhHost* b = (const B2BvhHost*)p;
    BvhView v; v.nodes = (const float4*)b->nodes; v.tris = (const float4*)b->tris;
    v.bx = b->abs_max[0]; v.by = b->abs_max[1]; v.bz = b->abs_max[2];
    return v;
}
EMUL_API void* emul_stein_scene(const float* verts, uint32_t nv, const uint32_t* faces, uint32_t nf)
{
    B2BvhHost* b = new B2BvhHost();
    const char* err = "";
    if (b2_build_bvh8_host(verts, nv, faces, nf, b, &err) != 0) { delete b; return nullptr; }
    return b;
}
EMUL_API void emul_stein_scene_free(void* p)
{
    if (p) { b2_free_bvh8_host((B2BvhHost*)p); delete (B2BvhHost*)p; }
}
static DfieldView field_of(const float* lo, const float* hi, float h, float trunc, const uint32_t* index, const float* bricks)
{
    DfieldView f; uint64_t nb = 0;
    df_grid(lo, hi, h, trunc, &f, &nb);
    f.index = index; f.bricks = bricks;
    return f;
}

EMUL_API void emul_exp_f(const float* x, uint64_t n, float* out)
{
    #pragma omp parallel for schedule(static)
    for (int64_t i = 0; i < (int64_t)n; i++) out[i] = exp_f(x[i]);
}
// (float) atan2_d(y, x), (float) sin_d(a), (float) cos_d(a): the chart's and the step's library forms
EMUL_API void emul_lib_f(int which, const float* a, const float* b, uint64_t n, float* out)
{
    for (uint64_t i = 0; i < n; i++)
        out[i] = which == 0 ? (float)atan2_d((double)a[i], (double)b[i]) : which == 1 ? (float)sin_d((double)a[i]) : (float)cos_d((double)a[i]);
}
EMUL_API void emul_df_lookup_grad(const float* lo, const float* hi, float h, float trunc, const uint32_t* index, const float* bricks, const float* pts, uint32_t n,
                                  float* val, float* grad)
{
    const DfieldView f = field_of(lo, hi, h, trunc, index, bricks);
    #pragma omp parallel for schedule(static)
    for (int64_t i = 0; i < (int64_t)n; i++) {
        V3 g;
        val[i] = df_lookup_grad(f, mk3(pts[3 * i], pts[3 * i + 1], pts[3 * i + 2]), g);
        grad[3 * i] = g.x; grad[3 * i + 1] = g.y; grad[3 * i + 2] = g.z;
    }
}
EMUL_API void emul_stein_ref_index(uint32_t m, uint32_t n, uint32_t n_ref, uint64_t seed, uint32_t step, uint32_t it, uint32_t* out)
{
    for (uint32_t r = 0; r < m; r++) out[r] = stein_ref_index(r, n, n_ref, seed, step, it);
}
EMUL_API void emul_chart(const b2_transform* poses, uint32_t n, float* c3)
{
    for (uint32_t i = 0; i < n; i++) stein_chart(tf_from_pod(poses[i]), c3 + 3 * (size_t)i);
}

// est_grid_reduce over one value per particle (NV per particle, row-major), blocks of B2_STEIN_BLOCK
static void butterfly(double v[32])
{
    for (int o = 16; o > 0; o >>= 1) {
        double t[32];
        for (int l = 0; l < 32; l++) t[l] = v[l] + v[l ^ o];
        for (int l = 0; l < 32; l++) v[l] = t[l];
    }
}
static void grid_reduce(const std::vector<double>& per, int NV, uint32_t n, double* tot)
{
    const uint32_t G = (n + B2_STEIN_BLOCK - 1) / B2_STEIN_BLOCK;
    std::vector<double> part((size_t)G * NV);
    for (uint32_t b = 0; b < G; b++)
        for (int j = 0; j < NV; j++) {
            double sw[8];
            for (int w = 0; w < 8; w++) {
                double v[32];
                for (int l = 0; l < 32; l++) {
                    const uint64_t i = (uint64_t)b * B2_STEIN_BLOCK + 32u * w + l;
                    v[l] = i < n ? per[i * NV + j] : 0.0;
                }
                butterfly(v);
                sw[w] = v[0];
            }
            double a = sw[0];
            for (int w = 1; w < 8; w++) a = a + sw[w];
            part[(size_t)b * NV + j] = a;
        }
    for (int j = 0; j < NV; j++) {
        double v[32];
        for (uint32_t l = 0; l < 32; l++) {
            double a = 0.0;
            for (uint32_t b = l; b < G; b += 32) a = a + part[(size_t)b * NV + j];
            v[l] = a;
        }
        butterfly(v);
        tot[j] = v[0];
    }
}

// k_pf_stein_score: J's snapshot (m x 6 floats)
EMUL_API void emul_stein_score(const float* lo, const float* hi, float h, float trunc, const uint32_t* index, const float* bricks, const b2_transform* poses, uint32_t n,
                               uint32_t m, uint32_t n_ref, uint64_t seed, uint32_t step, uint32_t it, const b2_transform* Tsb_val, const b2_range_meas* beams,
                               uint32_t n_beams, float dist_sigma, float w_rand, SteinRef* snap)
{
    const DfieldView f = field_of(lo, hi, h, trunc, index, bricks);
    const Tf Tsb = tf_from_pod(*Tsb_val);
    const float sigma2 = mul(dist_sigma, dist_sigma);
    #pragma omp parallel for schedule(dynamic, 16)
    for (int64_t r = 0; r < (int64_t)m; r++) {
        std::vector<float> terms(3 * (size_t)n_beams);
        const Tf T = tf_from_pod(poses[stein_ref_index((uint32_t)r, n, n_ref, seed, step, it)]);
        const Tf Tsm = tf_mul(T, Tsb);
        for (uint32_t b = 0; b < n_beams; b++) {
            const b2_range_meas& q = beams[b];
            const PfBeam pb{q.orig.x, q.orig.y, q.orig.z, q.dir.x, q.dir.y, q.dir.z, q.range, b};
            stein_beam_term(f, Tsm, T.t, pb, sigma2, w_rand, terms.data() + 3 * (size_t)b);
        }
        snap[r] = stein_ref_entry(T, terms.data(), n_beams);
    }
}
// k_pf_stein_bandwidth: h (3 floats); tot_out (7 doubles, may be null) the reduced sums
EMUL_API void emul_stein_bandwidth(const b2_transform* poses, uint32_t n, uint32_t m, float floor_t, float floor_r, float* h, double* tot_out)
{
    std::vector<double> per((size_t)n * B2_STEIN_NBW, 0.0);
    for (uint32_t i = 0; i < n; i++) stein_bw_terms(tf_from_pod(poses[i]), per.data() + (size_t)i * B2_STEIN_NBW);
    double tot[B2_STEIN_NBW];
    grid_reduce(per, B2_STEIN_NBW, n, tot);
    stein_bandwidth(tot, std::pow((double)m, -1.0 / 7.0), floor_t, floor_r, h);
    if (tot_out) for (int j = 0; j < B2_STEIN_NBW; j++) tot_out[j] = tot[j];
}
// the pair sums of charts ci (n x 3) over the snapshot: acc (n x 3); a reference with x = NaN is skipped, as in k_pf_stein_move
EMUL_API void emul_stein_pairs(const float* ci, uint32_t n, const SteinRef* snap, uint32_t m, const float* h, float* acc)
{
    float ih2[3];
    stein_inv_h2(h, ih2);
    #pragma omp parallel for schedule(static)
    for (int64_t i = 0; i < (int64_t)n; i++) {
        float a[3] = {0.0f, 0.0f, 0.0f};
        for (uint32_t j = 0; j < m; j++) if (snap[j].x == snap[j].x) stein_pair(ci + 3 * i, snap[j], ih2, a);
        acc[3 * i] = a[0]; acc[3 * i + 1] = a[1]; acc[3 * i + 2] = a[2];
    }
}
// k_pf_stein_move: poses in place, v (n x 3) the RMSProp state; rec's n_blocked is added to, its RMS steps are set
EMUL_API void emul_stein_move(void* scene, b2_transform* poses, uint32_t n, const SteinRef* snap, uint32_t m, uint32_t it, float step_t, float step_r, float* v,
                              const float* h, b2_stein_result* rec)
{
    const BvhView bvh = view_of(scene);
    float ih2[3];
    stein_inv_h2(h, ih2);
    std::vector<double> per((size_t)n * B2_STEIN_NMV, 0.0);
    uint64_t blocked = 0;
    #pragma omp parallel for schedule(static) reduction(+ : blocked)
    for (int64_t i = 0; i < (int64_t)n; i++) {
        const Tf T = tf_from_pod(poses[i]);
        float ci[3];
        stein_chart(T, ci);
        if (!stein_finite3(ci)) continue;
        float a[3] = {0.0f, 0.0f, 0.0f};
        for (uint32_t j = 0; j < m; j++) if (snap[j].x == snap[j].x) stein_pair(ci, snap[j], ih2, a);
        blocked += stein_move_one(bvh, poses + i, T, v + 3 * i, a, m, it, step_t, step_r, per.data() + (size_t)i * B2_STEIN_NMV);
    }
    double tot[B2_STEIN_NMV];
    grid_reduce(per, B2_STEIN_NMV, n, tot);
    rec->n_blocked += (uint32_t)blocked;
    rec->rms_step_t = tot[0] > 0.0 ? (float)std::sqrt(tot[1] / tot[0]) : 0.0f;
    rec->rms_step_r = tot[0] > 0.0 ? (float)std::sqrt(tot[2] / tot[0]) : 0.0f;
}
// b2_pf_stein_update as a whole: poses in place, the result record
EMUL_API void emul_stein_update(void* scene, const float* lo, const float* hi, float h, float trunc, const uint32_t* index, const float* bricks, b2_transform* poses,
                                uint32_t n, const b2_transform* Tsb, const b2_range_meas* beams, uint32_t n_beams, float dist_sigma, const b2_stein_config* cfg,
                                uint64_t seed, uint32_t step, b2_stein_result* rec)
{
    *rec = b2_stein_result{};
    if (n == 0 || cfg->iterations == 0) return;
    const uint32_t m = (cfg->n_ref == 0 || cfg->n_ref >= n) ? n : cfg->n_ref;
    std::vector<SteinRef> snap(m);
    std::vector<float> v(3 * (size_t)n, 0.0f);
    for (uint32_t it = 0; it < cfg->iterations; it++) {
        emul_stein_score(lo, hi, h, trunc, index, bricks, poses, n, m, cfg->n_ref, seed, step, it, Tsb, beams, n_beams, dist_sigma, cfg->w_rand, snap.data());
        emul_stein_bandwidth(poses, n, m, cfg->min_bandwidth_t, cfg->min_bandwidth_r, rec->bandwidth, nullptr);
        rec->n_ref = m;
        emul_stein_move(scene, poses, n, snap.data(), m, it, cfg->step_t, cfg->step_r, v.data(), rec->bandwidth, rec);
    }
}
