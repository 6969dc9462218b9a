/*
 * oracle.c -- CPU restatement of RMCL's ray-casting-correspondence hot path (see oracle.h).
 *
 * TEST INFRASTRUCTURE ONLY; PARITY UNPINNED (reference has no tests; rmagine/Embree not vendored).
 *
 * Build: gcc -O2 -fopenmp -ffp-contract=off -mavx2 -mfma -shared -fPIC   (see oracle/Makefile)
 * -ffp-contract=off is REQUIRED: every float op below is individually rounded unless fmaf() is written out.
 *
 * Arithmetic conventions
 *  - "rmagine-level" math (quaternion products, Transform algebra, dot products in P2L / PF error) is written
 *    as plain left-to-right mul/add, the way the reference's inline C++ evaluates without FMA contraction.
 *  - The ray/triangle kernel stands in for Embree's closest hit.  It is a Moeller-Trumbore test in scaled
 *    (division-free) form with explicit fmaf() chains, plus a VALIDATION step that makes the hit set independent of
 *    any acceleration structure.  With the monotone slab formula F (below) giving (tn, tf) for a box, define
 *        P1(box, tau): tn <= fl(tau * C1)      C1 = 1 + 2^-14
 *        P2(box, tau): tf >= fl(tau * C2)      C2 = 1 - 2^-14
 *    A candidate t > 0 is a HIT iff P1 and P2 hold for the triangle's own AABB (min/max of its vertices).
 *    A node box B may be skipped only if NOT V(B, tbest), V := tn <= fl(tbest*C1) && tf >= max(0, fl(tn*C3)), C3 = 1 - 2^-12.
 *    V is monotone in the box and implied by the existence of a HIT with t <= tbest inside it, so every BVH whose
 *    boxes contain the triangle AABBs and whose box test is at least as permissive as V returns exactly
 *    argmin (t, face id) over all HITs -- the same answer as the brute-force loop.
 */
#include "oracle.h"

#include <math.h>
#include <stdlib.h>
#include <string.h>
#include <float.h>
#ifdef _OPENMP
#include <omp.h>
#endif

#ifndef M_PI
#define M_PI 3.14159265358979323846
#endif

/* ------------------------------------------------------------------------------------------------ */
/* small vector helpers (plain ops)                                                                   */
/* ------------------------------------------------------------------------------------------------ */
static inline orc_vec3 v3(float x, float y, float z) { orc_vec3 r = {x, y, z}; return r; }
static inline orc_vec3 v3_add(orc_vec3 a, orc_vec3 b) { return v3(a.x + b.x, a.y + b.y, a.z + b.z); }
static inline orc_vec3 v3_sub(orc_vec3 a, orc_vec3 b) { return v3(a.x - b.x, a.y - b.y, a.z - b.z); }
static inline orc_vec3 v3_scale(orc_vec3 a, float s) { return v3(a.x * s, a.y * s, a.z * s); }
static inline orc_vec3 v3_neg(orc_vec3 a) { return v3(-a.x, -a.y, -a.z); }
/* rm::Vector3::dot : x*o.x + y*o.y + z*o.z */
static inline float v3_dot(orc_vec3 a, orc_vec3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
static inline float v3_l2norm(orc_vec3 a) { return sqrtf(a.x * a.x + a.y * a.y + a.z * a.z); }
/* rm::Vector3::normalize : component-wise division by l2norm */
static inline orc_vec3 v3_normalize(orc_vec3 a) { float n = v3_l2norm(a); return v3(a.x / n, a.y / n, a.z / n); }

/* Hamilton product, SURVEY.md A.1 */
static inline orc_quat q_mul(orc_quat a, orc_quat b)
{
    orc_quat r;
    r.w = a.w * b.w - a.x * b.x - a.y * b.y - a.z * b.z;
    r.x = a.w * b.x + a.x * b.w + a.y * b.z - a.z * b.y;
    r.y = a.w * b.y - a.x * b.z + a.y * b.w + a.z * b.x;
    r.z = a.w * b.z + a.x * b.y - a.y * b.x + a.z * b.w;
    return r;
}
static inline orc_quat q_conj(orc_quat a) { orc_quat r = {-a.x, -a.y, -a.z, a.w}; return r; }
/* q * v = vec(q (v,0) q^-1) */
static inline orc_vec3 q_rot(orc_quat q, orc_vec3 v)
{
    orc_quat p = {v.x, v.y, v.z, 0.0f};
    orc_quat r = q_mul(q_mul(q, p), q_conj(q));
    return v3(r.x, r.y, r.z);
}
static inline orc_quat q_normalize(orc_quat q)
{
    float n = sqrtf(q.x * q.x + q.y * q.y + q.z * q.z + q.w * q.w);
    orc_quat r = {q.x / n, q.y / n, q.z / n, q.w / n};
    return r;
}
static inline orc_transform T_identity(void)
{
    orc_transform T; T.R.x = T.R.y = T.R.z = 0.0f; T.R.w = 1.0f; T.t = v3(0, 0, 0); T.stamp = 0; return T;
}
/* T1*T2 = {R1R2, R1 t2 + t1} */
static inline orc_transform T_mul(orc_transform a, orc_transform b)
{
    orc_transform r; r.R = q_mul(a.R, b.R); r.t = v3_add(q_rot(a.R, b.t), a.t); r.stamp = a.stamp; return r;
}
/* ~T = {R^-1, -(R^-1 t)} */
static inline orc_transform T_inv(orc_transform a)
{
    orc_transform r; r.R = q_conj(a.R); r.t = v3_neg(q_rot(r.R, a.t)); r.stamp = a.stamp; return r;
}
static inline orc_vec3 T_apply(orc_transform T, orc_vec3 p) { return v3_add(q_rot(T.R, p), T.t); }

void orc_transform_mul(const orc_transform* a, const orc_transform* b, orc_transform* out) { *out = T_mul(*a, *b); }
void orc_transform_inv(const orc_transform* a, orc_transform* out) { *out = T_inv(*a); }
void orc_transform_point(const orc_transform* T, const float p[3], float out[3])
{
    orc_vec3 r = T_apply(*T, v3(p[0], p[1], p[2])); out[0] = r.x; out[1] = r.y; out[2] = r.z;
}
void orc_quat_rotate(const orc_quat* q, const float v[3], float out[3])
{
    orc_vec3 r = q_rot(*q, v3(v[0], v[1], v[2])); out[0] = r.x; out[1] = r.y; out[2] = r.z;
}

/* ------------------------------------------------------------------------------------------------ */
/* scene: triangle soup + binned-SAH BVH2                                                             */
/* ------------------------------------------------------------------------------------------------ */
typedef struct { float lo[3], hi[3]; uint32_t left_first; uint32_t count; } bvh_node;   /* count>0: leaf */

struct orc_scene {
    uint32_t nv, nf;
    float*    verts;     /* nv*3 */
    uint32_t* faces;     /* nf*3 */
    uint32_t* prim;      /* nf permutation (leaf order) */
    bvh_node* nodes; uint32_t n_nodes;
};

static inline float fmin3(float a, float b, float c) { float m = a < b ? a : b; return m < c ? m : c; }
static inline float fmax3(float a, float b, float c) { float m = a > b ? a : b; return m > c ? m : c; }

static void tri_bounds(const orc_scene* s, uint32_t f, float lo[3], float hi[3])
{
    const float* a = s->verts + 3 * (size_t)s->faces[3 * (size_t)f + 0];
    const float* b = s->verts + 3 * (size_t)s->faces[3 * (size_t)f + 1];
    const float* c = s->verts + 3 * (size_t)s->faces[3 * (size_t)f + 2];
    for (int k = 0; k < 3; k++) { lo[k] = fmin3(a[k], b[k], c[k]); hi[k] = fmax3(a[k], b[k], c[k]); }
}

#define ORC_BINS 16
#define ORC_LEAF_MAX 4

typedef struct { float lo[3], hi[3]; float c[3]; } prim_info;

static float half_area(const float lo[3], const float hi[3])
{
    float dx = hi[0] - lo[0], dy = hi[1] - lo[1], dz = hi[2] - lo[2];
    return dx * dy + dy * dz + dz * dx;
}

static void build_rec(orc_scene* s, const prim_info* pi, uint32_t node_idx, uint32_t first, uint32_t count)
{
    bvh_node* nd = &s->nodes[node_idx];
    float clo[3] = {FLT_MAX, FLT_MAX, FLT_MAX}, chi[3] = {-FLT_MAX, -FLT_MAX, -FLT_MAX};
    for (int k = 0; k < 3; k++) { nd->lo[k] = FLT_MAX; nd->hi[k] = -FLT_MAX; }
    for (uint32_t i = first; i < first + count; i++) {
        const prim_info* p = &pi[s->prim[i]];
        for (int k = 0; k < 3; k++) {
            if (p->lo[k] < nd->lo[k]) nd->lo[k] = p->lo[k];
            if (p->hi[k] > nd->hi[k]) nd->hi[k] = p->hi[k];
            if (p->c[k] < clo[k]) clo[k] = p->c[k];
            if (p->c[k] > chi[k]) chi[k] = p->c[k];
        }
    }
    if (count <= 2) { nd->left_first = first; nd->count = count; return; }

    /* binned SAH over the 3 axes */
    float best_cost = FLT_MAX; int best_axis = -1; int best_split = 0;
    for (int ax = 0; ax < 3; ax++) {
        float ext = chi[ax] - clo[ax];
        if (!(ext > 0.0f)) continue;
        float blo[ORC_BINS][3], bhi[ORC_BINS][3]; uint32_t bcnt[ORC_BINS];
        for (int b = 0; b < ORC_BINS; b++) { bcnt[b] = 0; for (int k = 0; k < 3; k++) { blo[b][k] = FLT_MAX; bhi[b][k] = -FLT_MAX; } }
        float scale = (float)ORC_BINS / ext;
        for (uint32_t i = first; i < first + count; i++) {
            const prim_info* p = &pi[s->prim[i]];
            int b = (int)((p->c[ax] - clo[ax]) * scale); if (b >= ORC_BINS) b = ORC_BINS - 1; if (b < 0) b = 0;
            bcnt[b]++;
            for (int k = 0; k < 3; k++) { if (p->lo[k] < blo[b][k]) blo[b][k] = p->lo[k]; if (p->hi[k] > bhi[b][k]) bhi[b][k] = p->hi[k]; }
        }
        float ralo[ORC_BINS][3], rahi[ORC_BINS][3]; uint32_t rcnt[ORC_BINS];
        float lo[3] = {FLT_MAX, FLT_MAX, FLT_MAX}, hi[3] = {-FLT_MAX, -FLT_MAX, -FLT_MAX}; uint32_t c = 0;
        for (int b = ORC_BINS - 1; b > 0; b--) {
            c += bcnt[b];
            for (int k = 0; k < 3; k++) { if (blo[b][k] < lo[k]) lo[k] = blo[b][k]; if (bhi[b][k] > hi[k]) hi[k] = bhi[b][k]; }
            rcnt[b] = c; for (int k = 0; k < 3; k++) { ralo[b][k] = lo[k]; rahi[b][k] = hi[k]; }
        }
        for (int k = 0; k < 3; k++) { lo[k] = FLT_MAX; hi[k] = -FLT_MAX; } c = 0;
        for (int b = 0; b < ORC_BINS - 1; b++) {
            c += bcnt[b];
            for (int k = 0; k < 3; k++) { if (blo[b][k] < lo[k]) lo[k] = blo[b][k]; if (bhi[b][k] > hi[k]) hi[k] = bhi[b][k]; }
            if (c == 0 || rcnt[b + 1] == 0) continue;
            float cost = half_area(lo, hi) * (float)c + half_area(ralo[b + 1], rahi[b + 1]) * (float)rcnt[b + 1];
            if (cost < best_cost) { best_cost = cost; best_axis = ax; best_split = b + 1; }
        }
    }
    uint32_t mid;
    if (best_axis < 0) {
        if (count <= ORC_LEAF_MAX) { nd->left_first = first; nd->count = count; return; }
        mid = first + count / 2;            /* all centroids coincide: split by index */
    } else {
        float leaf_cost = half_area(nd->lo, nd->hi) * (float)count;
        if (count <= ORC_LEAF_MAX && leaf_cost <= best_cost + half_area(nd->lo, nd->hi)) { nd->left_first = first; nd->count = count; return; }
        float ext = chi[best_axis] - clo[best_axis]; float scale = (float)ORC_BINS / ext;
        uint32_t i = first, j = first + count;
        while (i < j) {
            const prim_info* p = &pi[s->prim[i]];
            int b = (int)((p->c[best_axis] - clo[best_axis]) * scale); if (b >= ORC_BINS) b = ORC_BINS - 1; if (b < 0) b = 0;
            if (b < best_split) i++; else { j--; uint32_t t = s->prim[i]; s->prim[i] = s->prim[j]; s->prim[j] = t; }
        }
        mid = i;
        if (mid == first || mid == first + count) mid = first + count / 2;
    }
    uint32_t left;
    #pragma omp atomic capture
    { left = s->n_nodes; s->n_nodes += 2; }
    nd->left_first = left; nd->count = 0;
    uint32_t lcount = mid - first, rcount = count - lcount;
    if (count > 20000) {
        #pragma omp task
        build_rec(s, pi, left, first, lcount);
        #pragma omp task
        build_rec(s, pi, left + 1, mid, rcount);
        #pragma omp taskwait
    } else {
        build_rec(s, pi, left, first, lcount);
        build_rec(s, pi, left + 1, mid, rcount);
    }
}

orc_scene* orc_scene_create(const float* verts_xyz, uint32_t nv, const uint32_t* faces_ijk, uint32_t nf)
{
    orc_scene* s = (orc_scene*)calloc(1, sizeof(orc_scene));
    s->nv = nv; s->nf = nf;
    s->verts = (float*)malloc(sizeof(float) * 3 * (size_t)(nv ? nv : 1));
    s->faces = (uint32_t*)malloc(sizeof(uint32_t) * 3 * (size_t)(nf ? nf : 1));
    memcpy(s->verts, verts_xyz, sizeof(float) * 3 * (size_t)nv);
    memcpy(s->faces, faces_ijk, sizeof(uint32_t) * 3 * (size_t)nf);
    s->prim = (uint32_t*)malloc(sizeof(uint32_t) * (size_t)(nf ? nf : 1));
    s->nodes = (bvh_node*)malloc(sizeof(bvh_node) * (size_t)(2 * (size_t)nf + 2));
    s->n_nodes = 1;
    if (nf == 0) { s->nodes[0].count = 0; s->nodes[0].left_first = 0; s->n_nodes = 0; return s; }
    prim_info* pi = (prim_info*)malloc(sizeof(prim_info) * (size_t)nf);
    for (uint32_t f = 0; f < nf; f++) {
        s->prim[f] = f; tri_bounds(s, f, pi[f].lo, pi[f].hi);
        for (int k = 0; k < 3; k++) pi[f].c[k] = 0.5f * (pi[f].lo[k] + pi[f].hi[k]);
    }
    #pragma omp parallel
    {
        #pragma omp single
        build_rec(s, pi, 0, 0, nf);
    }
    free(pi);
    return s;
}

void orc_scene_destroy(orc_scene* s)
{
    if (!s) return;
    free(s->verts); free(s->faces); free(s->prim); free(s->nodes); free(s);
}
uint32_t orc_scene_num_faces(const orc_scene* s) { return s->nf; }

/* ------------------------------------------------------------------------------------------------ */
/* ray / box / triangle                                                                               */
/* ------------------------------------------------------------------------------------------------ */
typedef struct { float o[3], d[3], idir[3]; } ray_t;

/* slab formula F: idir_k = 1/(|d_k| < 1e-18 ? copysign(1e-18, d_k) : d_k); t = fl(fl(plane - o) * idir). Monotone in the box. */
static inline void ray_setup(ray_t* r, const float o[3], const float d[3])
{
    for (int k = 0; k < 3; k++) {
        r->o[k] = o[k]; r->d[k] = d[k];
        float dk = d[k];
        if (fabsf(dk) < 1e-18f) dk = copysignf(1e-18f, dk);
        r->idir[k] = 1.0f / dk;
    }
}
static inline void slab_F(const ray_t* r, const float lo[3], const float hi[3], float* tn, float* tf)
{
    float n = -INFINITY, f = INFINITY;
    for (int k = 0; k < 3; k++) {
        float t0 = (lo[k] - r->o[k]) * r->idir[k];
        float t1 = (hi[k] - r->o[k]) * r->idir[k];
        float a = t0 < t1 ? t0 : t1, b = t0 < t1 ? t1 : t0;
        if (a > n) n = a;
        if (b < f) f = b;
    }
    *tn = n; *tf = f;
}

#define ORC_C1 1.00006103515625f      /* 1 + 2^-14 */
#define ORC_C2 0.99993896484375f      /* 1 - 2^-14 */
#define ORC_C3 0.999755859375f        /* 1 - 2^-12 */
static inline int visit_V(float tn, float tf, float tbest)
{
    float lim = tn * ORC_C3; if (!(lim > 0.0f)) lim = 0.0f;
    return (tn <= tbest * ORC_C1) && (tf >= lim);
}

static inline float dot_fma(const float a[3], const float b[3]) { return fmaf(a[2], b[2], fmaf(a[1], b[1], a[0] * b[0])); }
static inline void cross_fma(const float a[3], const float b[3], float c[3])
{
    c[0] = fmaf(a[1], b[2], -(a[2] * b[1]));
    c[1] = fmaf(a[2], b[0], -(a[0] * b[2]));
    c[2] = fmaf(a[0], b[1], -(a[1] * b[0]));
}

/* returns 1 and t if the ray hits triangle f with t in (0, +inf) and passes validation; caller applies the tfar / tie rule */
static inline int tri_hit(const orc_scene* s, const ray_t* r, uint32_t f, float* t_out)
{
    const float* v0 = s->verts + 3 * (size_t)s->faces[3 * (size_t)f + 0];
    const float* v1 = s->verts + 3 * (size_t)s->faces[3 * (size_t)f + 1];
    const float* v2 = s->verts + 3 * (size_t)s->faces[3 * (size_t)f + 2];
    float e1[3] = {v1[0] - v0[0], v1[1] - v0[1], v1[2] - v0[2]};
    float e2[3] = {v2[0] - v0[0], v2[1] - v0[1], v2[2] - v0[2]};
    float pv[3]; cross_fma(r->d, e2, pv);
    float det = dot_fma(e1, pv);
    if (det == 0.0f || det != det) return 0;
    float tv[3] = {r->o[0] - v0[0], r->o[1] - v0[1], r->o[2] - v0[2]};
    float U = dot_fma(tv, pv);
    float qv[3]; cross_fma(tv, e1, qv);
    float V = dot_fma(r->d, qv);
    float T = dot_fma(e2, qv);
    if (det > 0.0f) { if (!(U >= 0.0f && V >= 0.0f && U + V <= det && T > 0.0f)) return 0; }
    else            { if (!(U <= 0.0f && V <= 0.0f && U + V >= det && T < 0.0f)) return 0; }
    float t = T / det;
    /* validation against the triangle's own AABB with formula F */
    float lo[3], hi[3];
    for (int k = 0; k < 3; k++) { lo[k] = fmin3(v0[k], v1[k], v2[k]); hi[k] = fmax3(v0[k], v1[k], v2[k]); }
    float tn, tf; slab_F(r, lo, hi, &tn, &tf);
    if (!(tn <= t * ORC_C1 && tf >= t * ORC_C2)) return 0;
    *t_out = t;
    return 1;
}

static inline void tri_ng(const orc_scene* s, uint32_t f, float ng[3])
{
    const float* v0 = s->verts + 3 * (size_t)s->faces[3 * (size_t)f + 0];
    const float* v1 = s->verts + 3 * (size_t)s->faces[3 * (size_t)f + 1];
    const float* v2 = s->verts + 3 * (size_t)s->faces[3 * (size_t)f + 2];
    float e1[3] = {v1[0] - v0[0], v1[1] - v0[1], v1[2] - v0[2]};
    float e2[3] = {v2[0] - v0[0], v2[1] - v0[1], v2[2] - v0[2]};
    cross_fma(e1, e2, ng);
}

#define ORC_NOFACE 0xFFFFFFFFu

static int closest_hit(const orc_scene* s, const ray_t* r, float tfar, int brute, float* t_best_out, uint32_t* face_out)
{
    float tbest = tfar; uint32_t fbest = ORC_NOFACE;
    if (s->nf == 0) return 0;
    if (brute) {
        for (uint32_t f = 0; f < s->nf; f++) {
            float t;
            if (tri_hit(s, r, f, &t) && (t < tbest || (t == tbest && f < fbest))) { tbest = t; fbest = f; }
        }
    } else {
        uint32_t stack[128]; int sp = 0; stack[sp++] = 0;
        while (sp) {
            const bvh_node* nd = &s->nodes[stack[--sp]];
            float tn, tf; slab_F(r, nd->lo, nd->hi, &tn, &tf);
            if (!visit_V(tn, tf, tbest)) continue;
            if (nd->count) {
                for (uint32_t i = 0; i < nd->count; i++) {
                    uint32_t f = s->prim[nd->left_first + i]; float t;
                    if (tri_hit(s, r, f, &t) && (t < tbest || (t == tbest && f < fbest))) { tbest = t; fbest = f; }
                }
            } else {
                /* push far child first; ordering only affects speed */
                const bvh_node* l = &s->nodes[nd->left_first]; const bvh_node* rr = l + 1;
                float ln, lf, rn, rf; slab_F(r, l->lo, l->hi, &ln, &lf); slab_F(r, rr->lo, rr->hi, &rn, &rf);
                if (sp + 2 > 128) continue; /* cannot happen for sane trees (depth << 128) */
                if (ln <= rn) { stack[sp++] = nd->left_first + 1; stack[sp++] = nd->left_first; }
                else          { stack[sp++] = nd->left_first;     stack[sp++] = nd->left_first + 1; }
            }
        }
    }
    if (fbest == ORC_NOFACE) return 0;
    *t_best_out = tbest; *face_out = fbest;
    return 1;
}

int orc_intersect(const orc_scene* s, const float o[3], const float d[3], float tfar, int brute,
                  float* t_out, uint32_t* face_out, float ng_out[3])
{
    ray_t r; ray_setup(&r, o, d);
    float t; uint32_t f;
    if (!closest_hit(s, &r, tfar, brute, &t, &f)) return 0;
    if (t_out) *t_out = t;
    if (face_out) *face_out = f;
    if (ng_out) tri_ng(s, f, ng_out);
    return 1;
}

void orc_intersect_batch(const orc_scene* s, uint32_t n, const float* origs, const float* dirs, float tfar, int brute,
                         float* t_out, uint32_t* face_out, float* ng_out, uint8_t* hit_out)
{
    #pragma omp parallel for schedule(dynamic, 256)
    for (int64_t i = 0; i < (int64_t)n; i++) {
        float t = 0.0f; uint32_t f = ORC_NOFACE; float ng[3] = {0, 0, 0};
        int h = orc_intersect(s, origs + 3 * i, dirs + 3 * i, tfar, brute, &t, &f, ng);
        if (t_out) t_out[i] = h ? t : INFINITY;
        if (face_out) face_out[i] = f;
        if (ng_out) { ng_out[3 * i] = ng[0]; ng_out[3 * i + 1] = ng[1]; ng_out[3 * i + 2] = ng[2]; }
        if (hit_out) hit_out[i] = (uint8_t)h;
    }
}

/* ------------------------------------------------------------------------------------------------ */
/* sensor models                                                                                      */
/* ------------------------------------------------------------------------------------------------ */
void orc_spherical_dirs(float phi_min, float phi_inc, uint32_t phi_n, float theta_min, float theta_inc, uint32_t theta_n, float* dirs_out)
{
    for (uint32_t vid = 0; vid < phi_n; vid++) {
        float phi = phi_min + (float)vid * phi_inc;
        for (uint32_t hid = 0; hid < theta_n; hid++) {
            float theta = theta_min + (float)hid * theta_inc;
            float* d = dirs_out + 3 * ((size_t)vid * theta_n + hid);     /* getBufferId = vid*W + hid */
            d[0] = cosf(phi) * cosf(theta);
            d[1] = cosf(phi) * sinf(theta);
            d[2] = sinf(phi);
        }
    }
}

void orc_pinhole_dirs(uint32_t width, uint32_t height, float fx, float fy, float cx, float cy, float* dirs_out)
{
    for (uint32_t vid = 0; vid < height; vid++)
        for (uint32_t hid = 0; hid < width; hid++) {
            float px = ((float)hid - cx) / fx;
            float py = ((float)vid - cy) / fy;
            orc_vec3 o = v3_normalize(v3(px, py, 1.0f));                  /* optical frame */
            float* d = dirs_out + 3 * ((size_t)vid * width + hid);
            d[0] = o.z; d[1] = -o.x; d[2] = -o.y;                         /* x forward, y left, z up */
        }
}

/* ------------------------------------------------------------------------------------------------ */
/* simulate == find                                                                                   */
/* ------------------------------------------------------------------------------------------------ */
static inline void put3(float* dst, size_t i, orc_vec3 v) { if (dst) { dst[3 * i] = v.x; dst[3 * i + 1] = v.y; dst[3 * i + 2] = v.z; } }

void orc_simulate_opt(const orc_scene* s, const orc_transform* Tbm, const orc_transform* Tsb,
                      uint32_t n, const float* origs_s, uint32_t n_origs, const float* dirs_s, float range_min, float range_max, const orc_sim_options* opt,
                      float* points, float* normals, uint8_t* hits, uint32_t* face_ids, float* ranges)
{
    const orc_transform Tsm = T_mul(*Tbm, *Tsb);
    const orc_transform Tms = T_inv(Tsm);
    const float tfar = (opt && opt->tfar_mode == 1) ? INFINITY : range_max;                 /* SURVEY A.3: tfar = range.max (default) vs +inf */
    const int cull_min = opt && opt->min_mode == 1;                                          /*             hits with t < range.min kept (default) vs dropped */
    const float fill = (opt && opt->miss_fill == 1) ? 0.0f : NAN;                            /*             miss fill NaN (default) vs zeros */
    #pragma omp parallel for schedule(dynamic, 256)
    for (int64_t i = 0; i < (int64_t)n; i++) {
        const float* op = origs_s + 3 * (size_t)(n_origs == 1 ? 0 : i);
        const orc_vec3 orig_s = v3(op[0], op[1], op[2]);
        const orc_vec3 dir_s = v3(dirs_s[3 * i], dirs_s[3 * i + 1], dirs_s[3 * i + 2]);
        const orc_vec3 orig_m = T_apply(Tsm, orig_s);
        const orc_vec3 dir_m = q_rot(Tsm.R, dir_s);
        float o[3] = {orig_m.x, orig_m.y, orig_m.z}, d[3] = {dir_m.x, dir_m.y, dir_m.z};
        ray_t r; ray_setup(&r, o, d);
        float t; uint32_t f;
        int hit = closest_hit(s, &r, tfar, 0, &t, &f);
        if (hit && cull_min && t < range_min) hit = 0;          /* the CLOSEST hit is below range.min: the ray reports a miss (nothing behind it is searched) */
        if (hit) {
            float ng[3]; tri_ng(s, f, ng);
            orc_vec3 p = v3_add(v3_scale(dir_s, t), orig_s);
            orc_vec3 nm = v3_normalize(v3(ng[0], ng[1], ng[2]));
            orc_vec3 ns = q_rot(Tms.R, nm);
            if (v3_dot(dir_s, ns) > 0.0f) ns = v3_neg(ns);
            ns = v3_normalize(ns);
            put3(points, (size_t)i, p); put3(normals, (size_t)i, ns);
            if (hits) hits[i] = 1;
            if (face_ids) face_ids[i] = f;
            if (ranges) ranges[i] = t;
        } else {
            orc_vec3 fv = v3(fill, fill, fill);
            put3(points, (size_t)i, fv); put3(normals, (size_t)i, fv);
            if (hits) hits[i] = 0;
            if (face_ids) face_ids[i] = ORC_NOFACE;
            if (ranges) ranges[i] = range_max + 1.0f;
        }
    }
}

void orc_simulate(const orc_scene* s, const orc_transform* Tbm, const orc_transform* Tsb,
                  uint32_t n, const float* origs_s, uint32_t n_origs, const float* dirs_s, float range_max,
                  float* points, float* normals, uint8_t* hits, uint32_t* face_ids, float* ranges)
{
    orc_simulate_opt(s, Tbm, Tsb, n, origs_s, n_origs, dirs_s, 0.0f, range_max, NULL, points, normals, hits, face_ids, ranges);
}

void orc_dataset_from_ranges(uint32_t n, const float* origs_s, uint32_t n_origs, const float* dirs_s, const float* ranges,
                             float range_min, float range_max, float* points, uint8_t* mask, uint32_t* n_valid)
{
    uint32_t valid = 0;
    for (uint32_t i = 0; i < n; i++) {
        const float* op = origs_s + 3 * (size_t)(n_origs == 1 ? 0 : i);
        const float r = ranges[i];
        points[3 * i + 0] = dirs_s[3 * i + 0] * r + op[0];
        points[3 * i + 1] = dirs_s[3 * i + 1] * r + op[1];
        points[3 * i + 2] = dirs_s[3 * i + 2] * r + op[2];
        if (r < range_min || r > range_max) mask[i] = 0;      /* NaN ranges compare false twice -> mask 1, like the reference */
        else { mask[i] = 1; valid++; }
    }
    if (n_valid) *n_valid = valid;
}

/* ------------------------------------------------------------------------------------------------ */
/* CrossStatistics                                                                                    */
/* ------------------------------------------------------------------------------------------------ */
void orc_cross_stats_identity(orc_cross_stats* s) { memset(s, 0, sizeof(*s)); }

void orc_cross_stats_merge(const orc_cross_stats* a, const orc_cross_stats* b, orc_cross_stats* out)
{
    orc_cross_stats r;
    const uint32_t n = a->n_meas + b->n_meas;
    if (n == 0) { orc_cross_stats_identity(out); return; }
    const float w1 = (float)a->n_meas / (float)n;
    const float w2 = (float)b->n_meas / (float)n;
    r.n_meas = n;
    r.dataset_mean = v3_add(v3_scale(a->dataset_mean, w1), v3_scale(b->dataset_mean, w2));
    r.model_mean = v3_add(v3_scale(a->model_mean, w1), v3_scale(b->model_mean, w2));
    const orc_vec3 ma = v3_sub(a->model_mean, r.model_mean), da = v3_sub(a->dataset_mean, r.dataset_mean);
    const orc_vec3 mb = v3_sub(b->model_mean, r.model_mean), db = v3_sub(b->dataset_mean, r.dataset_mean);
    const float mav[3] = {ma.x, ma.y, ma.z}, dav[3] = {da.x, da.y, da.z}, mbv[3] = {mb.x, mb.y, mb.z}, dbv[3] = {db.x, db.y, db.z};
    for (int c = 0; c < 3; c++)
        for (int rr = 0; rr < 3; rr++) {
            const float p1 = a->covariance.m[c * 3 + rr] * w1 + b->covariance.m[c * 3 + rr] * w2;
            const float p2 = (mav[rr] * dav[c]) * w1 + (mbv[rr] * dbv[c]) * w2;     /* (m - mbar)(d - dbar)^T */
            r.covariance.m[c * 3 + rr] = p1 + p2;
        }
    *out = r;
}

static void quat_to_mat(orc_quat q, float R[3][3])   /* R[r][c] */
{
    const float x = q.x, y = q.y, z = q.z, w = q.w;
    R[0][0] = 1.0f - 2.0f * (y * y + z * z); R[0][1] = 2.0f * (x * y - z * w);        R[0][2] = 2.0f * (x * z + y * w);
    R[1][0] = 2.0f * (x * y + z * w);        R[1][1] = 1.0f - 2.0f * (x * x + z * z); R[1][2] = 2.0f * (y * z - x * w);
    R[2][0] = 2.0f * (x * z - y * w);        R[2][1] = 2.0f * (y * z + x * w);        R[2][2] = 1.0f - 2.0f * (x * x + y * y);
}

void orc_cross_stats_transform(const orc_transform* T, const orc_cross_stats* s, orc_cross_stats* out)
{
    orc_cross_stats r;
    r.n_meas = s->n_meas;
    r.dataset_mean = T_apply(*T, s->dataset_mean);
    r.model_mean = T_apply(*T, s->model_mean);
    float R[3][3]; quat_to_mat(T->R, R);
    float RC[3][3];
    for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) {
        float acc = 0.0f; for (int k = 0; k < 3; k++) acc += R[i][k] * s->covariance.m[j * 3 + k];
        RC[i][j] = acc;
    }
    for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) {
        float acc = 0.0f; for (int k = 0; k < 3; k++) acc += RC[i][k] * R[j][k];
        r.covariance.m[j * 3 + i] = acc;
    }
    *out = r;
}

float orc_adaptive_max_dist(float max_dist, float adaptive_max_dist_min, double convergence_progress)
{
    /* CorrespondencesCPU.cpp:21-23: float*double + float*double -> float */
    return (float)(max_dist * (1.0 - convergence_progress) + adaptive_max_dist_min * convergence_progress);
}

/* per-element P2L in FP32; returns 1 if the pair is accepted */
static inline int p2l_elem(const orc_transform* Tpre, uint32_t i, const float* dpts, const uint8_t* dmask,
                           const float* mpts, const float* mnrm, const uint8_t* mmask, float max_dist,
                           orc_vec3* Di_out, orc_vec3* Mi_out)
{
    if (dmask && !(dmask[i] > 0)) return 0;
    if (mmask && !(mmask[i] > 0)) return 0;
    const orc_vec3 Di = T_apply(*Tpre, v3(dpts[3 * i], dpts[3 * i + 1], dpts[3 * i + 2]));
    const orc_vec3 Ii = v3(mpts[3 * i], mpts[3 * i + 1], mpts[3 * i + 2]);
    const orc_vec3 Ni = v3(mnrm[3 * i], mnrm[3 * i + 1], mnrm[3 * i + 2]);
    const float sd = v3_dot(v3_sub(Ii, Di), Ni);
    if (!(fabsf(sd) < max_dist)) return 0;
    *Di_out = Di;
    *Mi_out = v3_add(Di, v3_scale(Ni, sd));
    return 1;
}

void orc_statistics_p2l(const orc_transform* Tpre, uint32_t n, const float* dpts, const uint8_t* dmask,
                        const float* mpts, const float* mnrm, const uint8_t* mmask, float max_dist, orc_cross_stats* out)
{
    orc_cross_stats acc; orc_cross_stats_identity(&acc);
    for (uint32_t i = 0; i < n; i++) {
        orc_vec3 Di, Mi;
        if (!p2l_elem(Tpre, i, dpts, dmask, mpts, mnrm, mmask, max_dist, &Di, &Mi)) continue;
        orc_cross_stats one; orc_cross_stats_identity(&one);
        one.dataset_mean = Di; one.model_mean = Mi; one.n_meas = 1;
        orc_cross_stats merged; orc_cross_stats_merge(&acc, &one, &merged); acc = merged;
    }
    *out = acc;
}

/* Parallel variant used for TIMING the CPU baseline: rmagine reduces with TBB/OpenMP, i.e. per-thread partial CrossStatistics merged
 * at the end.  Fixed chunks of 1024 elements, FP32 merges inside a chunk, chunks merged in index order (deterministic). */
void orc_statistics_p2l_par(const orc_transform* Tpre, uint32_t n, const float* dpts, const uint8_t* dmask,
                            const float* mpts, const float* mnrm, const uint8_t* mmask, float max_dist, orc_cross_stats* out)
{
    const uint32_t chunk = 1024, nchunks = (n + chunk - 1) / chunk;
    orc_cross_stats* part = (orc_cross_stats*)malloc(sizeof(orc_cross_stats) * (nchunks ? nchunks : 1));
    #pragma omp parallel for schedule(static)
    for (int64_t c = 0; c < (int64_t)nchunks; c++) {
        orc_cross_stats acc; orc_cross_stats_identity(&acc);
        const uint32_t b = (uint32_t)c * chunk, e = b + chunk < n ? b + chunk : n;
        for (uint32_t i = b; i < e; i++) {
            orc_vec3 Di, Mi;
            if (!p2l_elem(Tpre, i, dpts, dmask, mpts, mnrm, mmask, max_dist, &Di, &Mi)) continue;
            orc_cross_stats one; orc_cross_stats_identity(&one);
            one.dataset_mean = Di; one.model_mean = Mi; one.n_meas = 1;
            orc_cross_stats merged; orc_cross_stats_merge(&acc, &one, &merged); acc = merged;
        }
        part[c] = acc;
    }
    orc_cross_stats acc; orc_cross_stats_identity(&acc);
    for (uint32_t c = 0; c < nchunks; c++) { orc_cross_stats merged; orc_cross_stats_merge(&acc, &part[c], &merged); acc = merged; }
    free(part);
    *out = acc;
}

void orc_statistics_p2l_f64(const orc_transform* Tpre, uint32_t n, const float* dpts, const uint8_t* dmask,
                            const float* mpts, const float* mnrm, const uint8_t* mmask, float max_dist, orc_cross_stats* out)
{
    double sd[3] = {0, 0, 0}, sm[3] = {0, 0, 0}, smd[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0}; uint32_t cnt = 0;
    for (uint32_t i = 0; i < n; i++) {
        orc_vec3 Di, Mi;
        if (!p2l_elem(Tpre, i, dpts, dmask, mpts, mnrm, mmask, max_dist, &Di, &Mi)) continue;
        const double d[3] = {Di.x, Di.y, Di.z}, m[3] = {Mi.x, Mi.y, Mi.z};
        for (int k = 0; k < 3; k++) { sd[k] += d[k]; sm[k] += m[k]; }
        for (int c = 0; c < 3; c++) for (int r = 0; r < 3; r++) smd[c * 3 + r] += m[r] * d[c];
        cnt++;
    }
    orc_cross_stats_identity(out);
    if (!cnt) return;
    const double inv = 1.0 / (double)cnt;
    double dm[3], mm[3];
    for (int k = 0; k < 3; k++) { dm[k] = sd[k] * inv; mm[k] = sm[k] * inv; }
    out->dataset_mean = v3((float)dm[0], (float)dm[1], (float)dm[2]);
    out->model_mean = v3((float)mm[0], (float)mm[1], (float)mm[2]);
    for (int c = 0; c < 3; c++) for (int r = 0; r < 3; r++) out->covariance.m[c * 3 + r] = (float)(smd[c * 3 + r] * inv - mm[r] * dm[c]);
    out->n_meas = cnt;
}

/* ------------------------------------------------------------------------------------------------ */
/* Umeyama: R = U S V^T from svd(C), t = mbar - R dbar                                                */
/* ------------------------------------------------------------------------------------------------ */
static double det3(double A[3][3])
{
    return A[0][0] * (A[1][1] * A[2][2] - A[1][2] * A[2][1]) - A[0][1] * (A[1][0] * A[2][2] - A[1][2] * A[2][0])
         + A[0][2] * (A[1][0] * A[2][1] - A[1][1] * A[2][0]);
}

/* one-sided Jacobi SVD, A = U diag(w) V^T, A is 3x3 row-major [r][c] */
static void svd3(double A[3][3], double U[3][3], double w[3], double V[3][3])
{
    double B[3][3];
    for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) { B[i][j] = A[i][j]; V[i][j] = (i == j); }
    for (int sweep = 0; sweep < 60; sweep++) {
        double off = 0.0;
        for (int p = 0; p < 2; p++) for (int q = p + 1; q < 3; q++) {
            double alpha = 0, beta = 0, gamma = 0;
            for (int i = 0; i < 3; i++) { alpha += B[i][p] * B[i][p]; beta += B[i][q] * B[i][q]; gamma += B[i][p] * B[i][q]; }
            if (gamma == 0.0) continue;
            double lim = 1e-16 * sqrt(alpha * beta);          /* relative only: an absolute floor stopped every rotation of a C below ~1e-15 */
            if (fabs(gamma) <= lim) continue;
            off += fabs(gamma);
            double zeta = (beta - alpha) / (2.0 * gamma);
            double t = (zeta >= 0 ? 1.0 : -1.0) / (fabs(zeta) + sqrt(1.0 + zeta * zeta));
            double c = 1.0 / sqrt(1.0 + t * t), sn = c * t;
            for (int i = 0; i < 3; i++) {
                double bp = B[i][p], bq = B[i][q]; B[i][p] = c * bp - sn * bq; B[i][q] = sn * bp + c * bq;
                double vp = V[i][p], vq = V[i][q]; V[i][p] = c * vp - sn * vq; V[i][q] = sn * vp + c * vq;
            }
        }
        if (off == 0.0) break;
    }
    /* sort descending */
    int idx[3] = {0, 1, 2}; double nrm[3];
    for (int j = 0; j < 3; j++) nrm[j] = sqrt(B[0][j] * B[0][j] + B[1][j] * B[1][j] + B[2][j] * B[2][j]);
    for (int a = 0; a < 2; a++) for (int b = a + 1; b < 3; b++) if (nrm[idx[b]] > nrm[idx[a]]) { int t = idx[a]; idx[a] = idx[b]; idx[b] = t; }
    double Vs[3][3], Bs[3][3];
    for (int j = 0; j < 3; j++) { w[j] = nrm[idx[j]]; for (int i = 0; i < 3; i++) { Vs[i][j] = V[i][idx[j]]; Bs[i][j] = B[i][idx[j]]; } }
    for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) V[i][j] = Vs[i][j];
    /* U columns: normalised B columns; complete degenerate ones */
    const double tiny = 1e-12 * (w[0] > 0 ? w[0] : 1.0);
    int good[3];
    for (int j = 0; j < 3; j++) {
        good[j] = w[j] > tiny;
        if (good[j]) for (int i = 0; i < 3; i++) U[i][j] = Bs[i][j] / w[j];
    }
    if (!good[0]) { for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) U[i][j] = (i == j); return; }
    if (!good[1]) {
        /* pick any unit vector orthogonal to U0 */
        double a[3] = {U[0][0], U[1][0], U[2][0]};
        int k = fabs(a[0]) < fabs(a[1]) ? (fabs(a[0]) < fabs(a[2]) ? 0 : 2) : (fabs(a[1]) < fabs(a[2]) ? 1 : 2);
        double e[3] = {0, 0, 0}; e[k] = 1.0;
        double b[3] = {a[1] * e[2] - a[2] * e[1], a[2] * e[0] - a[0] * e[2], a[0] * e[1] - a[1] * e[0]};
        double nb = sqrt(b[0] * b[0] + b[1] * b[1] + b[2] * b[2]);
        for (int i = 0; i < 3; i++) U[i][1] = b[i] / nb;
    }
    if (!good[2] || !good[1]) {
        /* U2 = +-(U0 x U1), sign chosen so that det(U) det(V) > 0 (no spurious reflection from the completion) */
        double c[3] = {U[1][0] * U[2][1] - U[2][0] * U[1][1], U[2][0] * U[0][1] - U[0][0] * U[2][1], U[0][0] * U[1][1] - U[1][0] * U[0][1]};
        double sgn = det3(V) < 0 ? -1.0 : 1.0;
        for (int i = 0; i < 3; i++) U[i][2] = sgn * c[i];
    }
}

static orc_quat mat_to_quat_d(double R[3][3])
{
    double q[4]; /* x y z w */
    double tr = R[0][0] + R[1][1] + R[2][2];
    if (tr > 0.0) {
        double s = sqrt(tr + 1.0) * 2.0; q[3] = 0.25 * s;
        q[0] = (R[2][1] - R[1][2]) / s; q[1] = (R[0][2] - R[2][0]) / s; q[2] = (R[1][0] - R[0][1]) / s;
    } else if (R[0][0] > R[1][1] && R[0][0] > R[2][2]) {
        double s = sqrt(1.0 + R[0][0] - R[1][1] - R[2][2]) * 2.0; q[3] = (R[2][1] - R[1][2]) / s;
        q[0] = 0.25 * s; q[1] = (R[0][1] + R[1][0]) / s; q[2] = (R[0][2] + R[2][0]) / s;
    } else if (R[1][1] > R[2][2]) {
        double s = sqrt(1.0 + R[1][1] - R[0][0] - R[2][2]) * 2.0; q[3] = (R[0][2] - R[2][0]) / s;
        q[0] = (R[0][1] + R[1][0]) / s; q[1] = 0.25 * s; q[2] = (R[1][2] + R[2][1]) / s;
    } else {
        double s = sqrt(1.0 + R[2][2] - R[0][0] - R[1][1]) * 2.0; q[3] = (R[1][0] - R[0][1]) / s;
        q[0] = (R[0][2] + R[2][0]) / s; q[1] = (R[1][2] + R[2][1]) / s; q[2] = 0.25 * s;
    }
    double n = sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
    orc_quat r = {(float)(q[0] / n), (float)(q[1] / n), (float)(q[2] / n), (float)(q[3] / n)};
    return r;
}

void orc_umeyama(const orc_cross_stats* s, orc_transform* out)
{
    *out = T_identity();
    if (s->n_meas == 0) return;
    double C[3][3], U[3][3], V[3][3], w[3];
    for (int r = 0; r < 3; r++) for (int c = 0; c < 3; c++) C[r][c] = s->covariance.m[c * 3 + r];
    svd3(C, U, w, V);
    double sgn = (det3(U) * det3(V) < 0.0) ? -1.0 : 1.0;
    double R[3][3];
    for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++)
        R[i][j] = U[i][0] * V[j][0] + U[i][1] * V[j][1] + sgn * U[i][2] * V[j][2];
    out->R = mat_to_quat_d(R);
    out->t = v3_sub(s->model_mean, q_rot(out->R, s->dataset_mean));
}

/* ------------------------------------------------------------------------------------------------ */
/* MICP drivers                                                                                       */
/* ------------------------------------------------------------------------------------------------ */
void orc_micp_correct_once(const orc_scene* s,
                           uint32_t n, const float* origs_s, uint32_t n_origs, const float* dirs_s, float range_max,
                           const float* dataset_pts, const uint8_t* dataset_mask,
                           const orc_transform* Tom, const orc_transform* Tbo, const orc_transform* Tsb,
                           uint32_t optimization_iterations, float max_dist, float adaptive_max_dist_min,
                           double convergence_progress, int f64_accum,
                           orc_transform* Tom_new, orc_transform* T_onew_oold_out, orc_cross_stats* Cmerged_out)
{
    float* mp = (float*)malloc(sizeof(float) * 3 * (size_t)n);
    float* mn = (float*)malloc(sizeof(float) * 3 * (size_t)n);
    uint8_t* mh = (uint8_t*)malloc((size_t)n);
    /* MICPSensor_::findCorrespondences (MICPSensor.hpp:146-151): Tbm = Tom * Tbo */
    const orc_transform Tbm = T_mul(*Tom, *Tbo);
    /* dirs_s == NULL selects closest-point correspondences (CPCEmbree::find, hits against the NON-adaptive params.max_dist) */
    if (dirs_s) orc_simulate(s, &Tbm, Tsb, n, origs_s, n_origs, dirs_s, range_max, mp, mn, mh, NULL, NULL);
    else        orc_cpc_find(s, &Tbm, Tsb, n, dataset_pts, max_dist, 0, mp, mn, mh, NULL, NULL);

    const float md = orc_adaptive_max_dist(max_dist, adaptive_max_dist_min, convergence_progress);
    orc_transform T_onew_oold = T_identity();
    orc_cross_stats Cmerged; orc_cross_stats_identity(&Cmerged);
    for (uint32_t it = 0; it < optimization_iterations; it++) {
        /* micp_localization.cpp:926 */
        const orc_transform T_bnew_bold = T_mul(T_mul(T_inv(*Tbo), T_onew_oold), *Tbo);
        /* MICPSensor.hpp:178 */
        const orc_transform T_snew_sold = T_mul(T_mul(T_inv(*Tsb), T_bnew_bold), *Tsb);
        orc_cross_stats stats_s, stats_b, Cs_o, ident;
        if (f64_accum == 1)      orc_statistics_p2l_f64(&T_snew_sold, n, dataset_pts, dataset_mask, mp, mn, mh, md, &stats_s);
        else if (f64_accum == 2) orc_statistics_p2l_par(&T_snew_sold, n, dataset_pts, dataset_mask, mp, mn, mh, md, &stats_s);
        else                     orc_statistics_p2l(&T_snew_sold, n, dataset_pts, dataset_mask, mp, mn, mh, md, &stats_s);
        orc_cross_stats_transform(Tsb, &stats_s, &stats_b);      /* MICPSensor.hpp:182 */
        orc_cross_stats_transform(Tbo, &stats_b, &Cs_o);         /* micp_localization.cpp:931 */
        orc_cross_stats_identity(&ident);
        orc_cross_stats_merge(&ident, &Cs_o, &Cmerged);          /* :918,:936 (single sensor, merge weight 1) */
        orc_transform T_inner; orc_umeyama(&Cmerged, &T_inner);  /* :952-953 */
        T_onew_oold = T_mul(T_onew_oold, T_inner);               /* :963 */
    }
    orc_transform Tn = T_mul(*Tom, T_onew_oold);                 /* :972 */
    if (Cmerged.n_meas > 0) Tn.R = q_normalize(Tn.R); else Tn = *Tom;   /* :974-984 */
    *Tom_new = Tn;
    if (T_onew_oold_out) *T_onew_oold_out = T_onew_oold;
    if (Cmerged_out) *Cmerged_out = Cmerged;
    free(mp); free(mn); free(mh);
}

/* MICPLocalizationNode::correctOnce over ALL sensors of the node (micp_localization.cpp:899-984), statement by statement. */
void orc_micp_correct_once_multi(const orc_scene* s, uint32_t n_sensors, const orc_micp_sensor* sen, const orc_transform* Tom,
                                 uint32_t optimization_iterations, double convergence_progress, int f64_accum,
                                 orc_transform* Tom_new, orc_transform* T_onew_oold_out, orc_cross_stats* Cmerged_out)
{
    float** mp = (float**)malloc(sizeof(float*) * n_sensors); float** mn = (float**)malloc(sizeof(float*) * n_sensors);
    uint8_t** mh = (uint8_t**)malloc(sizeof(uint8_t*) * n_sensors);
    for (uint32_t k = 0; k < n_sensors; k++) {                               /* :900-908 setTom + findCorrespondences */
        const orc_micp_sensor* S = &sen[k];
        mp[k] = (float*)malloc(sizeof(float) * 3 * (size_t)(S->n ? S->n : 1)); mn[k] = (float*)malloc(sizeof(float) * 3 * (size_t)(S->n ? S->n : 1));
        mh[k] = (uint8_t*)malloc((size_t)(S->n ? S->n : 1));
        const orc_transform Tbm = T_mul(*Tom, S->Tbo);                       /* MICPSensor.hpp:148 */
        if (S->dirs_s) orc_simulate(s, &Tbm, &S->Tsb, S->n, S->origs_s, S->n_origs, S->dirs_s, S->range_max, mp[k], mn[k], mh[k], NULL, NULL);
        else           orc_cpc_find(s, &Tbm, &S->Tsb, S->n, S->dataset_pts, S->max_dist, 0, mp[k], mn[k], mh[k], NULL, NULL);
    }
    orc_transform T_onew_oold = T_identity();                                /* :910 */
    orc_cross_stats Cmerged, Cmerged_w; orc_cross_stats_identity(&Cmerged); orc_cross_stats_identity(&Cmerged_w);
    for (uint32_t it = 0; it < optimization_iterations; it++) {              /* :915 */
        orc_cross_stats_identity(&Cmerged); orc_cross_stats_identity(&Cmerged_w);   /* :918-919 */
        for (uint32_t k = 0; k < n_sensors; k++) {                           /* :923 */
            const orc_micp_sensor* S = &sen[k];
            const orc_transform T_bnew_bold = T_mul(T_mul(T_inv(S->Tbo), T_onew_oold), S->Tbo);      /* :926 */
            const orc_transform T_snew_sold = T_mul(T_mul(T_inv(S->Tsb), T_bnew_bold), S->Tsb);      /* MICPSensor.hpp:178 */
            const float md = orc_adaptive_max_dist(S->max_dist, S->adaptive_max_dist_min, convergence_progress);   /* CorrespondencesCPU.cpp:21-23 */
            orc_cross_stats stats_s, Cs_b, Cs_o, Cs_w, tmp;
            if (f64_accum) orc_statistics_p2l_f64(&T_snew_sold, S->n, S->dataset_pts, S->dataset_mask, mp[k], mn[k], mh[k], md, &stats_s);
            else           orc_statistics_p2l(&T_snew_sold, S->n, S->dataset_pts, S->dataset_mask, mp[k], mn[k], mh[k], md, &stats_s);
            orc_cross_stats_transform(&S->Tsb, &stats_s, &Cs_b);             /* MICPSensor.hpp:182 */
            orc_cross_stats_transform(&S->Tbo, &Cs_b, &Cs_o);                /* :931 */
            Cs_w = Cs_o;
            Cs_w.n_meas = (uint32_t)((double)Cs_w.n_meas * S->merge_weight); /* :933-934: unsigned *= double */
            orc_cross_stats_merge(&Cmerged, &Cs_o, &tmp); Cmerged = tmp;     /* :936 */
            orc_cross_stats_merge(&Cmerged_w, &Cs_w, &tmp); Cmerged_w = tmp; /* :937 */
        }
        orc_transform T_inner; orc_umeyama(&Cmerged_w, &T_inner);            /* :952-953 */
        T_onew_oold = T_mul(T_onew_oold, T_inner);                           /* :963 */
    }
    orc_transform Tn = T_mul(*Tom, T_onew_oold);                             /* :972 */
    if (Cmerged.n_meas > 0) Tn.R = q_normalize(Tn.R); else Tn = *Tom;        /* :974-984 */
    *Tom_new = Tn;
    if (T_onew_oold_out) *T_onew_oold_out = T_onew_oold;
    if (Cmerged_out) *Cmerged_out = Cmerged;
    for (uint32_t k = 0; k < n_sensors; k++) { free(mp[k]); free(mn[k]); free(mh[k]); }
    free(mp); free(mn); free(mh);
}

void orc_correct_batch(const orc_scene* s, uint32_t n_poses, const orc_transform* Tbm, const orc_transform* Tsb,
                       uint32_t n, const float* origs_s, uint32_t n_origs, const float* dirs_s, float range_min, float range_max,
                       const float* ranges, float max_dist, int f64_accum,
                       orc_transform* Tdelta, uint32_t* ncorr, orc_cross_stats* stats_b_out)
{
    float* dp = (float*)malloc(sizeof(float) * 3 * (size_t)n);
    uint8_t* dm = (uint8_t*)malloc((size_t)n);
    orc_dataset_from_ranges(n, origs_s, n_origs, dirs_s, ranges, range_min, range_max, dp, dm, NULL);
    float* mp = (float*)malloc(sizeof(float) * 3 * (size_t)n);
    float* mn = (float*)malloc(sizeof(float) * 3 * (size_t)n);
    uint8_t* mh = (uint8_t*)malloc((size_t)n);
    const orc_transform I = T_identity();
    for (uint32_t p = 0; p < n_poses; p++) {
        orc_simulate(s, &Tbm[p], Tsb, n, origs_s, n_origs, dirs_s, range_max, mp, mn, mh, NULL, NULL);
        orc_cross_stats ss, sb;
        if (f64_accum) orc_statistics_p2l_f64(&I, n, dp, dm, mp, mn, mh, max_dist, &ss);
        else           orc_statistics_p2l(&I, n, dp, dm, mp, mn, mh, max_dist, &ss);
        orc_cross_stats_transform(Tsb, &ss, &sb);
        orc_umeyama(&sb, &Tdelta[p]);
        if (ncorr) ncorr[p] = sb.n_meas;
        if (stats_b_out) stats_b_out[p] = sb;
    }
    free(dp); free(dm); free(mp); free(mn); free(mh);
}

/* ------------------------------------------------------------------------------------------------ */
/* particle filter                                                                                    */
/* ------------------------------------------------------------------------------------------------ */
void orc_gaussian1d_add(orc_gaussian1d* a, const orc_gaussian1d* b)
{
    const uint32_t n = a->n_meas + b->n_meas;
    if (n == 0) return;
    const float w1 = (float)a->n_meas / (float)n;
    const float w2 = (float)b->n_meas / (float)n;
    const float mean = a->mean * w1 + b->mean * w2;
    const float d1 = a->mean - mean, d2 = b->mean - mean;
    const float sigma = (a->sigma * w1 + b->sigma * w2) + (d1 * d1 * w1 + d2 * d2 * w2);
    a->mean = mean; a->sigma = sigma; a->n_meas = n;
}

float orc_pf_evaluate_rcc(const orc_scene* s, const orc_range_meas* m, const orc_pf_params* p)
{
    const int real_hit = (p->range_min <= m->range) && (m->range <= p->range_max);      /* Interval::inside */
    float o[3] = {m->orig.x, m->orig.y, m->orig.z}, d[3] = {m->dir.x, m->dir.y, m->dir.z};
    ray_t r; ray_setup(&r, o, d);
    float t = INFINITY; uint32_t f = ORC_NOFACE;
    const int geom_hit = closest_hit(s, &r, INFINITY, 0, &t, &f);                       /* tnear 0, tfar +inf (:37-38) */
    const int sim_hit = geom_hit && (t > p->range_min);                                 /* :47 */
    float error;
    if (sim_hit) {
        if (real_hit) {
            float ng[3]; tri_ng(s, f, ng);
            orc_vec3 n = v3(ng[0], ng[1], ng[2]);
            if (p->ng_mode == 1) n = v3_normalize(n);
            const orc_vec3 preal = v3_add(m->orig, v3_scale(m->dir, m->range));         /* RangeMeasurement::mean */
            const orc_vec3 pint = v3_add(m->orig, v3_scale(m->dir, t));
            error = fabsf(v3_dot(v3_sub(pint, preal), n));
        } else error = p->real_miss_sim_hit_error;
    } else {
        error = real_hit ? p->real_hit_sim_miss_error : p->real_miss_sim_miss_error;
    }
    return error;
}

void orc_pf_sensor_update_one(const orc_scene* s, const orc_transform* Tsm, const orc_range_meas* meas_s,
                              const orc_pf_params* p, orc_particle_attr* attr)
{
    const float sigma_dist = p->dist_sigma;
    const float sigma_dist_quad = sigma_dist * sigma_dist;
    orc_range_meas mm;                                               /* RangeMeasurement.hpp:29-42; cov is never read (quirk D4) */
    mm.dir = q_rot(Tsm->R, meas_s->dir);
    mm.orig = T_apply(*Tsm, meas_s->orig);
    mm.range = meas_s->range;
    memset(&mm.cov, 0, sizeof(mm.cov));
    float error;
    if (p->correspondence_type == 1) {                               /* evaluate_cpc (:88-95): distance of meas_m.mean() to the surface */
        const orc_vec3 q = v3_add(mm.orig, v3_scale(mm.dir, mm.range));     /* RangeMeasurement.hpp:17-20 */
        const float qa[3] = {q.x, q.y, q.z};
        float d;
        error = orc_closest_point(s, qa, 0, &d, NULL, NULL, NULL) ? d : INFINITY;
    } else error = orc_pf_evaluate_rcc(s, &mm, p);
    /* :224  exp(-(e*e)/sq/2) / sqrt(2*sq*M_PI): float numerator argument, double exp / sqrt, stored to float */
    const float arg = -(error * error) / sigma_dist_quad / 2;
    const float eval = (float)(exp((double)arg) / sqrt((double)(2 * sigma_dist_quad) * M_PI));
    orc_gaussian1d meas = {eval, 0.0f, 1};
    orc_gaussian1d_add(&attr->likelihood, &meas);
    if (attr->likelihood.n_meas > 10000u) attr->likelihood.n_meas = 10000u;              /* MAX_N_MEAS */
}

void orc_pf_update(const orc_scene* s, uint32_t n_particles, const orc_transform* poses, orc_particle_attr* attrs,
                   const orc_transform* Tsb, uint32_t n_beams, const orc_range_meas* beams_s, const orc_pf_params* p)
{
    /* The reference loops beams-outer / particles-inner (:290-342); per particle the merge order over beams is the same,
     * so the loops are swapped here (particle-outer) for cache friendliness -- results are identical. */
    #pragma omp parallel for schedule(dynamic, 128)
    for (int64_t i = 0; i < (int64_t)n_particles; i++) {
        const orc_transform Tsm = T_mul(poses[i], *Tsb);
        orc_particle_attr a = attrs[i];
        for (uint32_t b = 0; b < n_beams; b++) orc_pf_sensor_update_one(s, &Tsm, &beams_s[b], p, &a);
        attrs[i] = a;
    }
}

/* ------------------------------------------------------------------------------------------------ */
/* closest-point correspondences: CPCEmbree::find (rmcl/src/rmcl/registration/CPCEmbree.cpp:17-43)       */
/* ------------------------------------------------------------------------------------------------ */
/* Stand-in for rm::EmbreeMap::closestPoint (Embree point query).  BVH-independent definition, mirrored op for op by the kernels:
 *   candidate(tri) = closest point on the triangle (C. Ericson's region tests, plain individually rounded ops), d2 = |p - q|^2;
 *   box bound      b2(box) = |max(lo - q, q - hi, 0)|^2  (monotone in the box);
 *   lim(d2)        = (sqrt(d2) + DELTA)^2, DELTA = 2^-16 * (1 + max|q_k|): dominates the rounding error of the candidate point;
 *   a candidate counts iff b2(triangle AABB) <= lim(d2); result = argmin (d2, face id); a node may be skipped only if b2(node) > lim(best). */
static inline float cp_b2(const float lo[3], const float hi[3], const float q[3])
{
    float acc[3];
    for (int k = 0; k < 3; k++) { float a = lo[k] - q[k], b = q[k] - hi[k]; float m = a > b ? a : b; acc[k] = m > 0.0f ? m : 0.0f; }
    return (acc[0] * acc[0] + acc[1] * acc[1]) + acc[2] * acc[2];
}
static inline float cp_lim(float d2, float delta) { float s = sqrtf(d2) + delta; return s * s; }
static inline float dot_plain(const float a[3], const float b[3]) { return (a[0] * b[0] + a[1] * b[1]) + a[2] * b[2]; }

static void cp_triangle(const float a[3], const float b[3], const float c[3], const float p[3], float out[3])
{
    float ab[3], ac[3], ap[3], bp[3], cp[3];
    for (int k = 0; k < 3; k++) { ab[k] = b[k] - a[k]; ac[k] = c[k] - a[k]; ap[k] = p[k] - a[k]; }
    const float d1 = dot_plain(ab, ap), d2 = dot_plain(ac, ap);
    if (d1 <= 0.0f && d2 <= 0.0f) { for (int k = 0; k < 3; k++) out[k] = a[k]; return; }
    for (int k = 0; k < 3; k++) bp[k] = p[k] - b[k];
    const float d3 = dot_plain(ab, bp), d4 = dot_plain(ac, bp);
    if (d3 >= 0.0f && d4 <= d3) { for (int k = 0; k < 3; k++) out[k] = b[k]; return; }
    const float vc = d1 * d4 - d3 * d2;
    /* d1 != d3: a == b (a segment a-c) gives d1 = d3 = 0, whose 0/0 made the candidate NaN; the ac region below takes it instead */
    if (vc <= 0.0f && d1 >= 0.0f && d3 <= 0.0f && d1 != d3) { const float v = d1 / (d1 - d3); for (int k = 0; k < 3; k++) out[k] = a[k] + ab[k] * v; return; }
    for (int k = 0; k < 3; k++) cp[k] = p[k] - c[k];
    const float d5 = dot_plain(ab, cp), d6 = dot_plain(ac, cp);
    if (d6 >= 0.0f && d5 <= d6) { for (int k = 0; k < 3; k++) out[k] = c[k]; return; }
    const float vb = d5 * d2 - d1 * d6;
    if (vb <= 0.0f && d2 >= 0.0f && d6 <= 0.0f) { const float w = d2 / (d2 - d6); for (int k = 0; k < 3; k++) out[k] = a[k] + ac[k] * w; return; }
    const float va = d3 * d6 - d5 * d4;
    if (va <= 0.0f && (d4 - d3) >= 0.0f && (d5 - d6) >= 0.0f) {
        const float w = (d4 - d3) / ((d4 - d3) + (d5 - d6));
        for (int k = 0; k < 3; k++) out[k] = b[k] + (c[k] - b[k]) * w;
        return;
    }
    const float denom = 1.0f / ((va + vb) + vc);
    const float v = vb * denom, w = vc * denom;
    for (int k = 0; k < 3; k++) out[k] = (a[k] + ab[k] * v) + ac[k] * w;
}

static int cp_candidate(const orc_scene* s, uint32_t f, const float q[3], float delta, float* d2_out, float p_out[3])
{
    const float* a = s->verts + 3 * (size_t)s->faces[3 * (size_t)f + 0];
    const float* b = s->verts + 3 * (size_t)s->faces[3 * (size_t)f + 1];
    const float* c = s->verts + 3 * (size_t)s->faces[3 * (size_t)f + 2];
    float p[3]; cp_triangle(a, b, c, q, p);
    const float dx = p[0] - q[0], dy = p[1] - q[1], dz = p[2] - q[2];
    const float d2 = (dx * dx + dy * dy) + dz * dz;
    float lo[3], hi[3];
    for (int k = 0; k < 3; k++) { lo[k] = fmin3(a[k], b[k], c[k]); hi[k] = fmax3(a[k], b[k], c[k]); }
    if (!(cp_b2(lo, hi, q) <= cp_lim(d2, delta))) return 0;
    *d2_out = d2; p_out[0] = p[0]; p_out[1] = p[1]; p_out[2] = p[2];
    return 1;
}

int orc_closest_point(const orc_scene* s, const float q[3], int brute, float* d_out, float p_out[3], float n_out[3], uint32_t* face_out)
{
    float qa = fabsf(q[0]); if (fabsf(q[1]) > qa) qa = fabsf(q[1]); if (fabsf(q[2]) > qa) qa = fabsf(q[2]);
    const float delta = 1.52587890625e-05f * (1.0f + qa);
    float best = INFINITY, bp[3] = {0, 0, 0}; uint32_t bf = ORC_NOFACE;
    if (s->nf == 0) return 0;
    if (!(isfinite(q[0]) && isfinite(q[1]) && isfinite(q[2]))) return 0;   /* no candidate can count for a non-finite query (every comparison fails) */
    if (brute) {
        for (uint32_t f = 0; f < s->nf; f++) {
            float d2, p[3];
            if (cp_candidate(s, f, q, delta, &d2, p) && (d2 < best || (d2 == best && f < bf))) { best = d2; bf = f; bp[0] = p[0]; bp[1] = p[1]; bp[2] = p[2]; }
        }
    } else {
        uint32_t stack[128]; int sp = 0; stack[sp++] = 0;
        while (sp) {
            const bvh_node* nd = &s->nodes[stack[--sp]];
            if (cp_b2(nd->lo, nd->hi, q) > cp_lim(best, delta)) continue;
            if (nd->count) {
                for (uint32_t i = 0; i < nd->count; i++) {
                    const uint32_t f = s->prim[nd->left_first + i]; float d2, p[3];
                    if (cp_candidate(s, f, q, delta, &d2, p) && (d2 < best || (d2 == best && f < bf))) { best = d2; bf = f; bp[0] = p[0]; bp[1] = p[1]; bp[2] = p[2]; }
                }
            } else if (sp + 2 <= 128) {
                const bvh_node* l = &s->nodes[nd->left_first]; const bvh_node* r = l + 1;
                if (cp_b2(l->lo, l->hi, q) <= cp_b2(r->lo, r->hi, q)) { stack[sp++] = nd->left_first + 1; stack[sp++] = nd->left_first; }
                else { stack[sp++] = nd->left_first; stack[sp++] = nd->left_first + 1; }
            }
        }
    }
    if (bf == ORC_NOFACE) return 0;
    if (d_out) *d_out = sqrtf(best);
    if (p_out) { p_out[0] = bp[0]; p_out[1] = bp[1]; p_out[2] = bp[2]; }
    if (face_out) *face_out = bf;
    if (n_out) { float ng[3]; tri_ng(s, bf, ng); orc_vec3 n = v3_normalize(v3(ng[0], ng[1], ng[2])); n_out[0] = n.x; n_out[1] = n.y; n_out[2] = n.z; }
    return 1;
}

/* CPCEmbree::find: per dataset point (mask NOT consulted, CPCEmbree.cpp:33-42): Pm = Tsm * d_i; cp = closestPoint(Pm);
 * hits = cp.d <= max_dist; points = Tms * cp.p; normals = Tms.R * cp.n */
void orc_cpc_find(const orc_scene* s, const orc_transform* Tbm, const orc_transform* Tsb, uint32_t n, const float* dataset_pts, float max_dist, int brute,
                  float* points, float* normals, uint8_t* hits, uint32_t* face_ids, float* dists)
{
    const orc_transform Tsm = T_mul(*Tbm, *Tsb);
    const orc_transform Tms = T_inv(Tsm);
    #pragma omp parallel for schedule(dynamic, 128)
    for (int64_t i = 0; i < (int64_t)n; i++) {
        const orc_vec3 Pm = T_apply(Tsm, v3(dataset_pts[3 * i], dataset_pts[3 * i + 1], dataset_pts[3 * i + 2]));
        const float q[3] = {Pm.x, Pm.y, Pm.z};
        float d, p[3], nn[3]; uint32_t f;
        if (orc_closest_point(s, q, brute, &d, p, nn, &f)) {
            put3(points, (size_t)i, T_apply(Tms, v3(p[0], p[1], p[2])));
            put3(normals, (size_t)i, q_rot(Tms.R, v3(nn[0], nn[1], nn[2])));
            if (hits) hits[i] = d <= max_dist;
            if (face_ids) face_ids[i] = f;
            if (dists) dists[i] = d;
        } else {
            put3(points, (size_t)i, v3(NAN, NAN, NAN)); put3(normals, (size_t)i, v3(NAN, NAN, NAN));
            if (hits) hits[i] = 0;
            if (face_ids) face_ids[i] = ORC_NOFACE;
            if (dists) dists[i] = INFINITY;
        }
    }
}

/* TFMotionUpdaterGPU: particle_move_and_forget_kernel (rmcl_ros/src/rmcl/particle_motion.cu:11-34): pose = pose * T_bnew_bold;
 * n_meas -= forget_rate * n_meas (uint32 -= double: computed in double, truncated on the store) */
void orc_pf_motion_update(uint32_t n, orc_transform* poses, orc_particle_attr* attrs, const orc_transform* T_bnew_bold, double forget_rate)
{
    orc_pf_motion_update_collide(NULL, n, poses, attrs, T_bnew_bold, forget_rate);
}

/* TFMotionUpdaterCPU::update inner loop (rmcl_ros/src/rmcl/TFMotionUpdaterCPU.cpp:184-224) with the optional wall check
 * collision_in_between (:17-50): a ray from the old to the new position, tfar = their distance (skipped below 1e-5 m); a hit sets the
 * likelihood to {0, 0, MAX_N_MEAS}.  s == NULL: no map, no check (the GPU updater, particle_motion.cu:11-34). */
void orc_pf_motion_update_collide(const orc_scene* s, uint32_t n, orc_transform* poses, orc_particle_attr* attrs, const orc_transform* T_bnew_bold, double forget_rate)
{
    #pragma omp parallel for schedule(static)
    for (int64_t i = 0; i < (int64_t)n; i++) {
        const orc_transform pose_old = poses[i];
        const orc_transform pose_new = T_mul(pose_old, *T_bnew_bold);
        orc_particle_attr a = attrs[i];
        const uint32_t nm = a.likelihood.n_meas;
        a.likelihood.n_meas = (uint32_t)((double)nm - forget_rate * (double)nm);
        if (s) {
            orc_vec3 vec = v3_sub(pose_new.t, pose_old.t);
            const float length = v3_l2norm(vec);
            if (!(length < 0.00001f)) {
                vec = v3(vec.x / length, vec.y / length, vec.z / length);
                const float o[3] = {pose_old.t.x, pose_old.t.y, pose_old.t.z}, d[3] = {vec.x, vec.y, vec.z};
                if (orc_intersect(s, o, d, length, 0, NULL, NULL, NULL)) { a.likelihood.mean = 0.0f; a.likelihood.sigma = 0.0f; a.likelihood.n_meas = 10000u; }
            }
        }
        poses[i] = pose_new; attrs[i] = a;
    }
}

/* compute_stats / simple_stats_kernel<512> with ONE block (rmcl_ros/src/rmcl/resampling.cu:41-92; GladiatorResamplerGPU sizes `stats` to 1):
 * lane tid accumulates L[tid], L[tid+512], ... in FP32 (sum) and max with initial 0, then a pairwise tree over the 512 lanes. */
void orc_pf_likelihood_stats(uint32_t n, const orc_particle_attr* attrs, float* sum_out, float* max_out)
{
    float sum[512], mx[512];
    for (uint32_t t = 0; t < 512; t++) { sum[t] = 0.0f; mx[t] = 0.0f; }
    for (uint32_t i = 0; i < n; i++) {
        const uint32_t t = i % 512u; const float L = attrs[i].likelihood.mean;
        sum[t] += L; if (L > mx[t]) mx[t] = L;
    }
    for (uint32_t s = 256; s > 0; s >>= 1)
        for (uint32_t t = 0; t < s; t++) { sum[t] = sum[t] + sum[t + s]; if (mx[t + s] > mx[t]) mx[t] = mx[t + s]; }
    *sum_out = sum[0]; *max_out = mx[0];
}

/* ------------------------------------------------------------------------------------------------ */
/* Gladiator resampling (resampling.cu:108-199)                                                      */
/* ------------------------------------------------------------------------------------------------ */
void orc_philox4x32_10(const uint32_t ctr_in[4], const uint32_t key_in[2], uint32_t out[4])
{
    uint32_t c[4] = {ctr_in[0], ctr_in[1], ctr_in[2], ctr_in[3]}, k[2] = {key_in[0], key_in[1]};
    for (int r = 0; r < 10; r++) {
        const uint64_t p0 = (uint64_t)0xD2511F53u * c[0], p1 = (uint64_t)0xCD9E8D57u * c[2];
        const uint32_t n0 = (uint32_t)(p1 >> 32) ^ c[1] ^ k[0], n1 = (uint32_t)p1, n2 = (uint32_t)(p0 >> 32) ^ c[3] ^ k[1], n3 = (uint32_t)p0;
        c[0] = n0; c[1] = n1; c[2] = n2; c[3] = n3;
        k[0] += 0x9E3779B9u; k[1] += 0xBB67AE85u;
    }
    out[0] = c[0]; out[1] = c[1]; out[2] = c[2]; out[3] = c[3];
}

static inline float u01_open(uint32_t r) { return ((float)(r >> 8) + 0.5f) * 5.9604644775390625e-08f; }   /* (0,1), exact in float */

void orc_pf_gladiator_randoms(uint64_t seed, uint32_t step, uint32_t first, uint32_t n, uint32_t* raw_out, float* normals_out)
{
    const uint32_t key[2] = {(uint32_t)seed, (uint32_t)(seed >> 32)};
    #pragma omp parallel for schedule(static)
    for (int64_t i = 0; i < (int64_t)n; i++) {
        uint32_t r[8];
        const uint32_t c0[4] = {first + (uint32_t)i, 0u, step, 0u}, c1[4] = {first + (uint32_t)i, 0u, step, 1u};
        orc_philox4x32_10(c0, key, r); orc_philox4x32_10(c1, key, r + 4);
        raw_out[i] = r[0];
        for (int p = 0; p < 3; p++) {                                  /* Box-Muller on (r[1+2p], r[2+2p]) */
            const float u1 = u01_open(r[1 + 2 * p]), u2 = u01_open(r[2 + 2 * p]);
            const float rad = sqrtf(-2.0f * logf(u1)), ang = 6.283185307179586f * u2;
            normals_out[6 * i + 2 * p] = rad * cosf(ang);
            normals_out[6 * i + 2 * p + 1] = rad * sinf(ang);
        }
    }
}

/* rm::EulerAngles <- Quaternion and back [RM-recalled: the standard ZYX conversions] */
static inline void quat_to_euler(orc_quat q, float* roll, float* pitch, float* yaw)
{
    const float sinr_cosp = 2.0f * (q.w * q.x + q.y * q.z), cosr_cosp = 1.0f - 2.0f * (q.x * q.x + q.y * q.y);
    *roll = atan2f(sinr_cosp, cosr_cosp);
    const float sinp = 2.0f * (q.w * q.y - q.z * q.x);
    *pitch = fabsf(sinp) >= 1.0f ? copysignf(1.5707963267948966f, sinp) : asinf(sinp);
    const float siny_cosp = 2.0f * (q.w * q.z + q.x * q.y), cosy_cosp = 1.0f - 2.0f * (q.y * q.y + q.z * q.z);
    *yaw = atan2f(siny_cosp, cosy_cosp);
}
static inline orc_quat euler_to_quat(float roll, float pitch, float yaw)
{
    const float cr = cosf(roll * 0.5f), sr = sinf(roll * 0.5f), cp = cosf(pitch * 0.5f), sp = sinf(pitch * 0.5f), cy = cosf(yaw * 0.5f), sy = sinf(yaw * 0.5f);
    orc_quat q;
    q.w = cr * cp * cy + sr * sp * sy;
    q.x = sr * cp * cy - cr * sp * sy;
    q.y = cr * sp * cy + sr * cp * sy;
    q.z = cr * cp * sy - sr * sp * cy;
    return q;
}

void orc_pf_gladiator_resample(uint32_t n_all, const orc_transform* poses, const orc_particle_attr* attrs, uint32_t first, uint32_t n_local,
                               const uint32_t* raw, const float* normals, const orc_gladiator_config* cfg,
                               orc_transform* poses_new, orc_particle_attr* attrs_new)
{
    #pragma omp parallel for schedule(static)
    for (int64_t i = 0; i < (int64_t)n_local; i++) {
        const uint32_t champion = first + (uint32_t)i;
        const uint32_t enemy = raw[i] % n_all;                                   /* :137 */
        const float Lc = attrs[champion].likelihood.mean, Le = attrs[enemy].likelihood.mean;
        if (Le > Lc) {                                                            /* :150 */
            const orc_transform pose = poses[enemy];
            orc_transform pn = pose; orc_particle_attr an = attrs[enemy];
            const float* N = normals + 6 * (size_t)i;
            pn.t.x += N[0] * cfg->min_noise_tx; pn.t.y += N[1] * cfg->min_noise_ty; pn.t.z += N[2] * cfg->min_noise_tz;    /* :166-168 */
            float roll, pitch, yaw; quat_to_euler(pn.R, &roll, &pitch, &yaw);
            roll += N[3] * cfg->min_noise_roll; pitch += N[4] * cfg->min_noise_pitch; yaw += N[5] * cfg->min_noise_yaw;    /* :169-173 */
            pn.R = euler_to_quat(roll, pitch, yaw);
            const orc_transform diff = T_mul(T_inv(pose), pn);                    /* :175 */
            const float trans_dist = v3_l2norm(diff.t);                           /* :178 (l2norm; the CPU variant squares it, quirk D7) */
            const float rot_dist = sqrtf(((diff.R.x * diff.R.x + diff.R.y * diff.R.y) + diff.R.z * diff.R.z) + diff.R.w * diff.R.w);   /* :179 Quaternion::l2norm [RM-recalled]: the 4-norm, ~1 */
            const float frs = (float)(1.0 - pow(1.0 - (double)cfg->likelihood_forget_per_meter, (double)trans_dist));      /* :182 */
            const float frr = (float)(1.0 - pow(1.0 - (double)cfg->likelihood_forget_per_radian, (double)rot_dist));       /* :183 */
            const float forget = frs > frr ? frs : frr;
            const float remember = (float)(1.0 - (double)forget);                 /* :185 */
            an.likelihood.n_meas = (uint32_t)((float)an.likelihood.n_meas * remember);     /* :187 uint *= float */
            poses_new[i] = pn; attrs_new[i] = an;
        } else { poses_new[i] = poses[champion]; attrs_new[i] = attrs[champion]; }
    }
}

/* ------------------------------------------------------------------------------------------------ */
/* scan-vs-map segmentation (scan_map_segmentation_embree.cpp:110-187)                               */
/* ------------------------------------------------------------------------------------------------ */
void orc_segment(uint32_t n, const float* origs_s, uint32_t n_origs, const float* dirs_s, float range_min, float range_max,
                 const float* ranges_real, const float* ranges_sim, const float* normals_sim, float min_dist_outlier_scan, float min_dist_outlier_map,
                 float* outlier_scan, uint32_t* n_scan, float* outlier_map, uint32_t* n_map, uint8_t* labels)
{
    uint32_t ns = 0, nm = 0;
    for (uint32_t i = 0; i < n; i++) {
        const uint32_t oi = n_origs == 1 ? 0 : i;
        const orc_vec3 dir = v3(dirs_s[3 * i], dirs_s[3 * i + 1], dirs_s[3 * i + 2]);
        const orc_vec3 orig = v3(origs_s[3 * oi], origs_s[3 * oi + 1], origs_s[3 * oi + 2]);
        const float rr = ranges_real[i], rs = ranges_sim[i];
        const int real_valid = (range_min <= rr) && (rr <= range_max);           /* model.range.inside, :121-122 */
        const int sim_valid = (range_min <= rs) && (rs <= range_max);
        int label = 0; orc_vec3 p = v3(0, 0, 0);
        if (real_valid) {
            const orc_vec3 preal = v3_add(v3_scale(dir, rr), orig);              /* :126 */
            if (sim_valid) {
                const orc_vec3 pint = v3_scale(dir, rs);                          /* :130 -- without the origin, as in the reference */
                const orc_vec3 nint = v3_normalize(v3(normals_sim[3 * i], normals_sim[3 * i + 1], normals_sim[3 * i + 2]));   /* :131-132 */
                const float spd = v3_dot(v3_sub(preal, pint), nint);              /* :134 */
                const orc_vec3 pmesh = v3_add(preal, v3_scale(nint, spd));        /* :135 */
                const float plane_distance = v3_l2norm(v3_sub(pmesh, preal));     /* :136 */
                if (rr < rs) { if (plane_distance > min_dist_outlier_scan) { label = 1; p = preal; } }     /* :138-149 */
                else         { if (plane_distance > min_dist_outlier_map)  { label = 2; p = pint; } }      /* :150-161 */
            } else { label = 1; p = preal; }                                       /* :164-171 */
        } else if (sim_valid) { label = 2; p = v3_add(v3_scale(dir, rs), orig); }  /* :173-182 */
        if (labels) labels[i] = (uint8_t)label;
        if (label == 1) { put3(outlier_scan, ns, p); ns++; }
        if (label == 2) { put3(outlier_map, nm, p); nm++; }
    }
    *n_scan = ns; *n_map = nm;
}

int orc_num_threads(void)
{
#ifdef _OPENMP
    return omp_get_max_threads();
#else
    return 1;
#endif
}
void orc_set_num_threads(int n)
{
#ifdef _OPENMP
    if (n > 0) omp_set_num_threads(n);
#else
    (void)n;
#endif
}
