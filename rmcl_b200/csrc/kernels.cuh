// kernels.cuh -- CUDA kernels of the ray-casting-correspondence path (sm_90a).  Compiled with -fmad=false: every FMA is explicit.
#pragma once
#include <cstddef>
#include "trace.cuh"
#if defined(__CUDACC__)
#include <cooperative_groups.h>
#endif

// ---------------------------------------------------------------------------------------------------------------------
// device-side CrossStatistics helpers (mirror oracle/oracle.c op for op; tolerance-level parity is all that is required,
// but identical order keeps whole ICP chains bit-identical in practice)
// ---------------------------------------------------------------------------------------------------------------------
struct CStats { V3 dm, mm; float C[9]; uint32_t n; };     // C column-major [c*3+r]

B2_DEV CStats cs_identity() { CStats s; s.dm = mk3(0, 0, 0); s.mm = mk3(0, 0, 0); for (int i = 0; i < 9; i++) s.C[i] = 0.f; s.n = 0; return s; }
B2_DEV CStats cs_load(const b2_cross_stats* p)
{
    CStats s; s.dm = mk3(p->dataset_mean.x, p->dataset_mean.y, p->dataset_mean.z); s.mm = mk3(p->model_mean.x, p->model_mean.y, p->model_mean.z);
    for (int i = 0; i < 9; i++) s.C[i] = p->covariance.m[i]; s.n = p->n_meas; return s;
}
B2_DEV void cs_store(b2_cross_stats* p, const CStats& s)
{
    p->dataset_mean.x = s.dm.x; p->dataset_mean.y = s.dm.y; p->dataset_mean.z = s.dm.z;
    p->model_mean.x = s.mm.x; p->model_mean.y = s.mm.y; p->model_mean.z = s.mm.z;
    for (int i = 0; i < 9; i++) p->covariance.m[i] = s.C[i]; p->n_meas = s.n;
}
// rm::CrossStatistics::operator+= (oracle: orc_cross_stats_merge)
B2_DEV CStats cs_merge(const CStats& a, const CStats& b)
{
    CStats r;
    const uint32_t n = a.n + b.n;
    if (n == 0) return cs_identity();
    const float w1 = dvd((float)a.n, (float)n), w2 = dvd((float)b.n, (float)n);
    r.n = n;
    r.dm = v_add(v_scale(a.dm, w1), v_scale(b.dm, w2));
    r.mm = v_add(v_scale(a.mm, w1), v_scale(b.mm, w2));
    const V3 ma = v_sub(a.mm, r.mm), da = v_sub(a.dm, r.dm), mb = v_sub(b.mm, r.mm), db = v_sub(b.dm, r.dm);
    const float mav[3] = {ma.x, ma.y, ma.z}, dav[3] = {da.x, da.y, da.z}, mbv[3] = {mb.x, mb.y, mb.z}, dbv[3] = {db.x, db.y, db.z};
    #pragma unroll
    for (int c = 0; c < 3; c++)
        #pragma unroll
        for (int rr = 0; rr < 3; rr++) {
            const float p1 = add(mul(a.C[c * 3 + rr], w1), mul(b.C[c * 3 + rr], w2));
            const float p2 = add(mul(mul(mav[rr], dav[c]), w1), mul(mul(mbv[rr], dbv[c]), w2));
            r.C[c * 3 + rr] = add(p1, p2);
        }
    return r;
}
// Transform * CrossStatistics (oracle: orc_cross_stats_transform)
B2_DEV CStats cs_transform(Tf T, const CStats& s)
{
    CStats r; r.n = s.n; r.dm = tf_apply(T, s.dm); r.mm = tf_apply(T, s.mm);
    const float x = T.R.x, y = T.R.y, z = T.R.z, w = T.R.w;
    float R[3][3];
    R[0][0] = sub(1.0f, mul(2.0f, add(mul(y, y), mul(z, z)))); R[0][1] = mul(2.0f, sub(mul(x, y), mul(z, w))); R[0][2] = mul(2.0f, add(mul(x, z), mul(y, w)));
    R[1][0] = mul(2.0f, add(mul(x, y), mul(z, w))); R[1][1] = sub(1.0f, mul(2.0f, add(mul(x, x), mul(z, z)))); R[1][2] = mul(2.0f, sub(mul(y, z), mul(x, w)));
    R[2][0] = mul(2.0f, sub(mul(x, z), mul(y, w))); R[2][1] = mul(2.0f, add(mul(y, z), mul(x, w))); R[2][2] = sub(1.0f, mul(2.0f, add(mul(x, x), mul(y, y))));
    float RC[3][3];
    #pragma unroll
    for (int i = 0; i < 3; i++)
        #pragma unroll
        for (int j = 0; j < 3; j++) { float acc = 0.0f; for (int k = 0; k < 3; k++) acc = add(acc, mul(R[i][k], s.C[j * 3 + k])); RC[i][j] = acc; }
    #pragma unroll
    for (int i = 0; i < 3; i++)
        #pragma unroll
        for (int j = 0; j < 3; j++) { float acc = 0.0f; for (int k = 0; k < 3; k++) acc = add(acc, mul(RC[i][k], R[j][k])); r.C[j * 3 + i] = acc; }
    return r;
}

// ---------------------------------------------------------------------------------------------------------------------
// rm::umeyama_transform (micp_localization.cpp:952-953): 3x3 SVD in double, same algorithm / order as oracle svd3()
// ---------------------------------------------------------------------------------------------------------------------
B2_DEV double det3d(const double A[3][3])
{
    return A[0][0] * (A[1][1] * A[2][2] - A[1][2] * A[2][1]) - A[0][1] * (A[1][0] * A[2][2] - A[1][2] * A[2][0])
         + A[0][2] * (A[1][0] * A[2][1] - A[1][1] * A[2][0]);
}

__host__ __device__ __noinline__ void svd3_dev(const double A[3][3], double U[3][3], double w[3], double V[3][3])
{
    double B[3][3];
    for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) { B[i][j] = A[i][j]; V[i][j] = (i == j) ? 1.0 : 0.0; }
    for (int sweep = 0; sweep < 60; sweep++) {
        double off = 0.0;
        for (int p = 0; p < 2; p++) for (int q = p + 1; q < 3; q++) {
            double alpha = 0, beta = 0, gamma = 0;
            for (int i = 0; i < 3; i++) { alpha += B[i][p] * B[i][p]; beta += B[i][q] * B[i][q]; gamma += B[i][p] * B[i][q]; }
            if (gamma == 0.0) continue;
            const double lim = 1e-16 * sqrt(alpha * beta);        // relative only: an absolute floor stopped every rotation of a C below ~1e-15
            if (fabs(gamma) <= lim) continue;
            off += fabs(gamma);
            const double zeta = (beta - alpha) / (2.0 * gamma);
            const double t = (zeta >= 0 ? 1.0 : -1.0) / (fabs(zeta) + sqrt(1.0 + zeta * zeta));
            const double c = 1.0 / sqrt(1.0 + t * t), sn = c * t;
            for (int i = 0; i < 3; i++) {
                const double bp = B[i][p], bq = B[i][q]; B[i][p] = c * bp - sn * bq; B[i][q] = sn * bp + c * bq;
                const double vp = V[i][p], vq = V[i][q]; V[i][p] = c * vp - sn * vq; V[i][q] = sn * vp + c * vq;
            }
        }
        if (off == 0.0) break;
    }
    int idx[3] = {0, 1, 2}; double nrm[3];
    for (int j = 0; j < 3; j++) nrm[j] = sqrt(B[0][j] * B[0][j] + B[1][j] * B[1][j] + B[2][j] * B[2][j]);
    for (int a = 0; a < 2; a++) for (int b = a + 1; b < 3; b++) if (nrm[idx[b]] > nrm[idx[a]]) { int t = idx[a]; idx[a] = idx[b]; idx[b] = t; }
    double Vs[3][3], Bs[3][3];
    for (int j = 0; j < 3; j++) { w[j] = nrm[idx[j]]; for (int i = 0; i < 3; i++) { Vs[i][j] = V[i][idx[j]]; Bs[i][j] = B[i][idx[j]]; } }
    for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) V[i][j] = Vs[i][j];
    const double tiny = 1e-12 * (w[0] > 0 ? w[0] : 1.0);
    bool good[3];
    for (int j = 0; j < 3; j++) {
        good[j] = w[j] > tiny;
        if (good[j]) for (int i = 0; i < 3; i++) U[i][j] = Bs[i][j] / w[j];
    }
    if (!good[0]) { for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) U[i][j] = (i == j) ? 1.0 : 0.0; return; }
    if (!good[1]) {
        const double a[3] = {U[0][0], U[1][0], U[2][0]};
        const int k = fabs(a[0]) < fabs(a[1]) ? (fabs(a[0]) < fabs(a[2]) ? 0 : 2) : (fabs(a[1]) < fabs(a[2]) ? 1 : 2);
        double e[3] = {0, 0, 0}; e[k] = 1.0;
        const double b[3] = {a[1] * e[2] - a[2] * e[1], a[2] * e[0] - a[0] * e[2], a[0] * e[1] - a[1] * e[0]};
        const double nb = sqrt(b[0] * b[0] + b[1] * b[1] + b[2] * b[2]);
        for (int i = 0; i < 3; i++) U[i][1] = b[i] / nb;
    }
    if (!good[2] || !good[1]) {
        const double c[3] = {U[1][0] * U[2][1] - U[2][0] * U[1][1], U[2][0] * U[0][1] - U[0][0] * U[2][1], U[0][0] * U[1][1] - U[1][0] * U[0][1]};
        const double sgn = det3d(V) < 0 ? -1.0 : 1.0;
        for (int i = 0; i < 3; i++) U[i][2] = sgn * c[i];
    }
}

#if B2_ON_DEVICE
B2_DEV float b2_rcp_approx(float x) { float r; asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x)); return r; }
B2_DEV float b2_rsqrt_approx(float x) { float r; asm("rsqrt.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x)); return r; }
#else
B2_DEV float b2_rcp_approx(float x) { return 1.0f / x; }
B2_DEV float b2_rsqrt_approx(float x) { return 1.0f / std::sqrt(x); }
#endif

// orthogonal polar factor of a 3x3 matrix with positive determinant; false if not applicable / not converged.
// Frobenius-scaled Newton iteration X <- (g X + X^-T / g) / 2 in FP32 (4-cycle ops, MUFU-based div/sqrt: ~3x shorter serial chain than
// FP64 on the one thread that executes it), then one unscaled FP64 step that makes the result orthogonal to double precision.
// Accuracy: FP32 rounding of the iterates perturbs the rotation by ~1e-7 rad (the reference's own rmagine SVD is FP32 as well); the
// translation inherits ~1e-7 * |mean| -- two orders below the 1e-5 tolerance on dT.
__host__ __device__ __noinline__ bool polar_newton3(const float A[3][3], double Q[3][3])
{
    // scale to unit Frobenius norm so that the iteration starts in its well-behaved range; the polar factor does not depend on the scale,
    // so the approximate reciprocal square root is as good as the exact one here
    float fro = 0.0f;
    for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) fro += A[i][j] * A[i][j];
    if (!(fro > 1e-30f)) return false;
    const float inv_n = b2_rsqrt_approx(fro);
    float X[3][3];
    for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) X[i][j] = A[i][j] * inv_n;
    bool conv = false;
    for (int it = 0; it < 40 && !conv; it++) {
        float Cf[3][3];                                           // cofactor matrix = det * X^-T
        Cf[0][0] = X[1][1] * X[2][2] - X[1][2] * X[2][1]; Cf[0][1] = X[1][2] * X[2][0] - X[1][0] * X[2][2]; Cf[0][2] = X[1][0] * X[2][1] - X[1][1] * X[2][0];
        Cf[1][0] = X[0][2] * X[2][1] - X[0][1] * X[2][2]; Cf[1][1] = X[0][0] * X[2][2] - X[0][2] * X[2][0]; Cf[1][2] = X[0][1] * X[2][0] - X[0][0] * X[2][1];
        Cf[2][0] = X[0][1] * X[1][2] - X[0][2] * X[1][1]; Cf[2][1] = X[0][2] * X[1][0] - X[0][0] * X[1][2]; Cf[2][2] = X[0][0] * X[1][1] - X[0][1] * X[1][0];
        const float det = X[0][0] * Cf[0][0] + X[0][1] * Cf[0][1] + X[0][2] * Cf[0][2];
        if (!(det > 1e-12f)) return false;                        // reflection, singular or NaN: let the SVD decide
        float a, b;
        if (it < 3) {
            // Frobenius scaling g^2 = |X^-T|_F / |X|_F only matters while X is far from orthogonal; approximate reciprocal / rsqrt are
            // enough (any g > 0 keeps the iteration convergent, and its errors are corrected by the following steps)
            float nx = 0.f, nc = 0.f;
            for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) { nx += X[i][j] * X[i][j]; nc += Cf[i][j] * Cf[i][j]; }
            const float rdet = b2_rcp_approx(det);
            const float q = nc * b2_rcp_approx(nx);                                  // (|Cf|/|X|)^2
            const float g2 = q * b2_rsqrt_approx(q) * rdet;                          // sqrt(q) / det
            const float rg = b2_rsqrt_approx(g2);                                    // 1 / g
            a = 0.5f * g2 * rg; b = 0.5f * rg * rdet;
        } else {
            a = 0.5f; b = 0.5f * b2_rcp_approx(det);
        }
        float diff = 0.f;
        for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) {
            const float y = a * X[i][j] + b * Cf[i][j];
            const float d = y - X[i][j]; diff += d * d;
            X[i][j] = y;
        }
        conv = (it >= 3) && diff < 1e-10f;                        // |dX|_F < 1e-5 on an unscaled step: the FP64 step finishes the job
    }
    if (!conv) return false;
    double Y[3][3];
    for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) Y[i][j] = (double)X[i][j];
    for (int it = 0; it < 1; it++) {                              // unscaled FP64 step: orthogonality 1e-6 -> 1e-12
        double Cf[3][3];
        Cf[0][0] = Y[1][1] * Y[2][2] - Y[1][2] * Y[2][1]; Cf[0][1] = Y[1][2] * Y[2][0] - Y[1][0] * Y[2][2]; Cf[0][2] = Y[1][0] * Y[2][1] - Y[1][1] * Y[2][0];
        Cf[1][0] = Y[0][2] * Y[2][1] - Y[0][1] * Y[2][2]; Cf[1][1] = Y[0][0] * Y[2][2] - Y[0][2] * Y[2][0]; Cf[1][2] = Y[0][1] * Y[2][0] - Y[0][0] * Y[2][1];
        Cf[2][0] = Y[0][1] * Y[1][2] - Y[0][2] * Y[1][1]; Cf[2][1] = Y[0][2] * Y[1][0] - Y[0][0] * Y[1][2]; Cf[2][2] = Y[0][0] * Y[1][1] - Y[0][1] * Y[1][0];
        const double det = Y[0][0] * Cf[0][0] + Y[0][1] * Cf[0][1] + Y[0][2] * Cf[0][2];
        const double b = 0.5 / det;
        for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) Y[i][j] = 0.5 * Y[i][j] + b * Cf[i][j];
    }
    for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) Q[i][j] = Y[i][j];
    return true;
}

__host__ __device__ __noinline__ Tf umeyama_dev(const CStats& s)
{
    Tf out = tf_identity();
    if (s.n == 0) return out;
    float Cf[3][3]; double R[3][3];
    for (int r = 0; r < 3; r++) for (int c = 0; c < 3; c++) Cf[r][c] = s.C[c * 3 + r];
    // Fast path: for det(C) > 0 the Umeyama rotation U S V^T (S = I) is the orthogonal polar factor of C, obtained with the scaled
    // Newton iteration X <- (g X + X^-T / g) / 2 (quadratically convergent, ~100 serial FP64 instructions per step instead of the
    // ~4000 of a Jacobi SVD -- this code runs on ONE thread between two reductions of the ICP loop, so its latency is the step's).
    // det(C) <= 0 (reflection case), a singular C or no convergence fall back to the SVD.
    if (!polar_newton3(Cf, R)) {
        double C[3][3], U[3][3], V[3][3], w[3];
        for (int r = 0; r < 3; r++) for (int c = 0; c < 3; c++) C[r][c] = (double)Cf[r][c];
        svd3_dev(C, U, w, V);
        const double sgn = (det3d(U) * det3d(V) < 0.0) ? -1.0 : 1.0;
        for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) R[i][j] = U[i][0] * V[j][0] + U[i][1] * V[j][1] + sgn * U[i][2] * V[j][2];
    }
    // rotation matrix -> quaternion in FP32 (the reference's rm::Quaternion::set(Matrix3x3) is FP32 as well); R is orthogonal to 1e-12
    float Rf[3][3];
    for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) Rf[i][j] = (float)R[i][j];
    float q[4];
    const float tr = Rf[0][0] + Rf[1][1] + Rf[2][2];
    if (tr > 0.0f) {
        const float sc = sqrt_rn(tr + 1.0f) * 2.0f; q[3] = 0.25f * sc;
        q[0] = dvd(Rf[2][1] - Rf[1][2], sc); q[1] = dvd(Rf[0][2] - Rf[2][0], sc); q[2] = dvd(Rf[1][0] - Rf[0][1], sc);
    } else if (Rf[0][0] > Rf[1][1] && Rf[0][0] > Rf[2][2]) {
        const float sc = sqrt_rn(1.0f + Rf[0][0] - Rf[1][1] - Rf[2][2]) * 2.0f; q[3] = dvd(Rf[2][1] - Rf[1][2], sc);
        q[0] = 0.25f * sc; q[1] = dvd(Rf[0][1] + Rf[1][0], sc); q[2] = dvd(Rf[0][2] + Rf[2][0], sc);
    } else if (Rf[1][1] > Rf[2][2]) {
        const float sc = sqrt_rn(1.0f + Rf[1][1] - Rf[0][0] - Rf[2][2]) * 2.0f; q[3] = dvd(Rf[0][2] - Rf[2][0], sc);
        q[0] = dvd(Rf[0][1] + Rf[1][0], sc); q[1] = 0.25f * sc; q[2] = dvd(Rf[1][2] + Rf[2][1], sc);
    } else {
        const float sc = sqrt_rn(1.0f + Rf[2][2] - Rf[0][0] - Rf[1][1]) * 2.0f; q[3] = dvd(Rf[1][0] - Rf[0][1], sc);
        q[0] = dvd(Rf[0][2] + Rf[2][0], sc); q[1] = dvd(Rf[1][2] + Rf[2][1], sc); q[2] = 0.25f * sc;
    }
    Q4 qq; qq.x = q[0]; qq.y = q[1]; qq.z = q[2]; qq.w = q[3];
    out.R = q_normalize(qq);
    out.t = v_sub(s.mm, q_rot(out.R, s.dm));
    return out;
}

// ---------------------------------------------------------------------------------------------------------------------
// P2L accumulation (rm::statistics_p2l, called at CorrespondencesCPU.cpp:26-30): FP32 per-element math identical to the oracle
// (=> identical gating, identical n_meas), sums in FP64 "sum form": n, S_d, S_m, S_{m d^T}
// ---------------------------------------------------------------------------------------------------------------------
#define B2_NACC 15
struct P2LAcc { double v[B2_NACC]; uint32_t n; };

B2_DEV void acc_zero(P2LAcc& a) { for (int i = 0; i < B2_NACC; i++) a.v[i] = 0.0; a.n = 0; }
B2_DEV void acc_add_pair(P2LAcc& a, V3 D, V3 M)
{
    const double d[3] = {(double)D.x, (double)D.y, (double)D.z}, m[3] = {(double)M.x, (double)M.y, (double)M.z};
    a.v[0] += d[0]; a.v[1] += d[1]; a.v[2] += d[2];
    a.v[3] += m[0]; a.v[4] += m[1]; a.v[5] += m[2];
    #pragma unroll
    for (int c = 0; c < 3; c++)
        #pragma unroll
        for (int r = 0; r < 3; r++) a.v[6 + c * 3 + r] += m[r] * d[c];
    a.n++;
}
// P2L gate for one pair; returns true and (D, M) if accepted
B2_DEV bool p2l_pair(Tf Tpre, V3 d, V3 I, V3 N, float max_dist, V3& D, V3& M)
{
    D = tf_apply(Tpre, d);
    const float sd = v_dot(v_sub(I, D), N);
    if (!(fabsf(sd) < max_dist)) return false;
    M = v_add(D, v_scale(N, sd));
    return true;
}
B2_DEV CStats acc_finalize(const double* v, uint32_t n)
{
    CStats s = cs_identity();
    if (n == 0) return s;
    const double inv = 1.0 / (double)n;
    double dm[3], mm[3];
    for (int k = 0; k < 3; k++) { dm[k] = v[k] * inv; mm[k] = v[3 + k] * inv; }
    s.dm = mk3((float)dm[0], (float)dm[1], (float)dm[2]);
    s.mm = mk3((float)mm[0], (float)mm[1], (float)mm[2]);
    for (int c = 0; c < 3; c++) for (int r = 0; r < 3; r++) s.C[c * 3 + r] = (float)(v[6 + c * 3 + r] * inv - mm[r] * dm[c]);
    s.n = n;
    return s;
}

// block-level sum of the accumulators; result valid in thread 0.  smem: double[(B2_NACC+1) * (BLOCK/32)]
//
// Warp stage = reduce-scatter: at each of four steps a lane hands half of its remaining values to its partner and adds the partner's half
// of the values it keeps, so 16 values cost 8+4+2+1 (+1 final) = 16 64-bit shuffles instead of 16 x 5 = 80 for 16 independent butterflies
// (the FP64 shuffles of the plain version were the longest part of the reduction pass by the clock stamps in k_icp_loop).
// After the four steps lane l holds value index ((l>>1) & 15) summed over the 16 lanes that share its bit 0; one xor-1 step completes it.
#if defined(__CUDACC__)
template <int H>
__device__ __forceinline__ void rs_step(double (&v)[16], int offset, bool upper)
{
    #pragma unroll
    for (int i = 0; i < H; i++) {
        const double send = upper ? v[i] : v[i + H];
        const double keep = upper ? v[i + H] : v[i];
        v[i] = keep + __shfl_xor_sync(0xffffffffu, send, offset);
    }
}
template <int BLOCK>
__device__ __forceinline__ void block_reduce_acc(P2LAcc& a, double* smem)
{
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    constexpr int NW = BLOCK / 32;
    double v[16];
    #pragma unroll
    for (int i = 0; i < B2_NACC; i++) v[i] = a.v[i];
    v[15] = 0.0;
    rs_step<8>(v, 16, (lane & 16) != 0);      // keeps values [8,16) if bit 4 set else [0,8)
    rs_step<4>(v, 8, (lane & 8) != 0);
    rs_step<2>(v, 4, (lane & 4) != 0);
    rs_step<1>(v, 2, (lane & 2) != 0);
    const double tot = v[0] + __shfl_xor_sync(0xffffffffu, v[0], 1);
    const int vidx = ((lane >> 4) & 1) * 8 + ((lane >> 3) & 1) * 4 + ((lane >> 2) & 1) * 2 + ((lane >> 1) & 1);
    a.n = warp_sum_u32(a.n);
    if ((lane & 1) == 0 && vidx < B2_NACC) smem[vidx * NW + warp] = tot;
    if (lane == 0) smem[B2_NACC * NW + warp] = (double)a.n;
    __syncthreads();
    if (warp == 0) {
        // lane i < 16 sums value i over the NW warps (fixed order)
        if (lane <= B2_NACC) {
            double x = 0.0;
            #pragma unroll
            for (int w = 0; w < NW; w++) x += smem[lane * NW + w];
            smem[lane * NW] = x;
        }
        __syncwarp();
        if (lane == 0) {
            #pragma unroll
            for (int i = 0; i < B2_NACC; i++) a.v[i] = smem[i * NW];
            a.n = (uint32_t)(smem[B2_NACC * NW] + 0.5);
        }
    }
    __syncthreads();
}
#endif

// ---------------------------------------------------------------------------------------------------------------------
// ICP state kept on the device between the kernels of one correctOnce (micp_localization.cpp:899-984)
// ---------------------------------------------------------------------------------------------------------------------
struct alignas(16) IcpState {
    b2_transform Tom, Tbo, Tsb;          // inputs
    b2_transform T_onew_oold;            // :910, :963
    b2_transform T_snew_sold;            // pre-transform of the NEXT reduction (MICPSensor.hpp:178)
    b2_transform Tom_new;                // :972-984
    b2_transform Tos, Tso;               // Tos = Tbo * Tsb (sensor -> odom), Tso = ~Tos: composed once per correctOnce on the host
    b2_cross_stats Cmerged_o;            // :918-937 (single sensor)
    b2_cross_stats stats_s;              // last sensor-frame statistics
    float max_dist;
    uint32_t iter;
    float Ros[9];                        // rotation matrix of Tos, row-major
    uint32_t pad_[1];
    unsigned long long dbg[8];           // SM-clock stamps of the last reduction's tail (profiling aid, b2_rcc_debug_clocks)
};

// rotation matrix (row-major) of a unit quaternion
B2_DEV void quat_to_mat(Q4 q, float R[9])
{
    const float x = q.x, y = q.y, z = q.z, w = q.w;
    R[0] = sub(1.0f, mul(2.0f, add(mul(y, y), mul(z, z)))); R[1] = mul(2.0f, sub(mul(x, y), mul(z, w))); R[2] = mul(2.0f, add(mul(x, z), mul(y, w)));
    R[3] = mul(2.0f, add(mul(x, y), mul(z, w))); R[4] = sub(1.0f, mul(2.0f, add(mul(x, x), mul(z, z)))); R[5] = mul(2.0f, sub(mul(y, z), mul(x, w)));
    R[6] = mul(2.0f, sub(mul(x, z), mul(y, w))); R[7] = mul(2.0f, add(mul(y, z), mul(x, w))); R[8] = sub(1.0f, mul(2.0f, add(mul(x, x), mul(y, y))));
}

static_assert(offsetof(IcpState, Tos) % 16 == 0 && offsetof(IcpState, Tso) % 16 == 0 && offsetof(IcpState, Cmerged_o) % 16 == 0 && sizeof(IcpState) % 16 == 0, "IcpState alignment");

B2_DEV Tf icp_pretransform(Tf Tbo, Tf Tsb, Tf T_onew_oold)
{
    const Tf T_bnew_bold = tf_mul(tf_mul(tf_inv(Tbo), T_onew_oold), Tbo);      // micp_localization.cpp:926
    return tf_mul(tf_mul(tf_inv(Tsb), T_bnew_bold), Tsb);                      // MICPSensor.hpp:178
}

// one inner iteration after the reduction delivered stats_s (thread 0 only)
B2_DEV void icp_step(IcpState* st, const CStats& stats_s)
{
    const Tf Tbo = tf_load(&st->Tbo), Tsb = tf_load(&st->Tsb), Tom = tf_load(&st->Tom);
    Tf T_onew_oold = tf_load(&st->T_onew_oold);
    const CStats stats_b = cs_transform(Tsb, stats_s);                        // MICPSensor.hpp:182
    const CStats Cs_o = cs_transform(Tbo, stats_b);                           // micp_localization.cpp:931
    const CStats Cmerged = cs_merge(cs_identity(), Cs_o);                     // :918,:936
    const Tf T_inner = umeyama_dev(Cmerged);                                  // :952-953
    T_onew_oold = tf_mul(T_onew_oold, T_inner);                               // :963
    tf_store(&st->T_onew_oold, T_onew_oold);
    tf_store(&st->T_snew_sold, icp_pretransform(Tbo, Tsb, T_onew_oold));
    Tf Tn = tf_mul(Tom, T_onew_oold);                                         // :972
    if (Cmerged.n > 0) Tn.R = q_normalize(Tn.R); else Tn = Tom;               // :974-984
    tf_store(&st->Tom_new, Tn);
    cs_store(&st->Cmerged_o, Cmerged);
    cs_store(&st->stats_s, stats_s);
    st->iter++;
}

// ---------------------------------------------------------------------------------------------------------------------
// generic closest hit for arbitrary rays (b2_mesh_intersect)
// ---------------------------------------------------------------------------------------------------------------------
template <bool STATS>
__global__ void __launch_bounds__(128) k_intersect(BvhView bvh, const float* __restrict__ origs, const float* __restrict__ dirs, uint32_t n, float tfar,
                                                   float* __restrict__ t_out, uint32_t* __restrict__ face_out, float* __restrict__ ng_out, uint8_t* __restrict__ hit_out,
                                                   unsigned long long* __restrict__ counters)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t nn = 0, nt = 0;
    if (i < n) {
        const RaySetup r = ray_setup(mk3(origs[3 * i], origs[3 * i + 1], origs[3 * i + 2]), mk3(dirs[3 * i], dirs[3 * i + 1], dirs[3 * i + 2]), bvh);
        HitRec h = trace_init(tfar);
        trace_closest<STATS>(bvh, r, h, nn, nt);
        const bool hit = h.face != B2_NOFACE;
        if (t_out) t_out[i] = hit ? h.t : u2f(0x7f800000u);
        if (face_out) face_out[i] = h.face;
        if (hit_out) hit_out[i] = hit ? 1 : 0;
        if (ng_out) {
            V3 ng = mk3(0.f, 0.f, 0.f);
            if (hit) ng = tri_ng(bvh, h.tri);
            ng_out[3 * i] = ng.x; ng_out[3 * i + 1] = ng.y; ng_out[3 * i + 2] = ng.z;
        }
    }
    if (STATS) {
        const uint32_t sn = warp_sum_u32(nn), stt = warp_sum_u32(nt);
        if ((threadIdx.x & 31) == 0) { atomicAdd(counters, (unsigned long long)sn); atomicAdd(counters + 1, (unsigned long long)stt); }
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// MICP*Sensor*::unpackMessage on the device (MICPSphericalSensorCPU.cpp:181-233)
// ---------------------------------------------------------------------------------------------------------------------
// one dataset entry: point = dir * range + orig, mask = range in [range_min, range_max] (MICPO1DnSensorCUDA.cpp:201-215)
// (dir[di ..], orig[oi ..]: 32-bit element indices, as the tables are indexed everywhere else)
B2_DEV void dataset_entry(uint32_t i, float r, const float* dir, uint32_t di, const float* orig, uint32_t oi, float range_min, float range_max, float* pts, uint8_t* mask)
{
    pts[3 * i + 0] = add(mul(dir[di + 0], r), orig[oi + 0]);
    pts[3 * i + 1] = add(mul(dir[di + 1], r), orig[oi + 1]);
    pts[3 * i + 2] = add(mul(dir[di + 2], r), orig[oi + 2]);
    mask[i] = (r < range_min || r > range_max) ? 0 : 1;
}

__global__ void k_dataset_from_ranges(const float* __restrict__ ranges, const float* __restrict__ dirs, const float* __restrict__ origs, uint32_t n_origs,
                                      uint32_t n, float range_min, float range_max, float* __restrict__ pts, uint8_t* __restrict__ mask)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float r = ranges[i];
    const uint32_t oi = n_origs == 1 ? 0 : i;
    dataset_entry(i, r, dirs, 3 * i, origs, 3 * oi, range_min, range_max, pts, mask);
}

// ---------------------------------------------------------------------------------------------------------------------
// Pc2ToO1DnNode::convert on the device: estimateModelAndData (conversions.cpp:869-1073) + filter (scan_operations.cpp:41-143)
// ---------------------------------------------------------------------------------------------------------------------
struct CloudO1Dn {
    uint32_t w_out, h_out;                  // output raster (filtered)
    uint64_t row_step; uint32_t point_step;
    uint32_t off[3];                        // byte offsets of x, y, z inside a point
    uint32_t f64;                           // 1: FLOAT64 fields (narrowed to float), 0: FLOAT32
    uint32_t h_inc, h_begin, w_inc, w_begin;
    float range_min, range_max;
};

// little-endian loads at any byte address (PointField offsets need not be aligned)
B2_DEV uint32_t cloud_u32(const uint8_t* p)
{
    if (!((uintptr_t)p & 3u)) return *reinterpret_cast<const uint32_t*>(p);
    return (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24);
}
B2_DEV float cloud_coord(const uint8_t* p, bool f64)
{
    if (!f64) return u2f(cloud_u32(p));
    const unsigned long long u = (unsigned long long)cloud_u32(p) | ((unsigned long long)cloud_u32(p + 4) << 32);
    double d;
#if B2_ON_DEVICE
    d = __longlong_as_double((long long)u);
#else
    memcpy(&d, &u, 8);
#endif
    return (float)d;                        // round to nearest, as the reference's implicit double -> float
}
B2_DEV bool finite_f32(float a) { return (f2u(a) & 0x7f800000u) != 0x7f800000u; }

// one point of the cloud -> ray direction and range (conversions.cpp:992-1011; rm::Vector::l2norm and operator/=)
B2_DEV void o1dn_from_point(float x, float y, float z, float* dir, float& range)
{
    if (finite_f32(x) && finite_f32(y) && finite_f32(z)) {
        range = v_l2norm(mk3(x, y, z));
        dir[0] = dvd(x, range); dir[1] = dvd(y, range); dir[2] = dvd(z, range);
    } else {
        dir[0] = 0.f; dir[1] = 0.f; dir[2] = 0.f; range = 0.f;
    }
}

// output ray k of the filtered raster (scan_operations.cpp:100-111): reads its source point, converts it, writes the ray table entry, the
// range and the dataset entry (the model's origin is 0)
B2_DEV void o1dn_cloud_entry(const uint8_t* cloud, const CloudO1Dn& c, uint32_t k, float* dirs, float* ranges, float* pts, uint8_t* mask)
{
    const uint32_t i = k / c.w_out, j = k - i * c.w_out;
    const uint64_t src_i = (uint64_t)i * c.h_inc + c.h_begin, src_j = (uint64_t)j * c.w_inc + c.w_begin;
    const uint8_t* p = cloud + src_i * c.row_step + src_j * c.point_step;
    const bool f64 = c.f64 != 0;
    float d[3], r;
    o1dn_from_point(cloud_coord(p + c.off[0], f64), cloud_coord(p + c.off[1], f64), cloud_coord(p + c.off[2], f64), d, r);
    dirs[3 * k + 0] = d[0]; dirs[3 * k + 1] = d[1]; dirs[3 * k + 2] = d[2];
    ranges[k] = r;
    const float orig[3] = {0.f, 0.f, 0.f};
    dataset_entry(k, r, d, 0, orig, 0, c.range_min, c.range_max, pts, mask);
}

// one thread per output ray
__global__ void k_o1dn_from_cloud(const uint8_t* __restrict__ cloud, CloudO1Dn c, float* __restrict__ dirs, float* __restrict__ ranges,
                                  float* __restrict__ pts, uint8_t* __restrict__ mask)
{
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= c.w_out * c.h_out) return;
    o1dn_cloud_entry(cloud, c, k, dirs, ranges, pts, mask);
}

// ---------------------------------------------------------------------------------------------------------------------
// Pc2ToScanNode::convert (pc2_to_scan.cpp:105-213) + fillEmpty (scan_operations.cpp:25-39) + MICPSphericalSensor*::unpackMessage
// (MICPSphericalSensorCUDA.cpp:176-235) on the device, as a scatter in two passes: every point proposes a key to its cell, every cell
// turns its key into a range and a dataset entry.  A key is ((point index + 1) << 32) | range bits, so the atomicMax of a cell keeps the
// point of the highest index -- the reference's last writer in index order, whatever order the atomics arrive in.  0 = no point.
// ---------------------------------------------------------------------------------------------------------------------
struct CloudScan {
    uint32_t width, n_points;               // points of the cloud (width * height, at most 2^32 - 2)
    uint64_t row_step; uint32_t point_step;
    uint32_t off[3];                        // byte offsets of x, y, z inside a point
    uint32_t f64;                           // 1: FLOAT64 fields (narrowed to float), 0: FLOAT32
    Tf T;                                   // T_sensor_cloud
    float phi_min, phi_inc, theta_min, theta_inc;
    uint32_t phi_n, theta_n;
    float range_min, range_max, fill;       // fill: fillEmpty's range_max + 1
};

// bin of one angle (pc2_to_scan.cpp:195-196): (a - min) / inc in float, + 0.5 in double, truncated toward zero, so (-1.5, -0.5] goes to 0
// and nothing wraps around (SURVEY D23); -1 outside [0, n).  A dimension of size 1 with increment 0 takes every angle (D24: the reference
// divides 0 by 0 there); an increment of 0 with more than one bin is refused before any launch.
B2_DEV int scan_bin(float a, float mn, float inc, uint32_t n)
{
    if (inc == 0.f) return n == 1 ? 0 : -1;
    const double b = add_d((double)dvd(sub(a, mn), inc), 0.5);
    return (b > -1.0 && b < (double)n) ? (int)b : -1;
}

// point i of the cloud (pc2_to_scan.cpp:186-209) -> its key, or 0 when it writes no cell; *cell receives the cell.  The angles are FP64
// atan2 rounded to float; the elevation is taken against the horizontal distance sqrt(x^2 + y^2), not the reference's 3-D norm (D21).
B2_DEV unsigned long long scan_point_key(float x, float y, float z, uint32_t i, const CloudScan& c, uint32_t& cell)
{
    if (!(finite_f32(x) && finite_f32(y) && finite_f32(z))) return 0ull;
    const V3 p = tf_apply(c.T, mk3(x, y, z));                               // rm::Transform * Vector
    const float r = v_l2norm(p);
    const double px = p.x, py = p.y, pz = p.z;
    const float theta = (float)atan2_d(py, px);
    const float phi = (float)atan2_d(pz, sqrt_d(add_d(mul_d(px, px), mul_d(py, py))));
    const int pid = scan_bin(phi, c.phi_min, c.phi_inc, c.phi_n), tid = scan_bin(theta, c.theta_min, c.theta_inc, c.theta_n);
    if (pid < 0 || tid < 0 || !(r >= c.range_min && r <= c.range_max)) return 0ull;     // model.range.inside
    cell = (uint32_t)pid * c.theta_n + (uint32_t)tid;
    return ((unsigned long long)(i + 1u) << 32) | f2u(r);
}

// point i read at row * row_step + col * point_step (D22: the reference ignores row_step)
B2_DEV unsigned long long scan_cloud_key(const uint8_t* cloud, const CloudScan& c, uint32_t i, uint32_t& cell)
{
    const uint32_t row = i / c.width, col = i - row * c.width;
    const uint8_t* p = cloud + (uint64_t)row * c.row_step + (uint64_t)col * c.point_step;
    const bool f64 = c.f64 != 0;
    return scan_point_key(cloud_coord(p + c.off[0], f64), cloud_coord(p + c.off[1], f64), cloud_coord(p + c.off[2], f64), i, c, cell);
}

// cell k: its range (fill when no point won it), the dataset entry through the model's direction table, and the key reset for the next call
B2_DEV void scan_cell_entry(uint32_t k, unsigned long long* keys, const CloudScan& c, const float* dirs, const float* origs, float* ranges,
                            float* pts, uint8_t* mask)
{
    const unsigned long long key = keys[k];
    keys[k] = 0ull;
    const float r = key ? u2f((uint32_t)key) : c.fill;
    ranges[k] = r;
    dataset_entry(k, r, dirs, 3 * k, origs, 0, c.range_min, c.range_max, pts, mask);
}

// one thread per point of the cloud
__global__ void k_scan_bin_cloud(const uint8_t* __restrict__ cloud, CloudScan c, unsigned long long* __restrict__ keys)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= c.n_points) return;
    uint32_t cell = 0;
    const unsigned long long key = scan_cloud_key(cloud, c, i, cell);
    if (key) atomicMax(keys + cell, key);
}

// one thread per cell of the model
__global__ void k_scan_cells(CloudScan c, unsigned long long* __restrict__ keys, const float* __restrict__ dirs, const float* __restrict__ origs,
                             float* __restrict__ ranges, float* __restrict__ pts, uint8_t* __restrict__ mask)
{
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= c.phi_n * c.theta_n) return;
    scan_cell_entry(k, keys, c, dirs, origs, ranges, pts, mask);
}

// ---------------------------------------------------------------------------------------------------------------------
// RCC*::find (RCCEmbree.cpp:26-36 ...): one thread per (pose, ray); writes the model buffers in the SENSOR frame
// ---------------------------------------------------------------------------------------------------------------------
struct RayModel {
    const float* dirs;      // n x 3 (sensor frame)
    const float* origs;     // n_origs x 3
    uint32_t n_origs;       // 1 or n
    uint32_t n;             // rays per pose
    float range_min, range_max;
    uint32_t width, height; // scan raster (buffer id = vid*width + hid); used for the coherent tile order
    uint32_t sim_opts;      // b2_rcc_set_sim_options (SURVEY A.3): bit 0 tfar = +inf instead of range.max; bit 1 a closest hit below range.min is a miss; bit 2 misses filled with zeros instead of NaN
};
B2_DEV float sim_tfar(const RayModel& m) { return (m.sim_opts & 1u) ? u2f(0x7f800000u) : m.range_max; }
B2_DEV bool sim_is_hit(const RayModel& m, const HitRec& h) { return h.face != B2_NOFACE && !((m.sim_opts & 2u) && h.t < m.range_min); }

// Rays are traced in 8x4 raster tiles (one tile per warp) instead of 32-long row segments: neighbouring rows/columns of a
// LiDAR / depth raster stay inside the same BVH subtrees, which shortens the warp's union of traversal paths.  Results are
// written at the original buffer id, so the order is invisible outside.
B2_DEV uint32_t tile_order(uint32_t k, uint32_t width, uint32_t height)
{
    if ((width & 7u) || (height & 3u)) return k;
    const uint32_t tile = k >> 5, within = k & 31u, tiles_per_row = width >> 3;
    const uint32_t hid = (tile % tiles_per_row) * 8u + (within & 7u);
    const uint32_t vid = (tile / tiles_per_row) * 4u + (within >> 3);
    return vid * width + hid;
}

struct ModelBuffers {
    float* pts; float* nrm; uint8_t* hits; uint32_t* faces; float* ranges;
};

// shared epilogue: hit record -> sensor-frame point / normal exactly like the oracle's orc_simulate
B2_DEV void hit_to_sensor(const BvhView& bvh, const HitRec& h, Q4 Rms, V3 dir_s, V3 orig_s, V3& p, V3& ns)
{
    const V3 ng = tri_ng(bvh, h.tri);
    p = v_add(v_scale(dir_s, h.t), orig_s);
    const V3 nm = v_normalize(ng);
    ns = q_rot(Rms, nm);
    if (v_dot(dir_s, ns) > 0.0f) ns = v_neg(ns);
    ns = v_normalize(ns);
}

// one ray of find(): trace + write the model buffers at index o
B2_DEV void find_one(const BvhView& bvh, Tf Tsm, const RayModel& model, uint32_t i, uint64_t o, const ModelBuffers& out)
{
    const Q4 Rms = q_conj(Tsm.R);
    const uint32_t oi = model.n_origs == 1 ? 0 : i;
    const V3 orig_s = mk3(model.origs[3 * oi], model.origs[3 * oi + 1], model.origs[3 * oi + 2]);
    const V3 dir_s = mk3(model.dirs[3 * i], model.dirs[3 * i + 1], model.dirs[3 * i + 2]);
    const RaySetup r = ray_setup(tf_apply(Tsm, orig_s), q_rot(Tsm.R, dir_s), bvh);
    HitRec h = trace_init(sim_tfar(model));
    uint32_t nn = 0, nt = 0;
    trace_closest<false>(bvh, r, h, nn, nt);
    if (sim_is_hit(model, h)) {
        V3 p, ns; hit_to_sensor(bvh, h, Rms, dir_s, orig_s, p, ns);
        out.pts[3 * o] = p.x; out.pts[3 * o + 1] = p.y; out.pts[3 * o + 2] = p.z;
        out.nrm[3 * o] = ns.x; out.nrm[3 * o + 1] = ns.y; out.nrm[3 * o + 2] = ns.z;
        out.hits[o] = 1; out.faces[o] = h.face; out.ranges[o] = h.t;
    } else {
        const float qnan = (model.sim_opts & 4u) ? 0.0f : u2f(0x7fc00000u);
        out.pts[3 * o] = qnan; out.pts[3 * o + 1] = qnan; out.pts[3 * o + 2] = qnan;
        out.nrm[3 * o] = qnan; out.nrm[3 * o + 1] = qnan; out.nrm[3 * o + 2] = qnan;
        out.hits[o] = 0; out.faces[o] = B2_NOFACE; out.ranges[o] = add(model.range_max, 1.0f);
    }
}

// bulk prefetch of slice `part` of `parts` of an array into L2 (UBLKPF): e.g. after a cold start the top of the tree then comes from
// L2 instead of one DRAM round trip per level.  16-byte granularity (a base that is not 16-byte aligned is not prefetched), fire and forget.
__device__ __forceinline__ void bulk_prefetch_slice(const void* base, uint64_t total, uint32_t part, uint32_t parts)
{
    if (reinterpret_cast<uintptr_t>(base) & 15u) return;
    const uint64_t per = ((total + parts - 1) / parts + 15ull) & ~15ull;
    const uint64_t beg = (uint64_t)part * per;
    if (beg < total) {
        const uint32_t bytes = (uint32_t)min(per, total - beg) & ~15u;
        const char* ptr = reinterpret_cast<const char*>(base) + beg;
        if (bytes) asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(ptr), "r"(bytes) : "memory");
    }
}
// mode 1: node array; mode 2: node array + leaf triangle records (the whole map: 85 MB for 1M triangles, more than the 50 MB L2 of an H100)
__device__ __forceinline__ void prefetch_map_l2(const BvhView& bvh, uint32_t n_nodes, uint32_t n_tris, int mode)
{
    if (threadIdx.x == 0 && mode >= 1) bulk_prefetch_slice(bvh.nodes, (uint64_t)n_nodes * (uint64_t)B2_NODE_BYTES, blockIdx.x, gridDim.x);
    if (threadIdx.x == 32 % blockDim.x && mode >= 2) bulk_prefetch_slice(bvh.tris, (uint64_t)n_tris * 48ull, blockIdx.x, gridDim.x);
}

#define B2_FIND_BLOCK 64
// profiling aid: when set (b2_rcc_debug_find_warp_times), lane 0 of the warp that traces a tile stores its {start, end} in %globaltimer nanoseconds
__device__ unsigned long long* g_find_warp_times = nullptr;
__device__ __forceinline__ unsigned long long globaltimer_ns() { unsigned long long t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)); return t; }

// 14 blocks per SM (72 registers).  16 blocks per SM (64 registers, twice the spill traffic) was measured slower on an H100 SXM (400 W power
// limit): with the shipped setting (no L2 prefetch), alternating runs of bench.py --no-extra gave a find alone of 49.6-50.0 vs 51.8-52.4 us and
// a C2 step of 81.2 vs 82.4-82.7 us; with the node-array prefetch on, 55 vs 60 us and 85.6 vs 90.0 us.
// One resident wave with a per-warp tile queue: the grid is the blocks that fit on the device at once (api.cu: find_slots).  Warp w traces
// tile w first, then takes tiles (8x4 rays) one after another from a per-handle ticket counter until the tickets pass the last tile: a warp
// that finishes early takes the next tile at once instead of idling beside the other warp of its block, and since every block is resident
// from the start, a dependent kernel that becomes resident early (k_icp_loop) never takes a slot a find block is waiting for.  The first
// tiles take no ticket because every warp asking for one at the same moment serialises on the counter's address (on an H100, tickets for
// the first tiles too delayed the median tile start by 1.3 us and made the C2 find ~4 us slower).
// Tickets: ticket k of a launch stands for tile warps + k, and every warp that traced a tile ends on one ticket past the last tile, so a
// launch takes exactly n_tiles tickets.  The host passes the counter's value at the launch (`ticket_base`) and advances its copy by
// n_tiles; no reset between launches.  k is an unsigned 32-bit difference, which stays right when the counter wraps around 2^32.
// Tile schedule (single-pose launches): the kernel ends with its slowest warp -- so the tiles that took longest in the PREVIOUS launch of
// this handle (same model, nearly the same pose: MICP-L corrects continuously) are handed out first.  Each tile leaves its duration (SM
// cycles from its ticket to its last write) in `tile_cost[tile]`; the ICP loop that follows the find turns the durations into the order
// `tile_perm` of the next launch (icp_loop.cuh: tile_perm_group, idle warps of one block).  Without a schedule tiles go in raster order.
// Purely a schedule: every tile is traced exactly once, at its own buffer index, so results do not depend on it.
__global__ void __launch_bounds__(B2_FIND_BLOCK, 14) k_rcc_find(BvhView bvh, uint32_t n_nodes, uint32_t n_tris, int prefetch_mode, const b2_transform* __restrict__ Tbm_dev,
                                                                const IcpState* __restrict__ icp, b2_transform Tbm_val, b2_transform Tsb_val, RayModel model, uint32_t n_poses,
                                                                ModelBuffers out, int early_dependents, const uint16_t* __restrict__ tile_perm, uint32_t* __restrict__ tile_cost,
                                                                unsigned int* __restrict__ tickets, unsigned int ticket_base, uint32_t n_tiles)
{
    // let a dependent kernel launched with programmatic stream serialization (k_icp_loop) become resident as SMs drain; it still waits
    // (griddepcontrol.wait) for this grid to complete and flush before it reads the model buffers
    if (early_dependents) asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    prefetch_map_l2(bvh, n_nodes, n_tris, prefetch_mode);
    __shared__ uint32_t s_t0[B2_FIND_BLOCK / 32], s_tile[B2_FIND_BLOCK / 32];                     // the tile's start clock and number: nothing extra stays live across the trace
    const uint32_t lane = threadIdx.x & 31u, warps = gridDim.x * (B2_FIND_BLOCK / 32u);
    uint32_t t = (blockIdx.x * B2_FIND_BLOCK + threadIdx.x) >> 5;                                  // first tile: the warp's own index, no ticket
    while (t < n_tiles) {
        const uint32_t tile = tile_perm ? (uint32_t)tile_perm[t] : t;                               // n_poses == 1 with a schedule; a permutation of the tiles
        if (lane == 0u) s_tile[threadIdx.x >> 5] = tile;
        if (tile_cost && lane == 0u) { uint32_t c; asm volatile("mov.u32 %0, %%clock;" : "=r"(c)); s_t0[threadIdx.x >> 5] = c; }
        if (g_find_warp_times && lane == 0u) g_find_warp_times[2 * (uint64_t)tile] = globaltimer_ns();
        const uint64_t gid = ((uint64_t)tile << 5) | (threadIdx.x & 31u);
        const uint32_t pose = (uint32_t)(gid / model.n);
        if (pose < n_poses) {
            const uint32_t i = tile_order((uint32_t)(gid % model.n), model.width, model.height);
            Tf Tbm;
            if (icp) Tbm = tf_mul(tf_load(&icp->Tom), tf_load(&icp->Tbo));           // MICPSensor.hpp:148
            else if (Tbm_dev) Tbm = tf_load(Tbm_dev + pose);
            else Tbm = tf_from_pod(Tbm_val);
            find_one(bvh, tf_mul(Tbm, tf_from_pod(Tsb_val)), model, i, (uint64_t)pose * model.n + i, out);
        }
        __syncwarp();
        if ((threadIdx.x & 31u) == 0u) {
            const uint32_t done = s_tile[threadIdx.x >> 5];
            if (tile_cost) { uint32_t c; asm volatile("mov.u32 %0, %%clock;" : "=r"(c)); tile_cost[done] = c - s_t0[threadIdx.x >> 5]; }
            if (g_find_warp_times) g_find_warp_times[2 * (uint64_t)done + 1] = globaltimer_ns();
        }
        uint32_t k = 0;
        if (lane == 0u) k = atomicAdd(tickets, 1u) - ticket_base;
        t = warps + __shfl_sync(0xffffffffu, k, 0);
    }
}

#ifdef __CUDACC__
// the tile order before any durations are known; also what a launch falls back to when the loop that should have sorted never ran
__global__ void k_perm_identity(uint16_t* __restrict__ perm, uint32_t n)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) perm[i] = (uint16_t)i;
}
#endif

// ---------------------------------------------------------------------------------------------------------------------
// CPCEmbree::find (CPCEmbree.cpp:17-43): one thread per dataset point (the mask is NOT consulted, as in the reference);
//   Pm = Tsm * d_i;  cp = closestPoint(Pm);  hits = cp.d <= max_dist;  points = Tms * cp.p;  normals = Tms.R * cp.n
// The model buffers get one entry per dataset point, so computeCrossStatistics / the ICP loop run unchanged on them.
// ---------------------------------------------------------------------------------------------------------------------
B2_DEV void cpc_find_one(const BvhView& bvh, Tf Tsm, Tf Tms, const float* __restrict__ dpts, float max_dist, uint32_t i, const ModelBuffers& out)
{
    const V3 q = tf_apply(Tsm, mk3(dpts[3 * i], dpts[3 * i + 1], dpts[3 * i + 2]));
    CpBest best; uint32_t nn = 0, nt = 0;
    closest_point<false>(bvh, q, best, nn, nt);
    if (best.face != B2_NOFACE) {
        const float d = sqrtf(best.d2);
        const V3 p = tf_apply(Tms, best.p);
        const V3 ns = q_rot(Tms.R, v_normalize(tri_ng(bvh, best.tri)));
        out.pts[3 * i] = p.x; out.pts[3 * i + 1] = p.y; out.pts[3 * i + 2] = p.z;
        out.nrm[3 * i] = ns.x; out.nrm[3 * i + 1] = ns.y; out.nrm[3 * i + 2] = ns.z;
        out.hits[i] = d <= max_dist ? 1 : 0; out.faces[i] = best.face; out.ranges[i] = d;
    } else {
        const float qnan = u2f(0x7fc00000u);
        out.pts[3 * i] = qnan; out.pts[3 * i + 1] = qnan; out.pts[3 * i + 2] = qnan;
        out.nrm[3 * i] = qnan; out.nrm[3 * i + 1] = qnan; out.nrm[3 * i + 2] = qnan;
        out.hits[i] = 0; out.faces[i] = B2_NOFACE; out.ranges[i] = u2f(0x7f800000u);
    }
}

#ifdef __CUDACC__
__global__ void __launch_bounds__(B2_FIND_BLOCK) k_cpc_find(BvhView bvh, uint32_t n_nodes, uint32_t n_tris, int prefetch_mode, const IcpState* __restrict__ icp,
                                                            b2_transform Tbm_val, b2_transform Tsb_val, const float* __restrict__ dpts, uint32_t n, float max_dist,
                                                            ModelBuffers out, const uint8_t* __restrict__ skip_mask)
{
    prefetch_map_l2(bvh, n_nodes, n_tris, prefetch_mode);
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    if (skip_mask && !(skip_mask[i] > 0)) {
        // b2_rcc_set_cpc_options(skip_masked): a masked-out dataset point (e.g. a dropped beam unpacked to range.max + 1, far outside the map) never
        // enters the statistics; its query is the most expensive of the scan (2 % of the points cost a third of the kernel: one such lane keeps
        // its whole warp) and is skipped -- the entry reads hits = 0, NaN, like a miss.  Off by default: the reference queries every point.
        const float qnan = u2f(0x7fc00000u);
        out.pts[3 * i] = qnan; out.pts[3 * i + 1] = qnan; out.pts[3 * i + 2] = qnan;
        out.nrm[3 * i] = qnan; out.nrm[3 * i + 1] = qnan; out.nrm[3 * i + 2] = qnan;
        out.hits[i] = 0; out.faces[i] = B2_NOFACE; out.ranges[i] = u2f(0x7f800000u);
        return;
    }
    const Tf Tbm = icp ? tf_mul(tf_load(&icp->Tom), tf_load(&icp->Tbo)) : tf_from_pod(Tbm_val);
    const Tf Tsm = tf_mul(Tbm, tf_from_pod(Tsb_val));
    cpc_find_one(bvh, Tsm, tf_inv(Tsm), dpts, max_dist, i, out);
}
#endif

// ---------------------------------------------------------------------------------------------------------------------
// refit of ONE node of the wide tree (b2_mesh_refit, lbvh.cuh:k_bvh8_refit_level): leaf children re-fetch their triangles, inner children
// take the union of the (already refitted) child node's boxes
// ---------------------------------------------------------------------------------------------------------------------
B2_DEV void bvh8_refit_node(uint32_t t, B2Node8* nodes, B2Tri* tris, const float* verts, const uint32_t* faces)
{
    B2Node8& nd = nodes[t];
    const float inf = u2f(0x7f800000u);
    for (int s = 0; s < 8; s++) {
        const uint32_t meta = nd.meta[s];
        float lo[3] = {inf, inf, inf}, hi[3] = {-inf, -inf, -inf};
        if ((nd.imask() >> s) & 1u) {
            const B2Node8& ch = nodes[nd.child_base + popc32(nd.imask() & ((1u << s) - 1u))];
            for (int c = 0; c < 8; c++) {
                if (!ch.meta[c]) continue;
                for (int k = 0; k < 3; k++) { lo[k] = fminf(lo[k], ch.lo[k][c]); hi[k] = fmaxf(hi[k], ch.hi[k][c]); }
            }
        } else if (meta) {
            const uint32_t cnt = (meta >> 5) == 7u ? 3u : ((meta >> 5) == 3u ? 2u : 1u), first = nd.tri_base + (meta & 0x1fu);
            for (uint32_t j = 0; j < cnt; j++) {
                B2Tri& tr = tris[first + j];
                const uint32_t f = tr.face_id;
                const float* a = verts + 3 * (size_t)faces[3 * (size_t)f + 0];
                const float* b = verts + 3 * (size_t)faces[3 * (size_t)f + 1];
                const float* c = verts + 3 * (size_t)faces[3 * (size_t)f + 2];
                for (int k = 0; k < 3; k++) {
                    tr.v0[k] = a[k]; tr.v1[k] = b[k]; tr.v2[k] = c[k];
                    lo[k] = fminf(lo[k], fminf(fminf(a[k], b[k]), c[k])); hi[k] = fmaxf(hi[k], fmaxf(fmaxf(a[k], b[k]), c[k]));
                }
            }
        }
        for (int k = 0; k < 3; k++) { nd.lo[k][s] = lo[k]; nd.hi[k][s] = hi[k]; }
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// scan-vs-map segmentation (SURVEY 8f4): classification loop of ScanMapSegmentationEmbreeNode
// (rmcl_ros/src/nodes/filter/scan_map_segmentation_embree.cpp:110-187) on the model buffers left by find() and the real ranges.
// label 0: neither cloud, 1: outlier_scan (point = preal), 2: outlier_map (point = pint)
// ---------------------------------------------------------------------------------------------------------------------
B2_DEV uint32_t segment_classify(const RayModel& model, uint32_t i, float rr, float rs, V3 nsim, float min_scan, float min_map, V3& p)
{
    const uint32_t oi = model.n_origs == 1 ? 0 : i;
    const V3 dir = mk3(model.dirs[3 * i], model.dirs[3 * i + 1], model.dirs[3 * i + 2]);
    const V3 orig = mk3(model.origs[3 * oi], model.origs[3 * oi + 1], model.origs[3 * oi + 2]);
    const bool real_valid = (model.range_min <= rr) && (rr <= model.range_max);           // model.range.inside, :121-122
    const bool sim_valid = (model.range_min <= rs) && (rs <= model.range_max);
    p = mk3(0.f, 0.f, 0.f);
    if (real_valid) {
        const V3 preal = v_add(v_scale(dir, rr), orig);                                   // :126
        if (!sim_valid) { p = preal; return 1u; }                                         // :164-171
        const V3 pint = v_scale(dir, rs);                                                 // :130 (no origin, as in the reference)
        const V3 nint = v_normalize(nsim);                                                // :131-132
        const float spd = v_dot(v_sub(preal, pint), nint);                                // :134
        const V3 pmesh = v_add(preal, v_scale(nint, spd));                                // :135
        const float plane_distance = v_l2norm(v_sub(pmesh, preal));                       // :136
        if (rr < rs) { if (plane_distance > min_scan) { p = preal; return 1u; } }         // :138-149
        else         { if (plane_distance > min_map)  { p = pint;  return 2u; } }         // :150-161
        return 0u;
    }
    if (sim_valid) { p = v_add(v_scale(dir, rs), orig); return 2u; }                      // :173-182
    return 0u;
}

#ifdef __CUDACC__
#define B2_SEG_BLOCK 256
// pass 1 (counts != nullptr, out_* == nullptr): per-block counts of both classes.  pass 3: recompute and write each outlier at
// block offset + its rank inside the block, so both clouds come out in raster order like the reference's push_back loop.
__global__ void __launch_bounds__(B2_SEG_BLOCK) k_segment(RayModel model, const float* __restrict__ ranges_real, const float* __restrict__ ranges_sim,
                                                          const float* __restrict__ normals_sim, float min_scan, float min_map, uint32_t* __restrict__ counts,
                                                          const uint32_t* __restrict__ offsets, float* __restrict__ out_scan, float* __restrict__ out_map, uint8_t* __restrict__ labels)
{
    __shared__ uint32_t s_cnt[2][B2_SEG_BLOCK / 32];
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x, lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
    uint32_t label = 0u; V3 p = mk3(0.f, 0.f, 0.f);
    if (i < model.n) label = segment_classify(model, i, ranges_real[i], ranges_sim[i], mk3(normals_sim[3 * i], normals_sim[3 * i + 1], normals_sim[3 * i + 2]), min_scan, min_map, p);
    const uint32_t b1 = __ballot_sync(0xffffffffu, label == 1u), b2 = __ballot_sync(0xffffffffu, label == 2u);
    if (lane == 0) { s_cnt[0][warp] = __popc(b1); s_cnt[1][warp] = __popc(b2); }
    __syncthreads();
    uint32_t before1 = 0u, before2 = 0u, tot1 = 0u, tot2 = 0u;
    #pragma unroll
    for (uint32_t w = 0; w < B2_SEG_BLOCK / 32; w++) { if (w < warp) { before1 += s_cnt[0][w]; before2 += s_cnt[1][w]; } tot1 += s_cnt[0][w]; tot2 += s_cnt[1][w]; }
    if (!out_scan) {
        if (threadIdx.x == 0) { counts[2 * blockIdx.x] = tot1; counts[2 * blockIdx.x + 1] = tot2; }
        return;
    }
    const uint32_t lt = (1u << lane) - 1u;
    if (label == 1u) { const size_t o = (size_t)offsets[2 * blockIdx.x] + before1 + __popc(b1 & lt); out_scan[3 * o] = p.x; out_scan[3 * o + 1] = p.y; out_scan[3 * o + 2] = p.z; }
    if (label == 2u) { const size_t o = (size_t)offsets[2 * blockIdx.x + 1] + before2 + __popc(b2 & lt); out_map[3 * o] = p.x; out_map[3 * o + 1] = p.y; out_map[3 * o + 2] = p.z; }
    if (labels && i < model.n) labels[i] = (uint8_t)label;
}
// pass 2: exclusive scan of the per-block counts (one block; a few thousand entries at most), totals to totals[0..1]
__global__ void __launch_bounds__(1024) k_segment_scan(const uint32_t* __restrict__ counts, uint32_t n_blocks, uint32_t* __restrict__ offsets, uint32_t* __restrict__ totals)
{
    __shared__ uint32_t s[2][1024];
    __shared__ uint32_t carry[2];
    if (threadIdx.x == 0) { carry[0] = 0u; carry[1] = 0u; }
    __syncthreads();
    for (uint32_t base = 0; base < n_blocks; base += 1024u) {
        const uint32_t b = base + threadIdx.x;
        const uint32_t v0 = b < n_blocks ? counts[2 * b] : 0u, v1 = b < n_blocks ? counts[2 * b + 1] : 0u;
        s[0][threadIdx.x] = v0; s[1][threadIdx.x] = v1;
        __syncthreads();
        for (uint32_t d = 1; d < 1024u; d <<= 1) {                      // Hillis-Steele inclusive scan
            const uint32_t a0 = threadIdx.x >= d ? s[0][threadIdx.x - d] : 0u, a1 = threadIdx.x >= d ? s[1][threadIdx.x - d] : 0u;
            __syncthreads();
            s[0][threadIdx.x] += a0; s[1][threadIdx.x] += a1;
            __syncthreads();
        }
        if (b < n_blocks) { offsets[2 * b] = carry[0] + s[0][threadIdx.x] - v0; offsets[2 * b + 1] = carry[1] + s[1][threadIdx.x] - v1; }
        __syncthreads();
        if (threadIdx.x == 1023) { carry[0] += s[0][1023]; carry[1] += s[1][1023]; }
        __syncthreads();
    }
    if (threadIdx.x == 0) { totals[0] = carry[0]; totals[1] = carry[1]; }
}
#endif

// ---------------------------------------------------------------------------------------------------------------------
// Correspondences*::computeCrossStatistics (CorrespondencesCPU.cpp:10-39): N-element masked reduction -> CrossStatistics.
// Deterministic: per-block partials, the last block to finish sums them in block order.  With `icp` set, the last block also
// performs the rest of the inner iteration (frame changes, Umeyama, compose) so one correctOnce needs 1 + iterations launches.
// ---------------------------------------------------------------------------------------------------------------------
#define B2_RED_BLOCK 256
__global__ void __launch_bounds__(B2_RED_BLOCK) k_p2l_reduce(const float* __restrict__ dpts, const uint8_t* __restrict__ dmask,
                                                             const float* __restrict__ mpts, const float* __restrict__ mnrm, const uint8_t* __restrict__ mmask,
                                                             uint32_t n, b2_transform Tpre_val, float max_dist_val, IcpState* icp,
                                                             double* __restrict__ partials, unsigned int* __restrict__ ticket, b2_cross_stats* __restrict__ out)
{
    __shared__ double smem[(B2_NACC + 1) * (B2_RED_BLOCK / 32)];
    __shared__ bool is_last;
    const long long c0 = clock64();
    const Tf Tpre = icp ? tf_load(&icp->T_snew_sold) : tf_from_pod(Tpre_val);
    const float max_dist = icp ? icp->max_dist : max_dist_val;
    P2LAcc acc; acc_zero(acc);
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        // all eleven loads are issued before the first use (no mask-dependent early-out): one memory round trip per element
        const uint8_t dm = dmask[i], mm = mmask[i];
        const V3 d = mk3(dpts[3 * i], dpts[3 * i + 1], dpts[3 * i + 2]);
        const V3 I = mk3(mpts[3 * i], mpts[3 * i + 1], mpts[3 * i + 2]);
        const V3 N = mk3(mnrm[3 * i], mnrm[3 * i + 1], mnrm[3 * i + 2]);
        V3 D, M;
        if ((dm > 0) && (mm > 0) && p2l_pair(Tpre, d, I, N, max_dist, D, M)) acc_add_pair(acc, D, M);
    }
    block_reduce_acc<B2_RED_BLOCK>(acc, smem);
    if (threadIdx.x == 0) {
        double* p = partials + (size_t)blockIdx.x * (B2_NACC + 1);
        for (int i = 0; i < B2_NACC; i++) p[i] = acc.v[i];
        p[B2_NACC] = (double)acc.n;
        __threadfence();
        const unsigned int t = atomicAdd(ticket, 1u);
        is_last = (t == gridDim.x - 1);
    }
    __syncthreads();
    if (!is_last) return;
    __threadfence();
    const long long c1 = clock64();
    // deterministic parallel sum of the block partials: thread (g, i) adds value i of blocks g, g+16, ...; then the 16 group sums in order
    __shared__ double s_part[16][B2_NACC + 1];
    {
        const uint32_t i = threadIdx.x & 15u, g = threadIdx.x >> 4;           // 256 threads = 16 groups x 16 values
        double a = 0.0;
        for (uint32_t b = g; b < gridDim.x; b += 16u) a += __ldcg(partials + (size_t)b * (B2_NACC + 1) + i);
        s_part[g][i] = a;
    }
    __syncthreads();
    if (threadIdx.x < B2_NACC + 1) {
        double a = 0.0;
        #pragma unroll
        for (int g = 0; g < 16; g++) a += s_part[g][threadIdx.x];
        s_part[0][threadIdx.x] = a;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        const long long c2 = clock64();
        const CStats st = acc_finalize(&s_part[0][0], (uint32_t)(s_part[0][B2_NACC] + 0.5));
        if (out) cs_store(out, st);
        const long long c3 = clock64();
        if (icp) {
            icp_step(icp, st);
            const long long c4 = clock64();
            icp->dbg[0] = (unsigned long long)(c1 - c0); icp->dbg[1] = (unsigned long long)(c2 - c1); icp->dbg[2] = (unsigned long long)(c3 - c2);
            icp->dbg[3] = (unsigned long long)(c4 - c3);
        }
        *ticket = 0u;
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// v1 batched correct(): fused trace -> P2L gate -> per-block partial statistics (no model buffers written)
// grid = n_poses * blocks_per_pose; each block handles `rays_per_block` consecutive rays of one pose
// ---------------------------------------------------------------------------------------------------------------------
#define B2_FUSED_BLOCK 128
// 6 blocks per SM (80 registers, a few spilled values): 2.5 % faster than the uncapped 128 registers / 4 blocks (3.06 -> 2.98 ms per 1000-pose call)
__global__ void __launch_bounds__(B2_FUSED_BLOCK, 6) k_rcc_fused_batch(BvhView bvh, const b2_transform* __restrict__ Tbm_dev, b2_transform Tsb_val, RayModel model,
                                                                    const float* __restrict__ dpts, const uint8_t* __restrict__ dmask, float max_dist,
                                                                    uint32_t blocks_per_pose, uint32_t rays_per_block, double* __restrict__ partials)
{
    __shared__ double smem[(B2_NACC + 1) * (B2_FUSED_BLOCK / 32)];
    const uint32_t pose = blockIdx.x / blocks_per_pose, chunk = blockIdx.x % blocks_per_pose;
    const Tf Tsm = tf_mul(tf_load(Tbm_dev + pose), tf_from_pod(Tsb_val));
    const Q4 Rms = q_conj(Tsm.R);
    const Tf I = tf_identity();
    P2LAcc acc; acc_zero(acc);
    const uint32_t begin = chunk * rays_per_block;
    const uint32_t end = min(begin + rays_per_block, model.n);
    for (uint32_t k = begin + threadIdx.x; k < end; k += blockDim.x) {
        const uint32_t i = tile_order(k, model.width, model.height);
        if (!(dmask[i] > 0)) continue;
        const uint32_t oi = model.n_origs == 1 ? 0 : i;
        const V3 orig_s = mk3(model.origs[3 * oi], model.origs[3 * oi + 1], model.origs[3 * oi + 2]);
        const V3 dir_s = mk3(model.dirs[3 * i], model.dirs[3 * i + 1], model.dirs[3 * i + 2]);
        const RaySetup r = ray_setup(tf_apply(Tsm, orig_s), q_rot(Tsm.R, dir_s), bvh);
        HitRec h = trace_init(sim_tfar(model));
        uint32_t nn = 0, nt = 0;
        trace_closest<false>(bvh, r, h, nn, nt);
        if (!sim_is_hit(model, h)) continue;
        V3 p, ns; hit_to_sensor(bvh, h, Rms, dir_s, orig_s, p, ns);
        V3 D, M;
        if (p2l_pair(I, mk3(dpts[3 * i], dpts[3 * i + 1], dpts[3 * i + 2]), p, ns, max_dist, D, M)) acc_add_pair(acc, D, M);
    }
    block_reduce_acc<B2_FUSED_BLOCK>(acc, smem);
    if (threadIdx.x == 0) {
        double* p = partials + (size_t)blockIdx.x * (B2_NACC + 1);
        for (int i = 0; i < B2_NACC; i++) p[i] = acc.v[i];
        p[B2_NACC] = (double)acc.n;
    }
}

// stage-split twin of k_rcc_fused_batch for the v1 benchmark() call ({sim, red, svd} seconds, lidar_corrector_optix_benchmark.cpp:143-155):
// the reduction alone over model buffers that k_rcc_find wrote for ALL poses (pose-major), same partial layout as the fused kernel
__global__ void __launch_bounds__(B2_FUSED_BLOCK) k_p2l_batch(const float* __restrict__ mpts, const float* __restrict__ mnrm, const uint8_t* __restrict__ mhits, uint32_t n,
                                                             const float* __restrict__ dpts, const uint8_t* __restrict__ dmask, float max_dist,
                                                             uint32_t blocks_per_pose, uint32_t rays_per_block, double* __restrict__ partials)
{
    __shared__ double smem[(B2_NACC + 1) * (B2_FUSED_BLOCK / 32)];
    const uint32_t pose = blockIdx.x / blocks_per_pose, chunk = blockIdx.x % blocks_per_pose;
    const Tf I = tf_identity();
    P2LAcc acc; acc_zero(acc);
    const uint32_t begin = chunk * rays_per_block, end = min(begin + rays_per_block, n);
    for (uint32_t i = begin + threadIdx.x; i < end; i += blockDim.x) {
        const size_t o = (size_t)pose * n + i;
        if (!(dmask[i] > 0) || !(mhits[o] > 0)) continue;
        V3 D, M;
        if (p2l_pair(I, mk3(dpts[3 * i], dpts[3 * i + 1], dpts[3 * i + 2]), mk3(mpts[3 * o], mpts[3 * o + 1], mpts[3 * o + 2]), mk3(mnrm[3 * o], mnrm[3 * o + 1], mnrm[3 * o + 2]), max_dist, D, M))
            acc_add_pair(acc, D, M);
    }
    block_reduce_acc<B2_FUSED_BLOCK>(acc, smem);
    if (threadIdx.x == 0) {
        double* p = partials + (size_t)blockIdx.x * (B2_NACC + 1);
        for (int i = 0; i < B2_NACC; i++) p[i] = acc.v[i];
        p[B2_NACC] = (double)acc.n;
    }
}

// per pose: sum the block partials in order -> stats_s -> stats_b = Tsb * stats_s -> Umeyama
__global__ void k_umeyama_from_partials(const double* __restrict__ partials, uint32_t blocks_per_pose, uint32_t n_poses, b2_transform Tsb_val,
                                        b2_transform* __restrict__ Tdelta, uint32_t* __restrict__ ncorr, b2_cross_stats* __restrict__ stats_b_out)
{
    const uint32_t pose = blockIdx.x * blockDim.x + threadIdx.x;
    if (pose >= n_poses) return;
    double v[B2_NACC]; for (int i = 0; i < B2_NACC; i++) v[i] = 0.0;
    double cnt = 0.0;
    for (uint32_t b = 0; b < blocks_per_pose; b++) {
        const double* p = partials + ((size_t)pose * blocks_per_pose + b) * (B2_NACC + 1);
        for (int i = 0; i < B2_NACC; i++) v[i] += p[i];
        cnt += p[B2_NACC];
    }
    const CStats ss = acc_finalize(v, (uint32_t)(cnt + 0.5));
    const CStats sb = cs_transform(tf_from_pod(Tsb_val), ss);
    const Tf T = umeyama_dev(sb);
    if (Tdelta) tf_store(Tdelta + pose, T);
    if (ncorr) ncorr[pose] = sb.n;
    if (stats_b_out) cs_store(stats_b_out + pose, sb);
}

__global__ void k_umeyama_batch(const b2_cross_stats* __restrict__ stats, uint32_t n, b2_transform* __restrict__ out)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    tf_store(out + i, umeyama_dev(cs_load(stats + i)));
}

// ---------------------------------------------------------------------------------------------------------------------
// particle filter: PCDSensorUpdaterEmbree::update hot loop (PCDSensorUpdaterEmbree.cpp:290-342) in ONE launch.
// A block owns PPB particles x all beams.  Phase 1: every (particle, beam) ray is traced by some thread, its Gaussian
// evaluation stored in shared memory.  Phase 2: one thread per particle merges the evaluations IN BEAM ORDER
// (the reference's sequential FP32 Gaussian1D += order, quirk D6) and read-modify-writes the 36-byte attrs once.
// ---------------------------------------------------------------------------------------------------------------------
struct PfBeam { float ox, oy, oz, dx, dy, dz, range; uint32_t slot; };   // slot = original beam index (merge order)

B2_DEV void gaussian1d_add(b2_gaussian1d& a, float b_mean, float b_sigma, uint32_t b_n)
{
    const uint32_t n = a.n_meas + b_n;
    if (n == 0) return;
    const float w1 = dvd((float)a.n_meas, (float)n), w2 = dvd((float)b_n, (float)n);
    const float mean = add(mul(a.mean, w1), mul(b_mean, w2));
    const float d1 = sub(a.mean, mean), d2 = sub(b_mean, mean);
    const float sigma = add(add(mul(a.sigma, w1), mul(b_sigma, w2)), add(mul(mul(d1, d1), w1), mul(mul(d2, d2), w2)));
    a.mean = mean; a.sigma = sigma; a.n_meas = n;
}

// Gaussian evaluation of one (particle, beam) pair: sensorUpdate() up to `eval` (PCDSensorUpdaterEmbree.cpp:197-224)
template <int CORR>
B2_DEV float pf_eval_one(const BvhView& bvh, Tf Tsm, const PfBeam& b, const b2_pf_params& prm, float sigma_quad, double denom)
{
    const V3 orig_m = tf_apply(Tsm, mk3(b.ox, b.oy, b.oz));                                // RangeMeasurement.hpp:29-42
    const V3 dir_m = q_rot(Tsm.R, mk3(b.dx, b.dy, b.dz));
    if (CORR == 1) {
        // evaluate_cpc (:88-95): error = distance of meas_m.mean() = orig + dir*range (RangeMeasurement.hpp:17-20) to the surface
        CpBest best; uint32_t nn = 0, nt = 0;
        closest_point<false>(bvh, v_add(orig_m, v_scale(dir_m, b.range)), best, nn, nt);
        const float error = best.face != B2_NOFACE ? sqrtf(best.d2) : u2f(0x7f800000u);
        const float arg = dvd(dvd(-mul(error, error), sigma_quad), 2.0f);                  // :224
        return (float)(exp((double)arg) / denom);
    }
    const bool real_hit = (prm.range_min <= b.range) && (b.range <= prm.range_max);        // :27
    const RaySetup r = ray_setup(orig_m, dir_m, bvh);
    HitRec h = trace_init(u2f(0x7f800000u));                                               // tfar = +inf (:38)
    uint32_t nn = 0, nt = 0;
    trace_closest<false>(bvh, r, h, nn, nt);
    const bool sim_hit = (h.face != B2_NOFACE) && (h.t > prm.range_min);                   // :47
    float error;
    if (sim_hit) {
        if (real_hit) {
            V3 n = tri_ng(bvh, h.tri);
            if (prm.ng_mode == 1) n = v_normalize(n);
            const V3 preal = v_add(orig_m, v_scale(dir_m, b.range));
            const V3 pint = v_add(orig_m, v_scale(dir_m, h.t));
            error = fabsf(v_dot(v_sub(pint, preal), n));                                   // :54-68
        } else error = prm.real_miss_sim_hit_error;
    } else error = real_hit ? prm.real_hit_sim_miss_error : prm.real_miss_sim_miss_error;
    const float arg = dvd(dvd(-mul(error, error), sigma_quad), 2.0f);                      // :224
    return (float)(exp((double)arg) / denom);
}
B2_DEV void pf_constants(const b2_pf_params& prm, float& sigma_quad, double& denom)
{
    sigma_quad = mul(prm.dist_sigma, prm.dist_sigma);
    denom = sqrt((double)mul(2.0f, sigma_quad) * 3.14159265358979323846);                  // sqrt(2*sq*M_PI)
}
// merge the evaluations of one particle in beam order (:232-238)
B2_DEV void pf_merge(b2_gaussian1d& lk, const float* e, uint32_t n_beams)
{
    for (uint32_t b = 0; b < n_beams; b++) {
        gaussian1d_add(lk, e[b], 0.0f, 1u);
        lk.n_meas = lk.n_meas < 10000u ? lk.n_meas : 10000u;                               // MAX_N_MEAS
    }
}

#define B2_PF_BLOCK 128
// 72 registers (7 blocks/SM) measured 8 % faster than the uncapped 84 (6 blocks/SM); a persistent-lane variant with dynamic ray fetch
// (idle lanes claim new rays) was measured SLOWER (2.3 vs 3.3 G rays/s: the extra live state and warp votes cost more than the refill gains)
// MAP 0: consecutive lanes = consecutive beams of one particle (rays of a warp share their origin: the mapping for particle sets spread over
// the map, where no two particles are close).  MAP 1: consecutive lanes = the particles of the block, same beam -- coherent when neighbouring
// particles have nearly the same pose, i.e. for a converged cloud after `order` sorted it by (heading, cell): 1.7x faster there, slower on
// spread-out sets (scripts/exp_pf_mapping.py); the host picks by timing both (api.cu).  `order` (may be nullptr) = particle processed at
// position p.  The per-particle merge runs over the beams in their original order either way: results are bit-identical.
template <int CORR, int MAP>
__global__ void __launch_bounds__(B2_PF_BLOCK, 7) k_pf_update(BvhView bvh, const b2_transform* __restrict__ poses, b2_particle_attr* __restrict__ attrs, uint32_t n_particles,
                                                           b2_transform Tsb_val, const PfBeam* __restrict__ beams, uint32_t n_beams, b2_pf_params prm, uint32_t ppb,
                                                           const uint32_t* __restrict__ order)
{
    extern __shared__ float s_eval[];            // [ppb][n_beams]
    const uint32_t p0 = blockIdx.x * ppb;
    const uint32_t np = min(ppb, n_particles - p0);
    float sigma_quad; double denom; pf_constants(prm, sigma_quad, denom);
    const Tf Tsb = tf_from_pod(Tsb_val);
    const uint32_t total = np * n_beams;
    for (uint32_t w = threadIdx.x; w < total; w += blockDim.x) {
        const uint32_t pl = MAP ? w % np : w / n_beams, bi = MAP ? w / np : w % n_beams;
        const uint32_t pi = order ? order[p0 + pl] : p0 + pl;
        const Tf Tsm = tf_mul(tf_load(poses + pi), Tsb);                                   // :337-338
        const PfBeam b = beams[bi];
        s_eval[pl * n_beams + b.slot] = pf_eval_one<CORR>(bvh, Tsm, b, prm, sigma_quad, denom);
    }
    __syncthreads();
    if (threadIdx.x < np) {
        b2_particle_attr* ap = attrs + (order ? order[p0 + threadIdx.x] : p0 + threadIdx.x);
        b2_gaussian1d lk = ap->likelihood;
        pf_merge(lk, s_eval + threadIdx.x * n_beams, n_beams);
        ap->likelihood = lk;
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// Truncated distance field of the map (b2_dfield_*; no reference counterpart, SURVEY appendix K) and the particle filter's sensor update
// from it (b2_pf_sensor_update_field).
// FIELD (origin, h, dims, trunc): node (i, j, k) sits at x = add(origin.x, mul((float)i, h)) (likewise y, z) and holds
//   v = min(sqrtf(d2), trunc), d2 the closest point's result (trace.cuh) at that position; no face within trunc gives trunc.  Every stored
//   value equals orc_closest_point's d_out clamped at trunc, whatever the BVH and builder: the bounded query (trace.cuh) returns the same
//   clamped value as the unbounded one.
// LAYOUT: sparse bricks of 8^3 cells.  A dense uint32 index over bdims = ceil((dims - 1) / 8) bricks per axis (z-major, x fastest) holds each
//   brick's slot or B2_NOBRICK; an allocated brick stores its 9^3 nodes 8b .. 8b + 8 per axis (z, y, x; x fastest), so the 8 corners of a
//   cell always sit in one brick.  A brick is allocated iff the distance from its centre node 8b + 4 is < trunc + 8h (bounded query at that
//   limit: strict, so that the bounded and the unbounded query decide alike).  Its nodes lie within 4 sqrt(3) h < 8h of the centre and the
//   distance is 1-Lipschitz, so every node of an unallocated brick has value trunc (up to float rounding of the positions, far below h).
// LOOKUP at p: g = mul(sub(p, origin), inv_h) per axis (inv_h = the float 1 / h).  Inside iff 0 <= g <= dims - 1 on every axis; the cell is
//   min(floor(g), dims - 2), t = sub(g, cell); trilinear in the fixed order x, y, z, each lerp add(mul(a, sub(1, t)), mul(b, t)).  An
//   unallocated brick or a finite point outside the box gives trunc; a non-finite point gives +inf (the closest-point update's miss).
// ACCURACY: min(d, trunc) is 1-Lipschitz and the trilinear weights w_i of the corners c_i satisfy sum w_i |c_i - p|^2 = h^2 sum_k u_k (1 - u_k)
//   <= 3h^2 / 4, so |field(p) - min(d_exact(p), trunc)| <= (sqrt(3) / 2) h, plus float rounding of the nodes and of the interpolation.
// ---------------------------------------------------------------------------------------------------------------------
#define B2_NOBRICK 0xFFFFFFFFu
#define B2_DF_NODES 729u                 // 9^3 nodes per brick

struct DfieldView {
    const uint32_t* index;               // [bz][by][bx] -> brick slot or B2_NOBRICK
    const float* bricks;                 // [slot][9][9][9]
    float ox, oy, oz, h, inv_h, trunc;
    uint32_t dx, dy, dz;                 // nodes per axis (>= 2)
    uint32_t bx, by, bz;                 // bricks per axis
};

// grid of a field over the box [lo, hi] (host): cells per axis max(1, ceil((hi - lo) / h)) in float64, dims = cells + 1, bricks per axis
// ceil(cells / 8).  Returns nullptr, or why the grid is refused: non-finite or empty box, h or trunc not finite and > 0, more than 2^24 nodes
// on an axis counting the last brick's far face (node coordinates must be exact in float), more than 2^32 - 2 bricks (B2_NOBRICK stays free).
inline const char* df_grid(const float lo[3], const float hi[3], float h, float trunc, DfieldView* f, uint64_t* n_bricks)
{
    if (!(std::isfinite(h) && h > 0.0f)) return "resolution must be finite and > 0";
    if (!(std::isfinite(trunc) && trunc > 0.0f)) return "truncation must be finite and > 0";
    uint64_t cells[3], bricks[3];
    for (int k = 0; k < 3; k++) {
        if (!(std::isfinite(lo[k]) && std::isfinite(hi[k]))) return "bounds must be finite";
        if (!(lo[k] < hi[k])) return "bb_min must be below bb_max on every axis";
        const double c = std::ceil(((double)hi[k] - (double)lo[k]) / (double)h);
        if (!(c <= 16777216.0)) return "more than 2^24 nodes on an axis";
        cells[k] = c < 1.0 ? 1u : (uint64_t)c;
        bricks[k] = (cells[k] + 7u) / 8u;
        if (8u * bricks[k] + 1u > 16777216u) return "more than 2^24 nodes on an axis";
    }
    const uint64_t total = bricks[0] * bricks[1] * bricks[2];
    if (total > 0xFFFFFFFEull) return "more than 2^32 - 2 bricks";
    f->index = nullptr; f->bricks = nullptr;
    f->ox = lo[0]; f->oy = lo[1]; f->oz = lo[2]; f->h = h; f->inv_h = 1.0f / h; f->trunc = trunc;
    f->dx = (uint32_t)cells[0] + 1u; f->dy = (uint32_t)cells[1] + 1u; f->dz = (uint32_t)cells[2] + 1u;
    f->bx = (uint32_t)bricks[0]; f->by = (uint32_t)bricks[1]; f->bz = (uint32_t)bricks[2];
    *n_bricks = total;
    return nullptr;
}

B2_DEV float df_coord(float o, uint32_t i, float h) { return add(o, mul((float)i, h)); }
// the build's limits: the allocation distance ta = add(trunc, mul(8, h)), its square and trunc2 = mul(trunc, trunc)
B2_DEV void df_limits(const DfieldView& f, float& ta, float& ta2, float& trunc2) { ta = add(f.trunc, mul(8.0f, f.h)); ta2 = mul(ta, ta); trunc2 = mul(f.trunc, f.trunc); }

// value of the node at global node coordinates (i, j, k); trunc2 = mul(trunc, trunc)
B2_DEV float df_node_value(const BvhView& bvh, const DfieldView& f, uint32_t i, uint32_t j, uint32_t k, float trunc2)
{
    CpBest best; uint32_t nn = 0, nt = 0;
    closest_point<false, true>(bvh, mk3(df_coord(f.ox, i, f.h), df_coord(f.oy, j, f.h), df_coord(f.oz, k, f.h)), best, nn, nt, trunc2);
    return fminf(sqrtf(best.d2), f.trunc);
}

// allocation rule of brick (bi, bj, bk): ta = add(trunc, mul(8, h)), ta2 = mul(ta, ta)
B2_DEV bool df_brick_alloc(const BvhView& bvh, const DfieldView& f, uint32_t bi, uint32_t bj, uint32_t bk, float ta, float ta2)
{
    CpBest best; uint32_t nn = 0, nt = 0;
    closest_point<false, true>(bvh, mk3(df_coord(f.ox, 8u * bi + 4u, f.h), df_coord(f.oy, 8u * bj + 4u, f.h), df_coord(f.oz, 8u * bk + 4u, f.h)), best, nn, nt, ta2);
    return sqrtf(best.d2) < ta;
}

// node l (0 .. 728) of the brick with linear index id -> global node coordinates
B2_DEV void df_brick_node(const DfieldView& f, uint32_t id, uint32_t l, uint32_t& i, uint32_t& j, uint32_t& k)
{
    const uint32_t bi = id % f.bx, bj = (id / f.bx) % f.by, bk = id / f.bx / f.by;
    i = 8u * bi + l % 9u; j = 8u * bj + (l / 9u) % 9u; k = 8u * bk + l / 81u;
}

B2_DEV float df_lerp(float a, float b, float t) { return add(mul(a, sub(1.0f, t)), mul(b, t)); }

B2_DEV float df_lookup(const DfieldView& f, V3 p)
{
    const float inf = u2f(0x7f800000u);
    if (!(fabsf(p.x) < inf && fabsf(p.y) < inf && fabsf(p.z) < inf)) return inf;
    const float gx = mul(sub(p.x, f.ox), f.inv_h), gy = mul(sub(p.y, f.oy), f.inv_h), gz = mul(sub(p.z, f.oz), f.inv_h);
    if (!(gx >= 0.0f && gy >= 0.0f && gz >= 0.0f && gx <= (float)(f.dx - 1u) && gy <= (float)(f.dy - 1u) && gz <= (float)(f.dz - 1u))) return f.trunc;
    auto cell = [](float g, uint32_t d) { const uint32_t c = (uint32_t)floorf(g); return c < d - 2u ? c : d - 2u; };
    const uint32_t cx = cell(gx, f.dx), cy = cell(gy, f.dy), cz = cell(gz, f.dz);
    const float tx = sub(gx, (float)cx), ty = sub(gy, (float)cy), tz = sub(gz, (float)cz);
    const uint32_t slot = ldg(f.index + ((size_t)(cz >> 3) * f.by + (cy >> 3)) * f.bx + (cx >> 3));
    if (slot == B2_NOBRICK) return f.trunc;
    const float* b = f.bricks + (size_t)slot * B2_DF_NODES + ((cz & 7u) * 9u + (cy & 7u)) * 9u + (cx & 7u);
    const float c00 = df_lerp(ldg(b + 0), ldg(b + 1), tx), c10 = df_lerp(ldg(b + 9), ldg(b + 10), tx);
    const float c01 = df_lerp(ldg(b + 81), ldg(b + 82), tx), c11 = df_lerp(ldg(b + 90), ldg(b + 91), tx);
    return df_lerp(df_lerp(c00, c10, ty), df_lerp(c01, c11, ty), tz);
}

// Gaussian evaluation of one (particle, beam) pair from the field: the closest-point branch of pf_eval_one with e = field(q)
B2_DEV float pf_eval_field(const DfieldView& f, Tf Tsm, const PfBeam& b, float sigma_quad, double denom)
{
    const V3 orig_m = tf_apply(Tsm, mk3(b.ox, b.oy, b.oz));
    const V3 dir_m = q_rot(Tsm.R, mk3(b.dx, b.dy, b.dz));
    const float error = df_lookup(f, v_add(orig_m, v_scale(dir_m, b.range)));
    const float arg = dvd(dvd(-mul(error, error), sigma_quad), 2.0f);
    return (float)(exp((double)arg) / denom);
}

#ifdef __CUDACC__
// build: one thread per brick writes its allocation flag (0 / 1) into the index ...
__global__ void k_dfield_classify(BvhView bvh, DfieldView f, uint64_t n_bricks, float ta, float ta2, uint32_t* __restrict__ flags)
{
    for (uint64_t id = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; id < n_bricks; id += (uint64_t)gridDim.x * blockDim.x) {
        const uint32_t bi = (uint32_t)(id % f.bx), bj = (uint32_t)(id / f.bx % f.by), bk = (uint32_t)(id / f.bx / f.by);
        flags[id] = df_brick_alloc(bvh, f, bi, bj, bk, ta, ta2) ? 1u : 0u;
    }
}
// ... an exclusive scan gives the slots; the index becomes slot / B2_NOBRICK in place, and the slot -> brick list is written
__global__ void k_dfield_index(uint64_t n_bricks, const uint32_t* __restrict__ offs, uint32_t* __restrict__ index, uint32_t* __restrict__ list)
{
    for (uint64_t id = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; id < n_bricks; id += (uint64_t)gridDim.x * blockDim.x) {
        const bool a = index[id] != 0u;
        index[id] = a ? offs[id] : B2_NOBRICK;
        if (a && list) list[offs[id]] = (uint32_t)id;
    }
}
// one thread per node of each allocated brick
__global__ void k_dfield_fill(BvhView bvh, DfieldView f, const uint32_t* __restrict__ list, uint64_t n_nodes, float trunc2, float* __restrict__ bricks)
{
    for (uint64_t t = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; t < n_nodes; t += (uint64_t)gridDim.x * blockDim.x) {
        uint32_t i, j, k;
        df_brick_node(f, list[t / B2_DF_NODES], (uint32_t)(t % B2_DF_NODES), i, j, k);
        bricks[t] = df_node_value(bvh, f, i, j, k, trunc2);
    }
}
__global__ void k_dfield_query(DfieldView f, const float* __restrict__ pts, uint32_t n, float* __restrict__ out)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    out[i] = df_lookup(f, mk3(pts[3 * (size_t)i], pts[3 * (size_t)i + 1], pts[3 * (size_t)i + 2]));
}
// The sensor update from the field: k_pf_update's contract (block of ppb particles x all beams, evaluations in shared memory, merge in beam
// order, attrs read-modified-written once) with e = field(q).  Lanes = consecutive beams of one particle: the beams are sorted by direction
// (pf_prepare_beams), so a warp's lookups land in neighbouring cells of the field.
__global__ void __launch_bounds__(B2_PF_BLOCK) k_pf_update_field(DfieldView f, const b2_transform* __restrict__ poses, b2_particle_attr* __restrict__ attrs,
                                                              uint32_t n_particles, b2_transform Tsb_val, const PfBeam* __restrict__ beams, uint32_t n_beams,
                                                              b2_pf_params prm, uint32_t ppb)
{
    extern __shared__ float s_eval[];            // [ppb][n_beams]
    const uint32_t p0 = blockIdx.x * ppb;
    const uint32_t np = min(ppb, n_particles - p0);
    float sigma_quad; double denom; pf_constants(prm, sigma_quad, denom);
    const Tf Tsb = tf_from_pod(Tsb_val);
    const uint32_t total = np * n_beams;
    for (uint32_t w = threadIdx.x; w < total; w += blockDim.x) {
        const uint32_t pl = w / n_beams, bi = w % n_beams;
        const Tf Tsm = tf_mul(tf_load(poses + p0 + pl), Tsb);
        const PfBeam b = beams[bi];
        s_eval[pl * n_beams + b.slot] = pf_eval_field(f, Tsm, b, sigma_quad, denom);
    }
    __syncthreads();
    if (threadIdx.x < np) {
        b2_particle_attr* ap = attrs + p0 + threadIdx.x;
        b2_gaussian1d lk = ap->likelihood;
        pf_merge(lk, s_eval + threadIdx.x * n_beams, n_beams);
        ap->likelihood = lk;
    }
}
#endif

#ifdef __CUDACC__
// sort key of a particle for MAP 1: 16 heading bins (yaw), then the Morton code of its (x, y) cell on a 1024 x 1024 lattice over the map
__global__ void k_pf_sort_keys(const b2_transform* __restrict__ poses, uint32_t n, float bx, float by, uint32_t* __restrict__ keys, uint32_t* __restrict__ idx)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const Tf T = tf_load(poses + i);
    const float yaw = atan2f(2.0f * (T.R.w * T.R.z + T.R.x * T.R.y), 1.0f - 2.0f * (T.R.y * T.R.y + T.R.z * T.R.z));
    const uint32_t yb = min(15u, (uint32_t)((yaw + 3.14159265f) * (16.0f / 6.2831853f)));
    auto cell = [](float v, float b) { const float u = (v / (b + 1e-6f)) * 0.5f + 0.5f; return (uint32_t)min(1023.0f, max(0.0f, u * 1023.0f)); };
    auto spread = [](uint32_t x) { x &= 0x3ffu; x = (x | (x << 8)) & 0x00ff00ffu; x = (x | (x << 4)) & 0x0f0f0f0fu; x = (x | (x << 2)) & 0x33333333u; x = (x | (x << 1)) & 0x55555555u; return x; };
    keys[i] = (yb << 20) | spread(cell(T.t.x, bx)) | (spread(cell(T.t.y, by)) << 1);
    idx[i] = i;
}
#endif

// ---------------------------------------------------------------------------------------------------------------------
// rest of the PF cycle (SURVEY 8f2)
// ---------------------------------------------------------------------------------------------------------------------
// particle_move_and_forget_kernel (rmcl_ros/src/rmcl/particle_motion.cu:11-34): HBM stream, 2 x (32 + 36) B per particle
// With COLLIDE the wall check of the CPU updater (TFMotionUpdaterCPU.cpp:17-50,205-216) rides along: one ray from the old to the new
// position, tfar = their distance; a hit pins the likelihood to {0, 0, MAX_N_MEAS}.
B2_DEV void pf_motion_one(const BvhView* bvh, b2_transform* pose_io, b2_particle_attr* attr_io, Tf T, double forget_rate)
{
    const Tf pose_old = tf_load(pose_io);
    const Tf pose_new = tf_mul(pose_old, T);
    b2_gaussian1d lk = attr_io->likelihood;
    lk.n_meas = (uint32_t)((double)lk.n_meas - forget_rate * (double)lk.n_meas);
    if (bvh) {
        const V3 vec = v_sub(pose_new.t, pose_old.t);
        const float length = v_l2norm(vec);
        if (!(length < 0.00001f)) {
            const RaySetup r = ray_setup(pose_old.t, mk3(dvd(vec.x, length), dvd(vec.y, length), dvd(vec.z, length)), *bvh);
            HitRec h = trace_init(length);
            uint32_t nn = 0, nt = 0;
            trace_closest<false>(*bvh, r, h, nn, nt);
            if (h.face != B2_NOFACE) { lk.mean = 0.0f; lk.sigma = 0.0f; lk.n_meas = 10000u; }
        }
    }
    tf_store(pose_io, pose_new);
    attr_io->likelihood = lk;
}
#ifdef __CUDACC__
template <bool COLLIDE>
__global__ void __launch_bounds__(128) k_pf_motion(BvhView bvh, b2_transform* __restrict__ poses, b2_particle_attr* __restrict__ attrs, uint32_t n, b2_transform T_val, double forget_rate)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    pf_motion_one(COLLIDE ? &bvh : nullptr, poses + i, attrs + i, tf_from_pod(T_val), forget_rate);
}
#endif

// The surface constraint of the motion stage (docs/RMCL.md:72 lists it as missing; no reference implementation, SURVEY appendix F).  One
// ray straight down (map -z) from probe_above over the particle, closest hit in (0, tfar]; the hit is ground iff the unit normal, turned
// to face the ray origin, has n.z >= cos_max.  On ground the particle is put base_height over it (along +z, or along n with align, where
// the smallest rotation also takes the body z-axis onto n); else it keeps its pose and gets the wall check's mark {0, 0, MAX_N_MEAS}.
// The stamp and the rest of the attributes are left as they are.  cos_max = (float)cos((double)max_slope), tfar = probe_above + probe_below.
// pf_surface_pose applies the rule to a pose in registers and reports the ground test; pf_surface_one applies it to a particle in memory.
B2_DEV bool pf_surface_pose(const BvhView& bvh, Tf& T, const b2_surface_config& cfg, float cos_max, float tfar)
{
    const float oz = add(T.t.z, cfg.probe_above);
    HitRec h = trace_init(tfar);
    // A non-finite pose is off surface.  A non-finite origin hits no triangle anyway, but its box tests pass everywhere (fmaxf / fminf drop
    // NaN): do not walk the whole tree for it.
    const float inf = u2f(0x7f800000u);
    if (fabsf(T.t.x) < inf && fabsf(T.t.y) < inf && fabsf(oz) < inf &&
        fabsf(T.R.x) < inf && fabsf(T.R.y) < inf && fabsf(T.R.z) < inf && fabsf(T.R.w) < inf) {
        const RaySetup r = ray_setup(mk3(T.t.x, T.t.y, oz), mk3(0.0f, 0.0f, -1.0f), bvh);
        uint32_t nn = 0, nt = 0;
        trace_closest<false>(bvh, r, h, nn, nt);
    }
    V3 n = mk3(0.0f, 0.0f, 0.0f);
    if (h.face != B2_NOFACE) {
        n = v_normalize(tri_ng(bvh, h.tri));
        if (n.z < 0.0f) n = v_neg(n);
    }
    if (!(h.face != B2_NOFACE && n.z >= cos_max)) return false;                       // no hit, too steep, or a NaN normal
    const V3 g = mk3(T.t.x, T.t.y, sub(oz, h.t));
    Tf out;
    if (cfg.align) {
        const V3 a = q_rot(T.R, mk3(0.0f, 0.0f, 1.0f));
        const float w = add(1.0f, v_dot(a, n));
        Q4 q;
        if (w < 1e-6f) {                                                               // body z-axis opposite to n: half turn about body x
            const V3 ex = q_rot(T.R, mk3(1.0f, 0.0f, 0.0f));
            q.x = ex.x; q.y = ex.y; q.z = ex.z; q.w = 0.0f;
        } else {                                                                       // a x n, rm::Vector3::cross
            q.x = sub(mul(a.y, n.z), mul(a.z, n.y)); q.y = sub(mul(a.z, n.x), mul(a.x, n.z)); q.z = sub(mul(a.x, n.y), mul(a.y, n.x)); q.w = w;
        }
        out.R = q_normalize(q_mul(q_normalize(q), T.R));
        out.t = v_add(g, v_scale(n, cfg.base_height));
    } else {
        out.R = T.R;
        out.t = mk3(g.x, g.y, add(g.z, cfg.base_height));
    }
    T = out;
    return true;
}
// true iff the particle stood on ground and was moved; else it is marked
B2_DEV bool pf_surface_one(const BvhView& bvh, b2_transform* pose_io, b2_particle_attr* attr_io, const b2_surface_config& cfg, float cos_max, float tfar)
{
    Tf T = tf_load(pose_io);
    if (!pf_surface_pose(bvh, T, cfg, cos_max, tfar)) {
        b2_gaussian1d lk = attr_io->likelihood;
        lk.mean = 0.0f; lk.sigma = 0.0f; lk.n_meas = 10000u;
        attr_io->likelihood = lk;
        return false;
    }
    // R and t only: the stamp stays
    pose_io->R.x = T.R.x; pose_io->R.y = T.R.y; pose_io->R.z = T.R.z; pose_io->R.w = T.R.w;
    pose_io->t.x = T.t.x; pose_io->t.y = T.t.y; pose_io->t.z = T.t.z;
    return true;
}
#ifdef __CUDACC__
__global__ void __launch_bounds__(128) k_pf_surface(BvhView bvh, b2_transform* __restrict__ poses, b2_particle_attr* __restrict__ attrs, uint32_t n,
                                                    b2_surface_config cfg, float cos_max, float tfar)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    pf_surface_one(bvh, poses + i, attrs + i, cfg, cos_max, tfar);
}
#endif

// ---------------------------------------------------------------------------------------------------------------------
// Gladiator resampling (rmcl_ros/src/rmcl/resampling.cu:108-199).  Draws: Philox4x32-10 (Salmon et al., SC'11), counter =
// (global particle index, 0, step, block), key = seed -- one raw u32 (opponent) + three Box-Muller pairs per particle; a function
// of the GLOBAL index only, so the result does not depend on how particles are sharded over GPUs.  See DESIGN.md for why the
// reference's cuRAND XORWOW stream is not reproduced.
// ---------------------------------------------------------------------------------------------------------------------
B2_DEV void philox4x32_10(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3, uint32_t k0, uint32_t k1, uint32_t out[4])
{
    #pragma unroll
    for (int r = 0; r < 10; r++) {
        const uint64_t p0 = (uint64_t)0xD2511F53u * c0, p1 = (uint64_t)0xCD9E8D57u * c2;
        const uint32_t n0 = (uint32_t)(p1 >> 32) ^ c1 ^ k0, n1 = (uint32_t)p1, n2 = (uint32_t)(p0 >> 32) ^ c3 ^ k1, n3 = (uint32_t)p0;
        c0 = n0; c1 = n1; c2 = n2; c3 = n3;
        k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
    }
    out[0] = c0; out[1] = c1; out[2] = c2; out[3] = c3;
}
B2_DEV float u01_open(uint32_t r) { return mul(add((float)(r >> 8), 0.5f), 5.9604644775390625e-08f); }
// three Box-Muller pairs on the words (r[0], r[1]), (r[2], r[3]), (r[4], r[5])
B2_DEV void box_muller3(const uint32_t* r, float N[6])
{
    #pragma unroll
    for (int p = 0; p < 3; p++) {
        const float u1 = u01_open(r[2 * p]), u2 = u01_open(r[2 * p + 1]);
        const float rad = sqrtf(mul(-2.0f, logf(u1))), ang = mul(6.283185307179586f, u2);
        N[2 * p] = mul(rad, cosf(ang)); N[2 * p + 1] = mul(rad, sinf(ang));
    }
}
B2_DEV void gladiator_draws(uint64_t seed, uint32_t step, uint32_t gidx, uint32_t& raw, float N[6])
{
    uint32_t r[8];
    philox4x32_10(gidx, 0u, step, 0u, (uint32_t)seed, (uint32_t)(seed >> 32), r);
    philox4x32_10(gidx, 0u, step, 1u, (uint32_t)seed, (uint32_t)(seed >> 32), r + 4);
    raw = r[0];
    box_muller3(r + 1, N);
}
// rm::EulerAngles <-> Quaternion [RM-recalled: standard ZYX conversions], op order as in oracle/oracle.c
B2_DEV void quat_to_euler(Q4 q, float& roll, float& pitch, float& yaw)
{
    roll = atan2f(mul(2.0f, add(mul(q.w, q.x), mul(q.y, q.z))), sub(1.0f, mul(2.0f, add(mul(q.x, q.x), mul(q.y, q.y)))));
    const float sinp = mul(2.0f, sub(mul(q.w, q.y), mul(q.z, q.x)));
    pitch = fabsf(sinp) >= 1.0f ? copysignf(1.5707963267948966f, sinp) : asinf(sinp);
    yaw = atan2f(mul(2.0f, add(mul(q.w, q.z), mul(q.x, q.y))), sub(1.0f, mul(2.0f, add(mul(q.y, q.y), mul(q.z, q.z)))));
}
B2_DEV Q4 euler_to_quat(float roll, float pitch, float yaw)
{
    const float cr = cosf(mul(roll, 0.5f)), sr = sinf(mul(roll, 0.5f)), cp = cosf(mul(pitch, 0.5f)), sp = sinf(mul(pitch, 0.5f)), cy = cosf(mul(yaw, 0.5f)), sy = sinf(mul(yaw, 0.5f));
    Q4 q;
    q.w = add(mul(mul(cr, cp), cy), mul(mul(sr, sp), sy));
    q.x = sub(mul(mul(sr, cp), cy), mul(mul(cr, sp), sy));
    q.y = add(mul(mul(cr, sp), cy), mul(mul(sr, cp), sy));
    q.z = sub(mul(mul(cr, cp), sy), mul(mul(sr, sp), cy));
    return q;
}
// the perturbed copy of a pose, shared by both resamplers (resampling.cu:166-175, ResidualResamplerCPU.cpp:150-162): t += N[0..2] * s[0..2],
// the Euler angles of R += N[3..5] * s[3..5]; diff = ~pose * pose_new.  The forget rule applied to diff is each resampler's own.
B2_DEV Tf pf_perturb(const Tf& pose, const float N[6], const float s[6], Tf& diff)
{
    Tf pnew = pose;
    pnew.t = mk3(add(pose.t.x, mul(N[0], s[0])), add(pose.t.y, mul(N[1], s[1])), add(pose.t.z, mul(N[2], s[2])));
    float roll, pitch, yaw; quat_to_euler(pose.R, roll, pitch, yaw);
    pnew.R = euler_to_quat(add(roll, mul(N[3], s[3])), add(pitch, mul(N[4], s[4])), add(yaw, mul(N[5], s[5])));
    diff = tf_mul(tf_inv(pose), pnew);
    return pnew;
}
// Quaternion::l2norm, the "rotation distance" of both resamplers: the 4-norm of diff.R, ~1 for any rotation (SURVEY D32)
B2_DEV float quat_l2norm(Q4 q) { return sqrtf(add(add(add(mul(q.x, q.x), mul(q.y, q.y)), mul(q.z, q.z)), mul(q.w, q.w))); }
// the opponent won (resampling.cu:150-192): the champion's slot receives a perturbed copy of the opponent whose n_meas is reduced by the forget rate
B2_DEV void gladiator_take(b2_transform pn, b2_particle_attr an, const float N[6], const b2_gladiator_config& cfg, b2_transform* out_p, b2_particle_attr* out_a)
{
    const float s[6] = {cfg.min_noise_tx, cfg.min_noise_ty, cfg.min_noise_tz, cfg.min_noise_roll, cfg.min_noise_pitch, cfg.min_noise_yaw};
    Tf diff;
    const Tf pnew = pf_perturb(tf_from_pod(pn), N, s, diff);                               // :166-175
    const float trans_dist = v_l2norm(diff.t);                                             // :178
    const float rot_dist = quat_l2norm(diff.R);                                            // :179
    const float frs = (float)(1.0 - pow(1.0 - (double)cfg.likelihood_forget_per_meter, (double)trans_dist));    // :182
    const float frr = (float)(1.0 - pow(1.0 - (double)cfg.likelihood_forget_per_radian, (double)rot_dist));     // :183
    const float forget = frs > frr ? frs : frr;
    const float remember = (float)(1.0 - (double)forget);                                  // :185
    an.likelihood.n_meas = (uint32_t)mul((float)an.likelihood.n_meas, remember);           // :187
    pn.R.x = pnew.R.x; pn.R.y = pnew.R.y; pn.R.z = pnew.R.z; pn.R.w = pnew.R.w; pn.t.x = pnew.t.x; pn.t.y = pnew.t.y; pn.t.z = pnew.t.z;   // stamp: the enemy's
    *out_p = pn; *out_a = an;
}
// one champion: poses/attrs are the n_all particles, champion = global index, outputs are written at out_p / out_a
B2_DEV void gladiator_one(const b2_transform* poses, const b2_particle_attr* attrs, uint32_t n_all, uint32_t champion, uint32_t raw, const float N[6],
                          const b2_gladiator_config& cfg, b2_transform* out_p, b2_particle_attr* out_a)
{
    const uint32_t enemy = raw % n_all;                                                    // :137
    const float Lc = attrs[champion].likelihood.mean, Le = attrs[enemy].likelihood.mean;
    if (!(Le > Lc)) { *out_p = poses[champion]; *out_a = attrs[champion]; return; }       // :150, :193-196
    gladiator_take(poses[enemy], attrs[enemy], N, cfg, out_p, out_a);
}

#ifdef __CUDACC__
// HBM stream: 68 B in (+68 B gathered from the opponent when it wins) and 68 B out per particle
__global__ void __launch_bounds__(256) k_pf_gladiator(const b2_transform* __restrict__ poses, const b2_particle_attr* __restrict__ attrs, uint32_t n_all, uint32_t first,
                                                      uint32_t n_local, b2_transform* __restrict__ poses_new, b2_particle_attr* __restrict__ attrs_new,
                                                      b2_gladiator_config cfg, uint64_t seed, uint32_t step, const uint32_t* __restrict__ raw_in, const float* __restrict__ normals_in)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_local) return;
    uint32_t raw; float N[6];
    if (raw_in) { raw = raw_in[i]; for (int k = 0; k < 6; k++) N[k] = normals_in[6 * (size_t)i + k]; }
    else gladiator_draws(seed, step, first + i, raw, N);
    gladiator_one(poses, attrs, n_all, first + i, raw, N, cfg, poses_new + i, attrs_new + i);
}
__global__ void k_pf_gladiator_randoms(uint64_t seed, uint32_t step, uint32_t first, uint32_t n, uint32_t* __restrict__ raw_out, float* __restrict__ normals_out)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint32_t raw; float N[6];
    gladiator_draws(seed, step, first + i, raw, N);
    raw_out[i] = raw;
    for (int k = 0; k < 6; k++) normals_out[6 * (size_t)i + k] = N[k];
}
#endif

// ---------------------------------------------------------------------------------------------------------------------
// Particle set initialisation: RmclNode::initSamplesUniform (rmcl_ros/src/nodes/rmcl_localization.cpp:277-342) and
// RmclNode::initSamples(PoseWithCovarianceStamped) (:165-275).  Draws: Philox4x32-10 with counter (global particle index, domain tag,
// 0, block) and key = seed.  The tags are non-zero and Gladiator's second counter word is always 0, so no two streams share a counter.
// The beam sampling of the sensor update (b2_pf_sample_cloud, below) draws with tag 3.
// ---------------------------------------------------------------------------------------------------------------------
#define B2_PF_INIT_TAG_UNIFORM 1u
#define B2_PF_INIT_TAG_GAUSSIAN 2u
#define B2_PF_BEAM_TAG 3u
struct PfInitBox { float lo[6], hi[6]; };                  // x, y, z, roll, pitch, yaw; lo <= hi, finite, hi - lo finite (checked on the host)
struct PfInitGauss { float L[36]; b2_transform Tlm; };     // Cholesky factor of the covariance (row-major, lower), message pose
B2_DEV float u01_closed_open(uint32_t r) { return mul((float)(r >> 8), 5.9604644775390625e-08f); }   // [0, 1), exact
// the attributes both initialisers give a particle (:252-255, :322-325): Gaussian1D::Identity() with mean 1.0, state_sigma 0
B2_DEV void pf_init_attr(b2_particle_attr* a)
{
    a->likelihood.mean = 1.0f; a->likelihood.sigma = 0.0f; a->likelihood.n_meas = 0u;
    #pragma unroll
    for (int k = 0; k < 6; k++) a->state_sigma[k] = 0.0f;
}
// uniform_real_distribution<float>(lo, hi) per dimension (:287-292, :318-319): lo + (hi - lo) u, u in [0, 1), never above hi; words r[0..5]
// give x, y, z, roll, pitch, yaw, the angles Euler ZYX.  Shared by the initialiser and the recovery's candidates.
B2_DEV Tf pf_box_pose(const PfInitBox& box, const uint32_t r[6])
{
    float v[6];
    #pragma unroll
    for (int k = 0; k < 6; k++) v[k] = fminf(add(box.lo[k], mul(sub(box.hi[k], box.lo[k]), u01_closed_open(r[k]))), box.hi[k]);
    Tf T; T.t = mk3(v[0], v[1], v[2]); T.R = euler_to_quat(v[3], v[4], v[5]);
    return T;
}
B2_DEV void pf_init_uniform_one(uint64_t seed, uint32_t gidx, const PfInitBox& box, b2_transform* out_p, b2_particle_attr* out_a)
{
    uint32_t r[8];
    philox4x32_10(gidx, B2_PF_INIT_TAG_UNIFORM, 0u, 0u, (uint32_t)seed, (uint32_t)(seed >> 32), r);
    philox4x32_10(gidx, B2_PF_INIT_TAG_UNIFORM, 0u, 1u, (uint32_t)seed, (uint32_t)(seed >> 32), r + 4);
    tf_store(out_p, pf_box_pose(box, r));
    pf_init_attr(out_a);
}
// x = L N(0, I6) (rm::Matrix_ product, sums over k = 0..5 in order), pose = Tlm * Transform{EulerAngles{x3, x4, x5}, {x0, x1, x2}} (:231-251)
B2_DEV void pf_init_gaussian_one(uint64_t seed, uint32_t gidx, const PfInitGauss& g, b2_transform* out_p, b2_particle_attr* out_a)
{
    uint32_t r[8];
    philox4x32_10(gidx, B2_PF_INIT_TAG_GAUSSIAN, 0u, 0u, (uint32_t)seed, (uint32_t)(seed >> 32), r);
    philox4x32_10(gidx, B2_PF_INIT_TAG_GAUSSIAN, 0u, 1u, (uint32_t)seed, (uint32_t)(seed >> 32), r + 4);
    float N[6], x[6];
    box_muller3(r, N);
    #pragma unroll
    for (int i = 0; i < 6; i++) {
        float a = 0.0f;
        #pragma unroll
        for (int k = 0; k < 6; k++) a = add(a, mul(g.L[6 * i + k], N[k]));
        x[i] = a;
    }
    Tf Pl; Pl.t = mk3(x[0], x[1], x[2]); Pl.R = euler_to_quat(x[3], x[4], x[5]);
    tf_store(out_p, tf_mul(tf_from_pod(g.Tlm), Pl));
    pf_init_attr(out_a);
}
#ifdef __CUDACC__
// write-only: 32 B pose + 36 B attrs per particle, nothing read from HBM
__global__ void __launch_bounds__(256) k_pf_init_uniform(b2_transform* __restrict__ poses, b2_particle_attr* __restrict__ attrs, uint32_t first, uint32_t n, PfInitBox box, uint64_t seed)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    pf_init_uniform_one(seed, first + i, box, poses + i, attrs + i);
}
__global__ void __launch_bounds__(256) k_pf_init_gaussian(b2_transform* __restrict__ poses, b2_particle_attr* __restrict__ attrs, uint32_t first, uint32_t n, PfInitGauss g, uint64_t seed)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    pf_init_gaussian_one(seed, first + i, g, poses + i, attrs + i);
}
#endif

// ---------------------------------------------------------------------------------------------------------------------
// Recovery from a kidnapping: Augmented MCL (Thrun, Burgard, Fox, Probabilistic Robotics, 8.3.5; AMCL's recovery_alpha_slow / _fast; no
// reference implementation, SURVEY appendix J).  The handle's record {w_avg, w_slow, w_fast, p_inject} (b2_recovery_state) follows the mean
// likelihood of the set (pf_recovery_filter, after each sensor update); after resampling each particle is replaced with probability
// p_inject by a random pose of a box, on the map's ground when a surface config is given (pf_recovery_one).  Draws: Philox4x32-10 with
// counter (global particle index, B2_PF_RECOVERY_TAG, step, block) and key = seed: block 0 word 0 decides, blocks 1 + 2t and 2 + 2t give try
// t's six words.  They depend on (seed, step, index, try) only, so slices of a sharded set concatenate to the whole result.
// ---------------------------------------------------------------------------------------------------------------------
#define B2_PF_RECOVERY_TAG 7u
#define B2_RECOVERY_MAX_TRIES 64u
// AMCL's recurrence on the record, all in FP64: w_avg = S / n; a non-finite or negative w_avg leaves the record as it is; each average w of
// rate alpha becomes w_avg when w == 0, else w + alpha (w_avg - w); p_inject = w_slow > 0 ? max(0, 1 - w_fast / w_slow) : 0
B2_DEV void pf_recovery_filter(double S, uint32_t n, double alpha_slow, double alpha_fast, b2_recovery_state* st)
{
    const double w_avg = S / (double)n;
    st->w_avg = w_avg;
    if (!(w_avg >= 0.0 && w_avg <= 1.7976931348623157e308)) return;
    st->w_slow = st->w_slow == 0.0 ? w_avg : st->w_slow + alpha_slow * (w_avg - st->w_slow);
    st->w_fast = st->w_fast == 0.0 ? w_avg : st->w_fast + alpha_fast * (w_avg - st->w_fast);
    const double p = st->w_slow > 0.0 ? 1.0 - st->w_fast / st->w_slow : 0.0;
    st->p_inject = p > 0.0 ? p : 0.0;
}
// what happened to one particle
#define B2_RECOVERY_KEPT 0u          // not chosen
#define B2_RECOVERY_REPLACED 1u
#define B2_RECOVERY_FAILED 2u        // chosen, but no candidate of max_tries was taken: the particle is unchanged
// particle g of the set with the record's p: chosen iff (double)word * 2^-32 < p; try t's candidate is pf_box_pose of its six words, taken
// as it is without a surface (bvh == nullptr), else iff pf_surface_pose finds ground under it, as it moved it.  A taken candidate is written
// with stamp 0 (tf_store, as the initialiser writes it) and the attributes {0, 0, 0}, state_sigma 0: no weight until a sensor update
// evaluates it, whose Gaussian merge then takes the fresh likelihood alone (n_meas 0).
B2_DEV uint32_t pf_recovery_one(const BvhView* bvh, b2_transform* pose_io, b2_particle_attr* attr_io, uint32_t g, double p, const PfInitBox& box,
                                const b2_surface_config& cfg, float cos_max, float tfar, uint32_t max_tries, uint64_t seed, uint32_t step)
{
    const uint32_t k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32);
    uint32_t r[8];
    philox4x32_10(g, B2_PF_RECOVERY_TAG, step, 0u, k0, k1, r);
    if (!((double)r[0] * 2.3283064365386963e-10 < p)) return B2_RECOVERY_KEPT;
    for (uint32_t t = 0; t < max_tries; t++) {
        philox4x32_10(g, B2_PF_RECOVERY_TAG, step, 1u + 2u * t, k0, k1, r);
        philox4x32_10(g, B2_PF_RECOVERY_TAG, step, 2u + 2u * t, k0, k1, r + 4);
        Tf T = pf_box_pose(box, r);
        if (bvh && !pf_surface_pose(*bvh, T, cfg, cos_max, tfar)) continue;
        tf_store(pose_io, T);
        b2_particle_attr a;
        a.likelihood.mean = 0.0f; a.likelihood.sigma = 0.0f; a.likelihood.n_meas = 0u;
        #pragma unroll
        for (int k = 0; k < 6; k++) a.state_sigma[k] = 0.0f;
        *attr_io = a;
        return B2_RECOVERY_REPLACED;
    }
    return B2_RECOVERY_FAILED;
}
#ifdef __CUDACC__
// one thread: the record's update from the S that k_pf_residual_stats left in device memory (bit-equal to the estimate's L_sum)
__global__ void k_pf_recovery_filter(const double* __restrict__ S, uint32_t n, double alpha_slow, double alpha_fast, b2_recovery_state* __restrict__ st)
{
    pf_recovery_filter(*S, n, alpha_slow, alpha_fast, st);
}
// one thread per particle first + i of the slice; 128 threads per block as k_pf_surface, since replaced particles trace rays.  res (may be
// null) receives the p used and the counts: every lane of a warp votes (lanes past the slice with "kept"), lane 0 adds the warp's counts.
template <bool SURFACE>
__global__ void __launch_bounds__(128) k_pf_recovery_inject(BvhView bvh, b2_transform* __restrict__ poses, b2_particle_attr* __restrict__ attrs, uint32_t first,
                                                            uint32_t n, PfInitBox box, b2_surface_config cfg, float cos_max, float tfar, uint32_t max_tries,
                                                            uint64_t seed, uint32_t step, const b2_recovery_state* __restrict__ st, b2_recovery_result* __restrict__ res)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t what = B2_RECOVERY_KEPT;
    if (i < n) {
        const double p = st->p_inject;
        if (res && i == 0) res->p_inject = p;
        what = pf_recovery_one(SURFACE ? &bvh : nullptr, poses + i, attrs + i, first + i, p, box, cfg, cos_max, tfar, max_tries, seed, step);
    }
    if (res) {                                                          // uniform over the grid; blocks are whole warps
        const unsigned rep = __ballot_sync(0xffffffffu, what == B2_RECOVERY_REPLACED), fl = __ballot_sync(0xffffffffu, what == B2_RECOVERY_FAILED);
        if ((threadIdx.x & 31u) == 0u) {
            if (rep) atomicAdd((unsigned long long*)&res->n_replaced, (unsigned long long)__popc(rep));
            if (fl) atomicAdd((unsigned long long*)&res->n_failed, (unsigned long long)__popc(fl));
        }
    }
}
// one thread, after k_pf_recovery_inject has read p: AMCL resets both averages after an injection
__global__ void k_pf_recovery_clear(b2_recovery_state* __restrict__ st)
{
    if (st->p_inject > 0.0) { st->w_slow = 0.0; st->w_fast = 0.0; st->p_inject = 0.0; }
}
#endif

// ---------------------------------------------------------------------------------------------------------------------
// The sensor update's beam sampling: PCDSensorUpdaterOptix::update (rmcl_ros/src/rmcl/PCDSensorUpdaterOptix.cpp:227-311).  Sample k makes
// up to B2_PF_BEAM_TRIES tries; try t reads point raw % n_points, raw = word t % 4 of Philox4x32-10 with counter (k, B2_PF_BEAM_TAG, step,
// t / 4) and key = seed.  The draws depend on (seed, step, k) only, so every rank of a sharded particle set samples the same beams.  The
// give-up rule over the samples (B2_PF_BEAM_MAX_INVALIDS) runs on the host (b2_pf_sample_cloud).
// ---------------------------------------------------------------------------------------------------------------------
#define B2_PF_BEAM_TRIES 100u                  // max_tries (:267)
#define B2_PF_BEAM_MAX_INVALIDS 10u            // max_invalids (:264)
struct CloudBeams {
    uint32_t width, n_points;               // points of the cloud (width * height, 1 .. 2^32 - 1)
    uint64_t row_step; uint32_t point_step;
    uint32_t off[3];                        // byte offsets of x, y, z inside a point
    uint32_t f64;                           // 1: FLOAT64 fields (narrowed to float), 0: FLOAT32
    uint64_t seed; uint32_t step;
};
struct PfBeamSample { b2_range_meas m; uint32_t valid; };         // one sample as the kernel hands it to the host (68 B)

// word w (0..3) of a Philox block, without indexing the array at run time (it stays in registers)
B2_DEV uint32_t philox_word(const uint32_t r[4], uint32_t w) { return w == 0u ? r[0] : w == 1u ? r[1] : w == 2u ? r[2] : r[3]; }
// NaN components are stored as 0x7fffffff whatever produced them, so that the host and the device write the same bytes
B2_DEV float canon_nan(float v) { return v == v ? v : u2f(0x7fffffffu); }

// sample k (:265-306): true and *m filled from the first try whose x, y and z are not NaN (an infinite coordinate passes, :278); false when
// every try failed.  orig = 0, range = |p|, dir = p / range (:291-293) -- a finite (0,0,0) gives range 0 and NaN directions -- cov = 0.1 I
// (:296-301).  Point i is read at row * row_step + col * point_step through the fields (the reference reads float32 at i * point_step, D26).
B2_DEV bool pf_sample_beam(const uint8_t* cloud, const CloudBeams& c, uint32_t k, b2_range_meas* m)
{
    const bool f64 = c.f64 != 0;
    uint32_t r[4] = {0u, 0u, 0u, 0u};
    for (uint32_t t = 0; t < B2_PF_BEAM_TRIES; t++) {
        if ((t & 3u) == 0u) philox4x32_10(k, B2_PF_BEAM_TAG, c.step, t >> 2, (uint32_t)c.seed, (uint32_t)(c.seed >> 32), r);
        const uint32_t i = philox_word(r, t & 3u) % c.n_points;
        const uint32_t row = i / c.width, col = i - row * c.width;
        const uint8_t* p = cloud + (uint64_t)row * c.row_step + (uint64_t)col * c.point_step;
        const float x = cloud_coord(p + c.off[0], f64), y = cloud_coord(p + c.off[1], f64), z = cloud_coord(p + c.off[2], f64);
        if (!(x == x && y == y && z == z)) continue;
        const float range = v_l2norm(mk3(x, y, z));
        m->orig.x = 0.f; m->orig.y = 0.f; m->orig.z = 0.f;
        m->dir.x = canon_nan(dvd(x, range)); m->dir.y = canon_nan(dvd(y, range)); m->dir.z = canon_nan(dvd(z, range));
        m->range = range;
        #pragma unroll
        for (int e = 0; e < 9; e++) m->cov.m[e] = (e % 4 == 0) ? 0.1f : 0.f;
        return true;
    }
    return false;
}

#ifdef __CUDACC__
// one thread per sample; reads at most B2_PF_BEAM_TRIES points, writes 68 B
__global__ void __launch_bounds__(128) k_pf_sample_cloud(const uint8_t* __restrict__ cloud, CloudBeams c, uint32_t n_samples, PfBeamSample* __restrict__ out)
{
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n_samples) return;
    PfBeamSample s = {};
    s.valid = pf_sample_beam(cloud, c, k, &s.m) ? 1u : 0u;
    out[k] = s;
}
#endif

#ifdef __CUDACC__
// Gladiator resampling with the particles SHARDED over GPUs and no all-gather: every rank publishes its particles in a buffer its peers map over
// NVLink (CUDA IPC); a champion reads its opponent's 4-byte likelihood straight from the owner's HBM and fetches the 68-byte record only when
// the opponent wins -- the reference draws opponents from ALL particles (resampling.cu:137), so this is the one stage of the cycle whose data
// crosses GPUs.  Shards have equal size n_per_rank; global index = rank * n_per_rank + local index; draws are keyed by the global index, so
// the concatenation over ranks equals the single-GPU result bit for bit.  `traffic` counts the bytes actually read from remote ranks.
#define B2_MAX_PEERS 16
struct PfPeers { const b2_transform* poses[B2_MAX_PEERS]; const b2_particle_attr* attrs[B2_MAX_PEERS]; uint32_t world, rank, n_per_rank, pad; };
__global__ void __launch_bounds__(256) k_pf_gladiator_p2p(PfPeers peers, b2_transform* __restrict__ poses_new, b2_particle_attr* __restrict__ attrs_new, b2_gladiator_config cfg,
                                                          uint64_t seed, uint32_t step, unsigned long long* __restrict__ traffic)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    unsigned long long remote = 0ull;
    if (i < peers.n_per_rank) {
        const uint32_t n_all = peers.n_per_rank * peers.world, champion = peers.rank * peers.n_per_rank + i;
        uint32_t raw; float N[6];
        gladiator_draws(seed, step, champion, raw, N);
        const uint32_t enemy = raw % n_all, er = enemy / peers.n_per_rank, ei = enemy % peers.n_per_rank;      // resampling.cu:137
        const b2_particle_attr* ea = peers.attrs[er] + ei;
        const float Lc = peers.attrs[peers.rank][i].likelihood.mean;
        const float Le = __ldcv(&ea->likelihood.mean);                                                       // peer memory: never from a stale cache line
        if (er != peers.rank) remote += 4ull;
        if (!(Le > Lc)) { poses_new[i] = peers.poses[peers.rank][i]; attrs_new[i] = peers.attrs[peers.rank][i]; }
        else {
            const b2_transform* ep = peers.poses[er] + ei;
            b2_transform pn; b2_particle_attr an;
            const uint4 p0 = __ldcv(reinterpret_cast<const uint4*>(ep)), p1 = __ldcv(reinterpret_cast<const uint4*>(ep) + 1);
            memcpy(&pn, &p0, 16); memcpy(reinterpret_cast<char*>(&pn) + 16, &p1, 16);
            const uint32_t* aw = reinterpret_cast<const uint32_t*>(ea);
            uint32_t w[9];
            #pragma unroll
            for (int k = 0; k < 9; k++) w[k] = __ldcv(aw + k);
            memcpy(&an, w, 36);
            if (er != peers.rank) remote += 68ull;
            gladiator_take(pn, an, N, cfg, poses_new + i, attrs_new + i);
        }
    }
    remote = warp_sum_u64(remote);
    if (traffic && (threadIdx.x & 31u) == 0u && remote) atomicAdd(traffic, remote);
}
#endif

// ---------------------------------------------------------------------------------------------------------------------
// Pose estimate of the particle set: RmclNode::estimateStats (rmcl_ros/src/nodes/rmcl_localization.cpp:642-731) in two read passes.
// Pass 1 (k_pf_estimate_moments): likelihood sums, min / max, translation AABB, sum L t and sum L q q^T; its last block forms the weighted
// Markley mean Tbm (SURVEY decision E1).  Pass 2 (k_pf_estimate_cov): the 6x6 covariance of (~Tbm * pose) about Tbm (decision E2).  Weights
// are w_i = L_i / L_sum; the sums are taken over L_i and divided by L_sum once, in FP64.
// ---------------------------------------------------------------------------------------------------------------------
#define B2_JACOBI_SWEEPS 16
B2_DEV double f64_from_bits(unsigned long long u)
{
#if B2_ON_DEVICE
    return __longlong_as_double((long long)u);
#else
    double d; memcpy(&d, &u, 8); return d;
#endif
}
B2_DEV double f64_nan() { return f64_from_bits(0x7ff8000000000000ull); }
B2_DEV double f64_inf() { return f64_from_bits(0x7ff0000000000000ull); }
// eigenvector of the largest eigenvalue of a symmetric 4x4 matrix (row-major, FP64): cyclic Jacobi, at most B2_JACOBI_SWEEPS sweeps; a
// non-finite entry gives a NaN vector.  Sign: w >= 0, and when w == 0 the first non-zero component is positive.
B2_DEV void sym4_top_eigvec(const double* Ain, double v[4], double* lambda)
{
    // fully unrolled so that A and V stay in registers on the device
    double A[4][4], V[4][4];
    bool finite = true;
    #pragma unroll
    for (int i = 0; i < 4; i++)
        #pragma unroll
        for (int j = 0; j < 4; j++) { A[i][j] = Ain[4 * i + j]; V[i][j] = i == j ? 1.0 : 0.0; finite = finite && A[i][j] - A[i][j] == 0.0; }
    if (!finite) {
        v[0] = v[1] = v[2] = v[3] = *lambda = f64_nan();
        return;
    }
    for (int sweep = 0; sweep < B2_JACOBI_SWEEPS; sweep++) {
        double off = 0.0;
        #pragma unroll
        for (int p = 0; p < 3; p++)
            #pragma unroll
            for (int q = p + 1; q < 4; q++) off += A[p][q] * A[p][q];
        if (!(off > 0.0)) break;
        #pragma unroll
        for (int p = 0; p < 3; p++)
            #pragma unroll
            for (int q = p + 1; q < 4; q++) {
                const double apq = A[p][q];
                if (apq == 0.0) continue;
                // rotation J (J_pp = J_qq = c, J_pq = s, J_qp = -s) with (J^T A J)_pq = 0; t = tan of the smaller rotation angle
                const double theta = (A[q][q] - A[p][p]) / (2.0 * apq);
                const double t = fabs(theta) > 1e150 ? 0.5 / theta : (theta >= 0.0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
                const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
                #pragma unroll
                for (int k = 0; k < 4; k++) {
                    const double akp = A[k][p], akq = A[k][q];
                    A[k][p] = c * akp - s * akq; A[k][q] = s * akp + c * akq;
                }
                #pragma unroll
                for (int k = 0; k < 4; k++) {
                    const double apk = A[p][k], aqk = A[q][k];
                    A[p][k] = c * apk - s * aqk; A[q][k] = s * apk + c * aqk;
                }
                A[p][q] = A[q][p] = 0.0;
                #pragma unroll
                for (int k = 0; k < 4; k++) {
                    const double vkp = V[k][p], vkq = V[k][q];
                    V[k][p] = c * vkp - s * vkq; V[k][q] = s * vkp + c * vkq;
                }
            }
    }
    double best = A[0][0], e[4] = {V[0][0], V[1][0], V[2][0], V[3][0]};
    #pragma unroll
    for (int i = 1; i < 4; i++)
        if (A[i][i] > best) { best = A[i][i]; e[0] = V[0][i]; e[1] = V[1][i]; e[2] = V[2][i]; e[3] = V[3][i]; }
    double sg = e[3] > 0.0 ? 1.0 : e[3] < 0.0 ? -1.0 : 0.0;
    #pragma unroll
    for (int i = 0; i < 3; i++) if (sg == 0.0) sg = e[i] > 0.0 ? 1.0 : e[i] < 0.0 ? -1.0 : 0.0;
    if (sg == 0.0) sg = 1.0;
    #pragma unroll
    for (int i = 0; i < 4; i++) v[i] = sg * e[i];
    *lambda = best;
}
// the 6-vector of one particle about the mean: d = ~Tbm * pose in rmagine's float Transform algebra, (d.t, roll, pitch, yaw of d.R)
B2_DEV void pf_deviation(const Tf& Tbm_inv, const Tf& pose, float v[6])
{
    const Tf d = tf_mul(Tbm_inv, pose);
    v[0] = d.t.x; v[1] = d.t.y; v[2] = d.t.z;
    quat_to_euler(d.R, v[3], v[4], v[5]);
}
// pass-1 accumulator slots (FP64): the sums, then min / max of L, then the AABB
#define B2_EST_SUM_L 0
#define B2_EST_SUM_L2 1
#define B2_EST_SUM_LT 2          /* 3 */
#define B2_EST_SUM_LQQ 5         /* 10: xx xy xz xw yy yz yw zz zw ww */
#define B2_EST_NSUM 15
#define B2_EST_MIN_L 15
#define B2_EST_MAX_L 16
#define B2_EST_BB_MIN 17         /* 3 */
#define B2_EST_BB_MAX 20         /* 3 */
#define B2_EST_NV1 23
#define B2_EST_NV2 21            /* pass 2: upper triangle of sum L v v^T, row by row */
#define B2_EST_NV_MAX 23          /* partials per block: the larger of the two passes */
struct PfEstimateScratch {
    b2_particle_stats rec;       // the result, copied to the host after pass 2
    b2_transform Tbm;            // float mean written by pass 1, read by pass 2
    double L_sum;                // pass 1's sum of L (the weights' denominator)
    unsigned int ticket[2];      // one last-block ticket per pass
};
// Which accumulator slots of a grid reduction are sums, minima and maxima (every other slot is a maximum).  Pass 1: the slots below
// B2_EST_NSUM are sums; every pass-2 slot is a sum.  Min and max ignore NaN like std::min / std::max with the running value first.
struct EstSlots1 {
    static B2_DEV bool is_sum(int slot) { return slot < B2_EST_NSUM; }
    static B2_DEV bool is_min(int slot) { return slot == B2_EST_MIN_L || (slot >= B2_EST_BB_MIN && slot < B2_EST_BB_MAX); }
};
struct EstSlots2 {
    static B2_DEV bool is_sum(int) { return true; }
    static B2_DEV bool is_min(int) { return false; }
};
template <class SLOTS> B2_DEV double est_combine(int slot, double a, double b)
{
    if (SLOTS::is_sum(slot)) return a + b;
    if (SLOTS::is_min(slot)) return b < a ? b : a;
    return a < b ? b : a;
}
template <class SLOTS> B2_DEV double est_identity(int slot)
{
    if (SLOTS::is_sum(slot)) return 0.0;
    return SLOTS::is_min(slot) ? f64_inf() : -f64_inf();
}
#ifdef __CUDACC__
template <class SLOTS> __device__ __forceinline__ double est_warp(int slot, double v)
{
    #pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = est_combine<SLOTS>(slot, v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}
// block reduction of NV per-thread values to partials[blockIdx.x * NV + slot]; then the last block reduces the partials in a fixed order
// (warp w handles slots w, w + 8, ...; lane l takes blocks l, l + 32, ...; then a warp butterfly) into tot[NV].  True in the last block only.
template <int NV, class SLOTS>
__device__ __forceinline__ bool est_grid_reduce(double (&acc)[NV], double* __restrict__ partials, unsigned int* __restrict__ ticket, double* s_w /* [8][NV] */, double* tot,
                                                bool& is_last)
{
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    #pragma unroll
    for (int j = 0; j < NV; j++) acc[j] = est_warp<SLOTS>(j, acc[j]);
    if (lane == 0) for (int j = 0; j < NV; j++) s_w[warp * NV + j] = acc[j];
    __syncthreads();
    if (threadIdx.x < NV) {
        double a = s_w[threadIdx.x];
        for (int w = 1; w < 8; w++) a = est_combine<SLOTS>(threadIdx.x, a, s_w[w * NV + threadIdx.x]);
        partials[(size_t)blockIdx.x * NV + threadIdx.x] = a;
        __threadfence();
    }
    __syncthreads();
    if (threadIdx.x == 0) is_last = atomicAdd(ticket, 1u) == gridDim.x - 1;
    __syncthreads();
    if (!is_last) return false;
    __threadfence();
    for (int j = warp; j < NV; j += 8) {
        double a = est_identity<SLOTS>(j);
        for (uint32_t b = lane; b < gridDim.x; b += 32) a = est_combine<SLOTS>(j, a, __ldcg(partials + (size_t)b * NV + j));
        a = est_warp<SLOTS>(j, a);
        if (lane == 0) tot[j] = a;
    }
    __syncthreads();
    return true;
}
// pass 1: 36 B read per particle (32 B pose, the 4 B likelihood.mean)
__global__ void __launch_bounds__(256) k_pf_estimate_moments(const b2_transform* __restrict__ poses, const b2_particle_attr* __restrict__ attrs, uint32_t k,
                                                             double* __restrict__ partials, PfEstimateScratch* __restrict__ sc)
{
    __shared__ double s_w[8 * B2_EST_NV1], tot[B2_EST_NV1];
    __shared__ bool is_last;
    double acc[B2_EST_NV1];
    #pragma unroll
    for (int j = 0; j < B2_EST_NSUM; j++) acc[j] = 0.0;
    acc[B2_EST_MIN_L] = 1.7976931348623157e308; acc[B2_EST_MAX_L] = 0.0;                  // L_min = DBL_MAX, L_max = 0.0 (:664-665)
    #pragma unroll
    for (int c = 0; c < 3; c++) { acc[B2_EST_BB_MIN + c] = 3.402823466e38; acc[B2_EST_BB_MAX + c] = -3.402823466e38; }   // rm::AABB::init [RM-recalled]
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < k; i += gridDim.x * blockDim.x) {
        const Tf P = tf_load(poses + i);
        const double L = (double)attrs[i].likelihood.mean;
        acc[B2_EST_SUM_L] += L; acc[B2_EST_SUM_L2] += L * L;
        acc[B2_EST_MIN_L] = est_combine<EstSlots1>(B2_EST_MIN_L, acc[B2_EST_MIN_L], L); acc[B2_EST_MAX_L] = est_combine<EstSlots1>(B2_EST_MAX_L, acc[B2_EST_MAX_L], L);
        const double t[3] = {(double)P.t.x, (double)P.t.y, (double)P.t.z}, q[4] = {(double)P.R.x, (double)P.R.y, (double)P.R.z, (double)P.R.w};
        #pragma unroll
        for (int c = 0; c < 3; c++) {
            acc[B2_EST_SUM_LT + c] += L * t[c];
            acc[B2_EST_BB_MIN + c] = est_combine<EstSlots1>(B2_EST_BB_MIN, acc[B2_EST_BB_MIN + c], t[c]);
            acc[B2_EST_BB_MAX + c] = est_combine<EstSlots1>(B2_EST_BB_MAX, acc[B2_EST_BB_MAX + c], t[c]);
        }
        int s = B2_EST_SUM_LQQ;
        #pragma unroll
        for (int a = 0; a < 4; a++) {
            const double La = L * q[a];
            #pragma unroll
            for (int b = a; b < 4; b++) acc[s++] += La * q[b];
        }
    }
    if (!est_grid_reduce<B2_EST_NV1, EstSlots1>(acc, partials, sc->ticket, s_w, tot, is_last)) return;
    if (threadIdx.x != 0) return;
    const double Ls = tot[B2_EST_SUM_L], n = (double)k, mean = Ls / n, var = tot[B2_EST_SUM_L2] / n - mean * mean;
    const bool ok = Ls > 0.0 && Ls < f64_inf();                                             // else the reference divides by zero (decision E3)
    const double nan = f64_nan();
    double M[16];
    int s = B2_EST_SUM_LQQ;
    for (int a = 0; a < 4; a++) for (int b = a; b < 4; b++) { M[4 * a + b] = M[4 * b + a] = ok ? tot[s] / Ls : nan; s++; }
    double qv[4], lambda;
    sym4_top_eigvec(M, qv, &lambda);
    b2_transform T; memset(&T, 0, sizeof(T));
    T.R.x = (float)qv[0]; T.R.y = (float)qv[1]; T.R.z = (float)qv[2]; T.R.w = (float)qv[3];
    T.t.x = (float)(ok ? tot[B2_EST_SUM_LT] / Ls : nan); T.t.y = (float)(ok ? tot[B2_EST_SUM_LT + 1] / Ls : nan); T.t.z = (float)(ok ? tot[B2_EST_SUM_LT + 2] / Ls : nan);
    sc->Tbm = T; sc->L_sum = Ls;
    b2_particle_stats& r = sc->rec;
    r.position[0] = T.t.x; r.position[1] = T.t.y; r.position[2] = T.t.z;
    r.orientation[0] = T.R.x; r.orientation[1] = T.R.y; r.orientation[2] = T.R.z; r.orientation[3] = T.R.w;
    r.shift = tot[B2_EST_MIN_L];
    for (int c = 0; c < 3; c++) { r.trans_bb_min[c] = (double)(float)tot[B2_EST_BB_MIN + c]; r.trans_bb_max[c] = (double)(float)tot[B2_EST_BB_MAX + c]; }
    r.likelihood.min = tot[B2_EST_MIN_L]; r.likelihood.max = tot[B2_EST_MAX_L];
    r.likelihood.mean = mean; r.likelihood.sigma = var < 0.0 ? 0.0 : sqrt(var);           // a rounding-only negative variance gives 0 (decision E4)
    r.nparticles = k;
    sc->ticket[0] = 0u;
}
// pass 2: the same 36 B per particle again, and Tbm from pass 1 (device memory)
__global__ void __launch_bounds__(256) k_pf_estimate_cov(const b2_transform* __restrict__ poses, const b2_particle_attr* __restrict__ attrs, uint32_t k,
                                                         double* __restrict__ partials, PfEstimateScratch* __restrict__ sc)
{
    __shared__ double s_w[8 * B2_EST_NV2], tot[B2_EST_NV2];
    __shared__ bool is_last;
    double acc[B2_EST_NV2];
    #pragma unroll
    for (int j = 0; j < B2_EST_NV2; j++) acc[j] = 0.0;
    const Tf Tinv = tf_inv(tf_from_pod(sc->Tbm));
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < k; i += gridDim.x * blockDim.x) {
        const double L = (double)attrs[i].likelihood.mean;
        float v[6];
        pf_deviation(Tinv, tf_load(poses + i), v);
        int s = 0;
        #pragma unroll
        for (int a = 0; a < 6; a++) {
            const double La = L * (double)v[a];
            #pragma unroll
            for (int b = a; b < 6; b++) acc[s++] += La * (double)v[b];
        }
    }
    if (!est_grid_reduce<B2_EST_NV2, EstSlots2>(acc, partials, sc->ticket + 1, s_w, tot, is_last)) return;
    if (threadIdx.x != 0) return;
    const double Ls = sc->L_sum;
    const bool ok = Ls > 0.0 && Ls < f64_inf();
    const double nan = f64_nan();
    int s = 0;
    for (int a = 0; a < 6; a++) for (int b = a; b < 6; b++) { sc->rec.covariance[6 * a + b] = sc->rec.covariance[6 * b + a] = ok ? tot[s] / Ls : nan; s++; }
    sc->ticket[1] = 0u;
}
#endif

// ---------------------------------------------------------------------------------------------------------------------
// Residual resampling: ResidualResamplerCPU::update (rmcl_ros/src/rmcl/ResidualResamplerCPU.cpp:55-202).  Draw j (64-bit) picks parent
// word j % 4 of Philox4x32-10 with counter (lo(j / 4), B2_PF_RESIDUAL_DRAW_TAG, step, hi(j / 4)) and key = seed, modulo n; it inserts
// min(floor(L / S * M), slots left) copies.  The copy in output slot k draws its six normals from words 0-5 of the counters
// (k, B2_PF_RESIDUAL_NOISE_TAG, step, 0 and 1).  Draws are keyed by their index and copies by their slot, so neither the chunking of the
// draws nor the slice of slots one call writes can change a byte.  The draws run in chunks: k_pf_residual_counts, an inclusive scan of the
// counts, k_pf_residual_find, then k_pf_residual_expand over the slots the chunk filled (b2_pf_resample_residual).  SURVEY D31-D34.
// ---------------------------------------------------------------------------------------------------------------------
#define B2_PF_RESIDUAL_DRAW_TAG 4u
#define B2_PF_RESIDUAL_NOISE_TAG 5u
// the parent of draw j among n particles (:104, std::uniform_int_distribution(0, n - 1) replaced, SURVEY D33)
B2_DEV uint32_t residual_parent(uint64_t seed, uint32_t step, uint64_t j, uint32_t n)
{
    uint32_t r[4];
    const uint64_t b = j >> 2;
    philox4x32_10((uint32_t)b, B2_PF_RESIDUAL_DRAW_TAG, step, (uint32_t)(b >> 32), (uint32_t)seed, (uint32_t)(seed >> 32), r);
    return philox_word(r, (uint32_t)(j & 3u)) % n;
}
// n_expected_insertions = (size_t)(L / weight_sum * (double)M) (:110-120); 0 <= L <= S (checked on the host) keeps it in [0, M]
B2_DEV uint64_t residual_count(float L, double S, uint64_t M)
{
    const double c = (double)L / S * (double)M;
    return c >= (double)M ? M : (uint64_t)c;
}
// the six N(0, 1) draws of output slot k, in the reference's order tx, ty, tz, roll, pitch, yaw (:151-157)
B2_DEV void residual_normals(uint64_t seed, uint32_t step, uint32_t k, float N[6])
{
    uint32_t r[8];
    philox4x32_10(k, B2_PF_RESIDUAL_NOISE_TAG, step, 0u, (uint32_t)seed, (uint32_t)(seed >> 32), r);
    philox4x32_10(k, B2_PF_RESIDUAL_NOISE_TAG, step, 1u, (uint32_t)seed, (uint32_t)(seed >> 32), r + 4);
    box_muller3(r, N);
}
// one copy of the parent (pn, an) (:129-177): noise scales (float)(min_noise / (L / L_max)), so less likely parents spread wider; n_meas
// *= (float)(pow(forget_per_meter, |d.t|^2) * pow(forget_per_radian, |d.R|)) with d = ~pose * pose_new, the squared translation and the
// quaternion norm as the reference takes them (SURVEY D32), double pow of the float arguments (SURVEY E5); the stamp is the parent's.
B2_DEV void residual_copy(b2_transform pn, b2_particle_attr an, double L_max, const float N[6], const b2_gladiator_config& cfg, b2_transform* out_p,
                          b2_particle_attr* out_a)
{
    const double Lmn = (double)an.likelihood.mean / L_max;                                  // L_max_normed (:112)
    const float s[6] = {(float)((double)cfg.min_noise_tx / Lmn), (float)((double)cfg.min_noise_ty / Lmn), (float)((double)cfg.min_noise_tz / Lmn),
                        (float)((double)cfg.min_noise_roll / Lmn), (float)((double)cfg.min_noise_pitch / Lmn), (float)((double)cfg.min_noise_yaw / Lmn)};   // :143-149
    Tf diff;
    const Tf pnew = pf_perturb(tf_from_pod(pn), N, s, diff);                               // :151-160
    const float trans_dist = add(add(mul(diff.t.x, diff.t.x), mul(diff.t.y, diff.t.y)), mul(diff.t.z, diff.t.z));   // :163 l2normSquared
    const float rot_dist = quat_l2norm(diff.R);                                            // :164
    const float f = (float)(pow((double)cfg.likelihood_forget_per_meter, (double)trans_dist) * pow((double)cfg.likelihood_forget_per_radian, (double)rot_dist));   // :165-166
    an.likelihood.n_meas = (uint32_t)mul((float)an.likelihood.n_meas, f);                 // :167 uint *= float
    pn.R.x = pnew.R.x; pn.R.y = pnew.R.y; pn.R.z = pnew.R.z; pn.R.w = pnew.R.w; pn.t.x = pnew.t.x; pn.t.y = pnew.t.y; pn.t.z = pnew.t.z;
    *out_p = pn; *out_a = an;
}
// slots of the statistics pass: the sum of L, its minimum (from DBL_MAX) and its maximum (from 0.0), as pass 1 of the estimate takes them
#define B2_RES_SUM 0
#define B2_RES_MIN 1
#define B2_RES_MAX 2
#define B2_RES_NV 3
struct ResidualSlots {
    static B2_DEV bool is_sum(int slot) { return slot == B2_RES_SUM; }
    static B2_DEV bool is_min(int slot) { return slot == B2_RES_MIN; }
};
// the device record the host reads back after the statistics pass and after every chunk
struct PfResidualState {
    double S, L_min, L_max;             // statistics pass
    unsigned long long filled, used;    // k_pf_residual_find: slots the chunk filled, draws it consumed
    unsigned int ticket, pad;
};
#ifdef __CUDACC__
// The set's weight statistics S, L_min and L_max (api.cu pf_weight_stats), for likelihoodStats (compute_stats, rmcl_ros/src/rmcl/
// resampling.cu:41-92), the residual and KLD resamplers, the clusters and the recovery.  4 B read per particle; grid, block and grid-stride
// order of k_pf_estimate_moments, so S is bit-equal to its L_sum for the same n
__global__ void __launch_bounds__(256) k_pf_residual_stats(const b2_particle_attr* __restrict__ attrs, uint32_t n, double* __restrict__ partials, PfResidualState* __restrict__ st)
{
    __shared__ double s_w[8 * B2_RES_NV], tot[B2_RES_NV];
    __shared__ bool is_last;
    double acc[B2_RES_NV];
    acc[B2_RES_SUM] = 0.0; acc[B2_RES_MIN] = 1.7976931348623157e308; acc[B2_RES_MAX] = 0.0;     // :73-83
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const double L = (double)attrs[i].likelihood.mean;
        acc[B2_RES_SUM] += L;
        acc[B2_RES_MIN] = est_combine<ResidualSlots>(B2_RES_MIN, acc[B2_RES_MIN], L); acc[B2_RES_MAX] = est_combine<ResidualSlots>(B2_RES_MAX, acc[B2_RES_MAX], L);
    }
    if (!est_grid_reduce<B2_RES_NV, ResidualSlots>(acc, partials, &st->ticket, s_w, tot, is_last)) return;
    if (threadIdx.x != 0) return;
    st->S = tot[B2_RES_SUM]; st->L_min = tot[B2_RES_MIN]; st->L_max = tot[B2_RES_MAX];
    st->ticket = 0u;
}
// one thread per draw d0 + i of the chunk: its parent and its count (4 B gathered per draw)
__global__ void __launch_bounds__(256) k_pf_residual_counts(const b2_particle_attr* __restrict__ attrs, uint32_t n, uint64_t M, double S, uint64_t seed, uint32_t step,
                                                            uint64_t d0, uint32_t len, uint32_t* __restrict__ parents, unsigned long long* __restrict__ counts)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= len) return;
    const uint32_t p = residual_parent(seed, step, d0 + i, n);
    parents[i] = p;
    counts[i] = residual_count(attrs[p].likelihood.mean, S, M);
}
// one thread: over the chunk's inclusive prefix of the counts, the first draw whose running fill reaches the `left` slots still empty
// (that draw ends the reference's loop, :102) -- or the whole chunk when the fill stays short of it
__global__ void k_pf_residual_find(const unsigned long long* __restrict__ prefix, uint32_t len, uint64_t left, PfResidualState* __restrict__ st)
{
    if (prefix[len - 1] < left) { st->filled = prefix[len - 1]; st->used = len; return; }
    uint32_t lo = 0, hi = len - 1;
    while (lo < hi) { const uint32_t mid = lo + (hi - lo) / 2; if (prefix[mid] < left) lo = mid + 1; else hi = mid; }
    st->filled = left; st->used = lo + 1u;
}
// one thread per output slot k = k0 + i that this chunk filled (k - fill0 < the chunk's fill): its draw is the first whose prefix exceeds
// k - fill0; writes entry k - first of the caller's slice.  68 B gathered from the parent and 68 B written per slot.
__global__ void __launch_bounds__(256) k_pf_residual_expand(const b2_transform* __restrict__ poses, const b2_particle_attr* __restrict__ attrs, const uint32_t* __restrict__ parents,
                                                            const unsigned long long* __restrict__ prefix, uint32_t len, uint64_t fill0, uint32_t k0, uint32_t n_k, uint32_t first,
                                                            double L_max, b2_gladiator_config cfg, uint64_t seed, uint32_t step, b2_transform* __restrict__ poses_new,
                                                            b2_particle_attr* __restrict__ attrs_new)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_k) return;
    const uint32_t k = k0 + i;
    const uint64_t local = (uint64_t)k - fill0;
    uint32_t lo = 0, hi = len - 1;
    while (lo < hi) { const uint32_t mid = lo + (hi - lo) / 2; if (prefix[mid] <= local) lo = mid + 1; else hi = mid; }
    const uint32_t p = parents[lo];
    float N[6];
    residual_normals(seed, step, k, N);
    residual_copy(poses[p], attrs[p], L_max, N, cfg, poses_new + (k - first), attrs_new + (k - first));
}
#endif

// ---------------------------------------------------------------------------------------------------------------------
// KLD-sampling (Fox, "Adapting the sample size in particle filters through KLD-sampling", IJRR 2003; the open TODO of rmcl/docs/RMCL.md:80-83,
// no reference implementation): draws parents one at a time and stops once the number drawn reaches the chi-square bound on the number of
// histogram bins they occupy (b2_pf_resample_kld).  Weights are integers w_i = (uint64)(L_i / L_max * 2^32) with the 64-bit inclusive prefix
// W; draw j takes u = words 2(j % 2) (low) and 2(j % 2) + 1 (high) of Philox4x32-10 with counter (lo(j / 2), 6, step, hi(j / 2)) and key =
// seed, and its parent is the smallest i with W[i] > mulhi64(u, W[n-1]).  A bin is the parent's (x, y, z, yaw sector) cell, computed without
// transcendental functions, so host and device agree bit for bit.  Slot j is draw j's parent copied as residual_copy copies (normals of
// residual_normals keyed by the slot).  The draws run in chunks: k_pf_kld_draw inserts the keys into a hash set that keeps each key's first
// draw, k_pf_kld_flags marks the first draws, a scan counts the bins, k_pf_kld_stop finds the first draw that meets the stop rule, one
// read-back, then k_pf_kld_expand over the slots the chunk filled.  SURVEY appendix G.
// ---------------------------------------------------------------------------------------------------------------------
#define B2_PF_KLD_DRAW_TAG 6u
#define B2_KLD_NONFINITE_KEY 0xFFFFFFFFFFFFFFFFull     // bit 15 is never set in a real key
#define B2_KLD_XY_HALF 524288.0f                        // 2^19: ix, iy in [-2^19, 2^19)
#define B2_KLD_Z_HALF 128.0f                            // 2^7:  iz in [-2^7, 2^7)
#define B2_KLD_MAX_SECTORS 32768u
#if B2_ON_DEVICE
B2_DEV uint64_t kld_mulhi64(uint64_t a, uint64_t b) { return __umul64hi(a, b); }
B2_DEV double kld_sub_d(double a, double b) { return __dadd_rn(a, -b); }
B2_DEV double kld_div_d(double a, double b) { return __ddiv_rn(a, b); }
#else
B2_DEV uint64_t kld_mulhi64(uint64_t a, uint64_t b) { return (uint64_t)(((unsigned __int128)a * b) >> 64); }
B2_DEV double kld_sub_d(double a, double b) { return a - b; }
B2_DEV double kld_div_d(double a, double b) { return a / b; }
#endif
// the integer weight of likelihood L: at most 2^32, exact sums in 64 bits for any n < 2^32
B2_DEV uint64_t kld_weight(float L, double L_max) { return (uint64_t)mul_d(kld_div_d((double)L, L_max), 4294967296.0); }
// the parent of draw j among the n particles of the inclusive weight prefix W (W[n-1] > 0): bias at most W[n-1] / 2^64 per particle
B2_DEV uint32_t kld_parent(uint64_t seed, uint32_t step, uint64_t j, const unsigned long long* W, uint32_t n)
{
    uint32_t r[4];
    const uint64_t b = j >> 1;
    philox4x32_10((uint32_t)b, B2_PF_KLD_DRAW_TAG, step, (uint32_t)(b >> 32), (uint32_t)seed, (uint32_t)(seed >> 32), r);
    const uint64_t u = (j & 1u) ? ((uint64_t)r[3] << 32 | r[2]) : ((uint64_t)r[1] << 32 | r[0]);
    const uint64_t x = kld_mulhi64(u, W[n - 1]);
    uint32_t lo = 0, hi = n - 1;                         // W[n-1] > x: the answer lies in [0, n-1]
    while (lo < hi) { const uint32_t mid = lo + (hi - lo) / 2; if ((uint64_t)W[mid] > x) hi = mid; else lo = mid + 1; }
    return lo;
}
// the bin resolution: res_z = 0 leaves z unbinned; cs = the K boundary vectors (cos, sin) of theta_k = -pi + 2 pi k / K as floats
struct KldBins { float res_xy, res_z; uint32_t K; const float* cs; };
// boundary k lies in the lower half (theta_k < 0) iff 2k < K; within one half, theta_k <= phi(h) iff c_k h.y - s_k h.x >= 0 (each product of
// two floats is exact in double, so the sign is exact)
B2_DEV bool kld_at_or_before(const float* cs, uint32_t k, float hx, float hy)
{
    return kld_sub_d(mul_d((double)cs[2 * k], (double)hy), mul_d((double)cs[2 * k + 1], (double)hx)) >= 0.0;
}
// the number of boundaries k in [1, K) with theta_k <= phi(h), phi in [-pi, pi); the predicate is monotone in k within a half
B2_DEV uint32_t kld_sector(float hx, float hy, const float* cs, uint32_t K)
{
    if (hx == 0.0f && hy == 0.0f) return 0u;
    const bool lower = hy < 0.0f || (hy == 0.0f && hx < 0.0f);
    const uint32_t n_low = (K - 1u) / 2u;               // boundaries 1 .. n_low are in the lower half
    uint32_t lo = lower ? 1u : n_low + 1u, hi = lower ? n_low + 1u : K;     // count the true prefix of [lo, hi)
    const uint32_t base = lo;
    while (lo < hi) { const uint32_t mid = lo + (hi - lo) / 2; if (kld_at_or_before(cs, mid, hx, hy)) lo = mid + 1; else hi = mid; }
    return (lower ? 0u : n_low) + (lo - base);
}
B2_DEV float kld_cell(float v, float res, float half)
{
    float c = floorf(dvd(v, res));
    c = c < -half ? -half : c;
    c = c > half - 1.0f ? half - 1.0f : c;
    return c;
}
// the bin key of pose p: (ix + 2^19) << 44 | (iy + 2^19) << 24 | (iz + 2^7) << 16 | yaw sector; roll and pitch are not binned
B2_DEV uint64_t kld_key(const b2_transform& p, const KldBins& b)
{
    if (!(finite_f32(p.t.x) && finite_f32(p.t.y) && finite_f32(p.t.z) && finite_f32(p.R.x) && finite_f32(p.R.y) && finite_f32(p.R.z) && finite_f32(p.R.w)))
        return B2_KLD_NONFINITE_KEY;
    const float ix = kld_cell(p.t.x, b.res_xy, B2_KLD_XY_HALF), iy = kld_cell(p.t.y, b.res_xy, B2_KLD_XY_HALF);
    const float iz = b.res_z > 0.0f ? kld_cell(p.t.z, b.res_z, B2_KLD_Z_HALF) : 0.0f;
    const float x = p.R.x, y = p.R.y, z = p.R.z, w = p.R.w;
    const float hx = sub(1.0f, mul(2.0f, add(mul(y, y), mul(z, z))));     // R e_x: 1 - 2(y^2 + z^2), 2(xy + wz)
    const float hy = mul(2.0f, add(mul(x, y), mul(w, z)));
    const uint64_t sector = kld_sector(hx, hy, b.cs, b.K);
    return (uint64_t)((int64_t)ix + 524288) << 44 | (uint64_t)((int64_t)iy + 524288) << 24 | (uint64_t)((int64_t)iz + 128) << 16 | sector;
}
// Fox's bound on the sample count for k occupied bins: ceil((k-1) / (2 eps) * x^3), x = 1 - 2 / (9(k-1)) + sqrt(2 / (9(k-1))) z, in double
// rounded in the order written (pf_resample_limit's arithmetic); k <= 1 (a converged set) gives n_min
B2_DEV uint64_t kld_bound(uint64_t k, double epsilon, double z, uint32_t n_min)
{
    if (k <= 1u) return n_min;
    const double km1 = (double)(k - 1u);
    const double a = kld_div_d(2.0, mul_d(9.0, km1));
    const double x = add_d(kld_sub_d(1.0, a), mul_d(sqrt_d(a), z));
    const double v = mul_d(kld_div_d(km1, mul_d(2.0, epsilon)), mul_d(mul_d(x, x), x));
    if (!(v > 0.0)) return 0u;
    const double c = ceil(v);
    return c >= 18446744073709551616.0 ? ~0ull : (uint64_t)c;
}
// the stop rule after draw j with k bins among draws 0 .. j
B2_DEV bool kld_stop(uint64_t j, uint64_t k, double epsilon, double z, uint32_t n_min, uint64_t n_max)
{
    const uint64_t b = kld_bound(k, epsilon, z, n_min);
    return j + 1u >= (b > n_min ? b : (uint64_t)n_min) || j + 1u == n_max;
}
// the device record the host reads back after every chunk
struct PfKldState {
    unsigned long long stop;     // min over the chunk's draws i that meet the stop rule of i << 32 | bins among the chunk's draws 0 .. i
    unsigned int bins, pad;      // bins among the chunk's draws
};
#ifdef __CUDACC__
B2_DEV uint64_t kld_hash(uint64_t v)                    // splitmix64's finaliser
{
    v ^= v >> 30; v *= 0xbf58476d1ce4e5b9ull; v ^= v >> 27; v *= 0x94d049bb133111ebull; v ^= v >> 31;
    return v;
}
__global__ void __launch_bounds__(256) k_pf_kld_weights(const b2_particle_attr* __restrict__ attrs, uint32_t n, double L_max, unsigned long long* __restrict__ w)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) w[i] = kld_weight(attrs[i].likelihood.mean, L_max);
}
// one thread per draw d0 + i: its parent, and its key into the hash set (stored as key ^ 0x8000, so the memset 0 marks empty slots and no
// key stores 0); each slot keeps the smallest draw index of its key, so membership and first draws do not depend on the insertion order
__global__ void __launch_bounds__(256) k_pf_kld_draw(const unsigned long long* __restrict__ W, uint32_t n, const b2_transform* __restrict__ poses, KldBins bins,
                                                     uint64_t seed, uint32_t step, uint64_t d0, uint32_t len, unsigned long long* __restrict__ keys,
                                                     unsigned int* __restrict__ first, uint64_t mask, uint32_t* __restrict__ parents, unsigned long long* __restrict__ slots,
                                                     PfKldState* __restrict__ st)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i == 0) { st->stop = ~0ull; st->bins = 0u; }
    if (i >= len) return;
    const uint64_t j = d0 + i;
    const uint32_t p = kld_parent(seed, step, j, W, n);
    parents[i] = p;
    const unsigned long long v = kld_key(poses[p], bins) ^ 0x8000ull;
    uint64_t s = kld_hash(v) & mask;
    for (;;) {
        const unsigned long long old = atomicCAS(keys + s, 0ull, v);
        if (old == 0ull || old == v) break;
        s = (s + 1u) & mask;
    }
    atomicMin(first + s, (unsigned int)j);
    slots[i] = s;
}
// a draw opens a bin iff it is the first draw of its key
__global__ void __launch_bounds__(256) k_pf_kld_flags(const unsigned int* __restrict__ first, const unsigned long long* __restrict__ slots, uint64_t d0, uint32_t len,
                                                      uint32_t* __restrict__ flags)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < len) flags[i] = first[slots[i]] == (unsigned int)(d0 + i) ? 1u : 0u;
}
// the first draw of the chunk that meets the stop rule: every draw is tested (the rule is not monotone in j), the lowest lane of each warp
// that meets it takes part in one atomicMin
__global__ void __launch_bounds__(256) k_pf_kld_stop(const uint32_t* __restrict__ cum, uint64_t d0, uint32_t len, uint64_t bins0, uint32_t n_min, uint64_t n_max,
                                                     double epsilon, double z, PfKldState* __restrict__ st)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    const bool in = i < len;
    const uint32_t c = in ? cum[i] : 0u;
    const bool hit = in && kld_stop(d0 + i, bins0 + c, epsilon, z, n_min, n_max);
    const unsigned m = __ballot_sync(0xffffffffu, hit);
    if (hit && (threadIdx.x & 31u) == (unsigned)(__ffs(m) - 1)) atomicMin(&st->stop, (unsigned long long)i << 32 | c);
    if (i + 1u == len) st->bins = c;
}
// one thread per output slot k = k0 + i that this chunk filled: slot k is draw k's parent, copied with the normals of slot k; writes entry
// k - first of the caller's slice.  68 B gathered from the parent and 68 B written per slot.
__global__ void __launch_bounds__(256) k_pf_kld_expand(const b2_transform* __restrict__ poses, const b2_particle_attr* __restrict__ attrs, const uint32_t* __restrict__ parents,
                                                       uint64_t d0, uint32_t k0, uint32_t n_k, uint32_t first, double L_max, b2_gladiator_config cfg, uint64_t seed,
                                                       uint32_t step, b2_transform* __restrict__ poses_new, b2_particle_attr* __restrict__ attrs_new)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_k) return;
    const uint32_t k = k0 + i;
    const uint32_t p = parents[k - d0];
    float N[6];
    residual_normals(seed, step, k, N);
    residual_copy(poses[p], attrs[p], L_max, N, cfg, poses_new + (k - first), attrs_new + (k - first));
}
#endif

// ---------------------------------------------------------------------------------------------------------------------
// Pose hypotheses of the particle set (b2_pf_cluster_stats; what AMCL reports as pf_cluster_stats; no reference implementation, SURVEY
// appendix H): the members (integer weight > 0, finite pose) are binned with kld_key, occupied bins that touch (each of x, y, z within one
// cell, the yaw sector within one modulo K) are joined, and every connected component is a cluster with the exact integer sum of its
// members' weights.  k_pf_cluster_insert puts the keys into KLD's hash set and sums weight and member count per slot; k_pf_cluster_hook
// joins every slot with its occupied neighbours of smaller key in a union-find forest over slot indices whose links only ever lead to a
// smaller key, so a component's root is its smallest key whatever the order of the threads (lock-free hooking of roots with path halving,
// after Jaiganesh and Burtscher's ECL-CC); k_pf_cluster_flatten points every slot at its root and sums weight, members and bins there.  The
// roots are then sorted by (weight descending, key ascending), every particle takes its root's rank as its label, a stable sort of the
// particle indices by min(label, n_records) lines the recorded clusters' members up in index order, and k_pf_estimate_moments /
// k_pf_estimate_cov run on each gathered segment.  Every sum is an integer, so no result depends on the order in which threads ran.
// ---------------------------------------------------------------------------------------------------------------------
#define B2_CLUSTER_NONE 0xFFFFFFFFu                     // the label of a particle in no cluster, and the slot of one in no bin
#define B2_CLUSTER_MAX_RECORDS 16u
#define B2_CLUSTER_MAX_ROUNDS 64u
// the key of the bin at offset (dx, dy, dz, ds), each in {-1, 0, 1}, from the bin `key` (kld_key's layout), or B2_KLD_NONFINITE_KEY where
// there is none: x, y and z end at their clamps, z has no neighbours when it is not binned, the yaw sector wraps modulo K.  With K <= 2
// several offsets name the same bin (or the bin itself); joining a pair twice changes nothing.
B2_DEV uint64_t kld_key_neighbour(uint64_t key, int dx, int dy, int dz, int ds, uint32_t K, bool has_z)
{
    const int64_t ix = (int64_t)(key >> 44) + dx, iy = (int64_t)((key >> 24) & 0xFFFFFu) + dy, iz = (int64_t)((key >> 16) & 0xFFu) + dz;
    if (ix < 0 || ix > 0xFFFFF || iy < 0 || iy > 0xFFFFF || iz < 0 || iz > 0xFF || (!has_z && dz != 0)) return B2_KLD_NONFINITE_KEY;
    const uint64_t s = (uint64_t)(((int64_t)(key & 0xFFFFu) + ds + (int64_t)K) % (int64_t)K);
    return (uint64_t)ix << 44 | (uint64_t)iy << 24 | (uint64_t)iz << 16 | s;
}
// offset o of the 81 (27 when z is not binned) around a bin, the bin itself included
B2_DEV uint64_t kld_key_offset(uint64_t key, uint32_t o, uint32_t K, bool has_z)
{
    return kld_key_neighbour(key, (int)(o / 3u % 3u) - 1, (int)(o / 9u % 3u) - 1, has_z ? (int)(o / 27u) - 1 : 0, (int)(o % 3u) - 1, K, has_z);
}
// the device record the host reads back after the labelling
struct PfClusterState {
    unsigned long long weight_total;   // the sum of the members' integer weights
    unsigned int n_clustered, bins, n_clusters;
    unsigned int retry;                // a bounded loop of k_pf_cluster_hook ran out: the round has to be repeated
    unsigned int fault, pad;           // the hash set had no free slot (it holds 2 n and more: cannot happen)
};
// what the host needs of each recorded cluster before the estimate runs on it
struct PfClusterHead { unsigned long long weight_int, key; unsigned int bins, members; };
#ifdef __CUDACC__
// The lanes of a warp that name the same slot add to it once: the lowest of them adds the sum of their values.  All 32 lanes call it; a lane
// with slot B2_CLUSTER_NONE adds nothing.
__device__ __forceinline__ void cluster_warp_add(uint32_t s, unsigned long long wv, uint32_t cv, uint32_t bv, unsigned long long* __restrict__ w,
                                                 unsigned int* __restrict__ cnt, unsigned int* __restrict__ aux)
{
    const uint32_t lane = threadIdx.x & 31u;
    unsigned long long ws = 0ull;
    uint32_t cs = 0u, bs = 0u;
    bool lowest = true;
    for (uint32_t l = 0; l < 32u; l++) {
        const uint32_t sl = __shfl_sync(0xffffffffu, s, l), cl = __shfl_sync(0xffffffffu, cv, l), bl = __shfl_sync(0xffffffffu, bv, l);
        const unsigned long long wl = __shfl_sync(0xffffffffu, wv, l);
        if (sl == s) { ws += wl; cs += cl; bs += bl; lowest = lowest && l >= lane; }
    }
    if (s == B2_CLUSTER_NONE || !lowest) return;
    if (ws) atomicAdd(w + s, ws);
    if (cs) atomicAdd(cnt + s, cs);
    if (bs) atomicAdd(aux + s, bs);
}
// one thread per particle: a member's key goes into the hash set (as k_pf_kld_draw stores it: key ^ 0x8000, 0 an empty slot); the thread
// that claims a slot makes it its own root.  36 B read per particle (the likelihood, then the pose of a particle of weight > 0).
__global__ void __launch_bounds__(256) k_pf_cluster_insert(const b2_transform* __restrict__ poses, const b2_particle_attr* __restrict__ attrs, uint32_t n, double L_max,
                                                           KldBins bins, unsigned long long* __restrict__ keys, uint64_t mask, unsigned int* __restrict__ parent,
                                                           unsigned long long* __restrict__ w, unsigned int* __restrict__ cnt, uint32_t* __restrict__ slot_of,
                                                           PfClusterState* __restrict__ st)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    unsigned long long wi = 0ull;
    uint32_t s = B2_CLUSTER_NONE;
    if (i < n) {
        wi = kld_weight(attrs[i].likelihood.mean, L_max);
        const uint64_t key = wi > 0ull ? kld_key(poses[i], bins) : B2_KLD_NONFINITE_KEY;
        if (key != B2_KLD_NONFINITE_KEY) {
            const unsigned long long v = key ^ 0x8000ull;
            uint64_t t = kld_hash(v) & mask;
            for (uint64_t probe = 0; probe <= mask; probe++) {          // at most n of the 2 n and more slots are taken: a free one turns up
                const unsigned long long old = atomicCAS(keys + t, 0ull, v);
                if (old == 0ull) parent[t] = (unsigned int)t;
                if (old == 0ull || old == v) { s = (uint32_t)t; break; }
                t = (t + 1u) & mask;
            }
            if (s == B2_CLUSTER_NONE) st->fault = 1u;
        }
        if (s == B2_CLUSTER_NONE) wi = 0ull;
        slot_of[i] = s;
    }
    cluster_warp_add(s, wi, 1u, 0u, w, cnt, nullptr);
    const uint32_t members = __popc(__ballot_sync(0xffffffffu, s != B2_CLUSTER_NONE));
    #pragma unroll
    for (int o = 16; o > 0; o >>= 1) wi += __shfl_xor_sync(0xffffffffu, wi, o);
    if ((threadIdx.x & 31u) == 0u && members) { atomicAdd(&st->weight_total, wi); atomicAdd(&st->n_clustered, members); }
}
// the root of slot x, halving the path on the way.  Keys fall strictly along the links, so a path is shorter than the table.
__device__ __forceinline__ uint32_t cluster_find(volatile unsigned int* parent, uint32_t x, uint64_t mask)
{
    for (uint64_t it = 0; it <= mask; it++) {
        const uint32_t p = parent[x];
        if (p == x) break;
        const uint32_t g = parent[p];
        if (g != p) parent[x] = g;
        x = g;
    }
    return x;
}
// one thread per slot: joins an occupied slot with each occupied neighbour of smaller key (so every pair is joined once, from its larger
// end).  The root with the larger key is hooked under the other tree by one atomicCAS; when another thread hooked it first, the walk goes on
// from where that thread put it, to a strictly smaller key.  Nothing waits for another thread, and every loop ends within the table's size.
__global__ void __launch_bounds__(256) k_pf_cluster_hook(const unsigned long long* __restrict__ keys, uint64_t mask, uint32_t K, int has_z, unsigned int* parent,
                                                         unsigned int* __restrict__ aux, PfClusterState* __restrict__ st)
{
    const uint64_t s = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (s > mask) return;
    const unsigned long long v = keys[s];
    if (v == 0ull) return;
    aux[s] = 0u;
    const uint64_t key = v ^ 0x8000ull;
    const uint32_t n_off = has_z ? 81u : 27u;
    for (uint32_t o = 0; o < n_off; o++) {
        const uint64_t nk = kld_key_offset(key, o, K, has_z != 0);
        if (nk >= key) continue;                                          // none, the bin itself, or a pair its other end joins
        const unsigned long long nv = nk ^ 0x8000ull;
        uint64_t t = kld_hash(nv) & mask;
        bool found = false;
        for (uint64_t probe = 0; probe <= mask; probe++) {
            const unsigned long long cur = keys[t];
            if (cur == 0ull) break;
            if (cur == nv) { found = true; break; }
            t = (t + 1u) & mask;
        }
        if (!found) continue;
        uint32_t a = cluster_find(parent, (uint32_t)s, mask), b = cluster_find(parent, (uint32_t)t, mask);
        bool joined = false;
        for (uint64_t it = 0; it <= mask; it++) {
            if (a == b) { joined = true; break; }
            if (keys[a] < keys[b]) { const uint32_t c = a; a = b; b = c; }   // a has the larger key
            const uint32_t old = atomicCAS(parent + a, a, b);
            if (old == a) { joined = true; break; }
            a = old;
        }
        if (!joined) st->retry = 1u;
    }
}
// one thread per slot, after a round that ran to its end: the slot's root (read only: the forest no longer changes but for these writes,
// which point a slot at its own root), then weight, members and one bin added to the root, and each root appended to the list of clusters
// (in no particular order: the sort that follows has distinct keys)
__global__ void __launch_bounds__(256) k_pf_cluster_flatten(const unsigned long long* __restrict__ keys, uint64_t mask, volatile unsigned int* parent,
                                                            unsigned long long* __restrict__ w, unsigned int* __restrict__ cnt, unsigned int* __restrict__ aux,
                                                            uint32_t* __restrict__ roots, unsigned long long* __restrict__ root_keys, PfClusterState* __restrict__ st)
{
    if (st->retry) return;
    const uint64_t s = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const unsigned long long v = s <= mask ? keys[s] : 0ull;
    uint32_t r = B2_CLUSTER_NONE;
    if (v != 0ull) {
        r = (uint32_t)s;
        for (uint64_t it = 0; it <= mask; it++) { const uint32_t p = parent[r]; if (p == r) break; r = p; }
        parent[s] = r;
    }
    const bool moved = v != 0ull && r != (uint32_t)s;                      // nothing is ever added to a slot that is not a root
    cluster_warp_add(r, moved ? w[s] : 0ull, moved ? cnt[s] : 0u, v != 0ull ? 1u : 0u, w, cnt, aux);
    const uint32_t occupied = __popc(__ballot_sync(0xffffffffu, v != 0ull));
    if ((threadIdx.x & 31u) == 0u && occupied) atomicAdd(&st->bins, occupied);
    if (v != 0ull && r == (uint32_t)s) {
        const uint32_t j = atomicAdd(&st->n_clusters, 1u);
        roots[j] = r; root_keys[j] = v ^ 0x8000ull;
    }
}
// the second sort key of the clusters, already in key order: the complement of the weight, so that the heaviest comes first
__global__ void __launch_bounds__(256) k_pf_cluster_weight_keys(const uint32_t* __restrict__ roots, const unsigned long long* __restrict__ w, uint32_t m,
                                                                unsigned long long* __restrict__ out)
{
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j < m) out[j] = ~w[roots[j]];
}
// one thread per cluster in rank order: the head of a recorded cluster, then the rank takes the place of the root's bin count
__global__ void __launch_bounds__(256) k_pf_cluster_rank(const uint32_t* __restrict__ roots, uint32_t m, uint32_t n_records, const unsigned long long* __restrict__ keys,
                                                         const unsigned long long* __restrict__ w, const unsigned int* __restrict__ cnt, unsigned int* __restrict__ aux,
                                                         PfClusterHead* __restrict__ heads)
{
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= m) return;
    const uint32_t r = roots[j];
    if (j < n_records) { PfClusterHead hd; hd.weight_int = w[r]; hd.key = keys[r] ^ 0x8000ull; hd.bins = aux[r]; hd.members = cnt[r]; heads[j] = hd; }
    aux[r] = j;
}
// one thread per particle: its label, and its place in the sort that gathers the recorded clusters (every other particle sorts behind them)
__global__ void __launch_bounds__(256) k_pf_cluster_labels(const uint32_t* __restrict__ slot_of, uint32_t n, const unsigned int* __restrict__ parent,
                                                           const unsigned int* __restrict__ aux, uint32_t n_records, uint32_t* __restrict__ labels,
                                                           uint32_t* __restrict__ sort_keys, uint32_t* __restrict__ index)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t s = slot_of[i];
    const uint32_t label = s == B2_CLUSTER_NONE ? B2_CLUSTER_NONE : aux[parent[s]];
    if (labels) labels[i] = label;
    sort_keys[i] = label < n_records ? label : n_records;
    index[i] = i;
}
// one thread per member of a recorded cluster: 68 B gathered and 68 B written
__global__ void __launch_bounds__(256) k_pf_cluster_gather(const uint32_t* __restrict__ index, uint32_t total, const b2_transform* __restrict__ poses,
                                                           const b2_particle_attr* __restrict__ attrs, b2_transform* __restrict__ poses_out,
                                                           b2_particle_attr* __restrict__ attrs_out)
{
    const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= total) return;
    const uint32_t i = index[p];
    poses_out[p] = poses[i]; attrs_out[p] = attrs[i];
}
#endif

// ---------------------------------------------------------------------------------------------------------------------
// b2_micp_pose_covariance (SURVEY appendix I): the point-to-plane information of a correction's final correspondences, in the body frame of
// the published pose, and its covariance
// ---------------------------------------------------------------------------------------------------------------------
#define B2_COV_NACC 24                 // per sensor: the 21 entries of J J^T on and above the diagonal (row-major), r^2, |q|^2, pairs
#define B2_COV_BLOCK 256
#define B2_COV_SENSORS 4               // = B2_MAX_SENSORS, the n_pairs of the record
struct MicpCovSensor {
    const float* dpts; const uint8_t* dmask; const float* mpts; const float* mnrm; const uint8_t* mmask;
    b2_transform Tpre;                 // T_snew_sold = Tso * T_onew_oold * Tos, as the ICP loop composes it
    float U[12];                       // ~Tbo_ref * Tbo * Tsb: rotation row-major, then translation (dataset point -> reference body frame)
    float RN[9];                       // R(U) R(Tpre)^T, row-major (model normal -> reference body frame)
    float max_dist;
    uint32_t n, blk0, nblk;            // pairs; blocks [blk0, blk0 + nblk)
    double weight;
};
struct MicpCovLaunch { MicpCovSensor s[B2_COV_SENSORS]; uint32_t n_sensors; double tau, degenerate_variance; };

// one accepted pair: q = U d, n = RN N, J = (n, q x n) in float, the sums in FP64
B2_DEV void micp_cov_add_pair(double* a, const float* U, const float* RN, V3 d, V3 N, float r)
{
    const V3 q = mk3(add(add(add(mul(U[0], d.x), mul(U[1], d.y)), mul(U[2], d.z)), U[9]),
                     add(add(add(mul(U[3], d.x), mul(U[4], d.y)), mul(U[5], d.z)), U[10]),
                     add(add(add(mul(U[6], d.x), mul(U[7], d.y)), mul(U[8], d.z)), U[11]));
    const V3 n = mk3(add(add(mul(RN[0], N.x), mul(RN[1], N.y)), mul(RN[2], N.z)),
                     add(add(mul(RN[3], N.x), mul(RN[4], N.y)), mul(RN[5], N.z)),
                     add(add(mul(RN[6], N.x), mul(RN[7], N.y)), mul(RN[8], N.z)));
    const double J[6] = {(double)n.x, (double)n.y, (double)n.z, (double)sub(mul(q.y, n.z), mul(q.z, n.y)),
                         (double)sub(mul(q.z, n.x), mul(q.x, n.z)), (double)sub(mul(q.x, n.y), mul(q.y, n.x))};
    int e = 0;
    #pragma unroll
    for (int i = 0; i < 6; i++)
        #pragma unroll
        for (int j = i; j < 6; j++) a[e++] += J[i] * J[j];
    a[21] += (double)r * (double)r;
    a[22] += (double)q.x * (double)q.x + (double)q.y * (double)q.y + (double)q.z * (double)q.z;
    a[23] += 1.0;
}

// The record from the per-sensor sums (sums[k * B2_COV_NACC ..]): weighted information, scaling, cyclic Jacobi, pseudo-inverse.  One thread.
// The main loops stay rolled so that the 6x6 arrays live in local memory: unrolled, they would take ~160 registers of the calling kernel.
B2_DEV void micp_cov_finalize(const double* sums, const double* weights, uint32_t n_sensors, double tau, double degenerate_variance, b2_micp_covariance* o)
{
#if B2_ON_DEVICE
    const double qnan = __longlong_as_double(0x7ff8000000000000ll);
#else
    const double qnan = std::nan("");
#endif
    double H[36], R2 = 0.0, Q2 = 0.0, W = 0.0;
    for (int i = 0; i < 36; i++) H[i] = 0.0;
    for (int k = 0; k < B2_COV_SENSORS; k++) o->n_pairs[k] = 0;
    #pragma unroll 1
    for (uint32_t k = 0; k < n_sensors; k++) {
        const double* s = sums + (size_t)k * B2_COV_NACC;
        const double w = weights[k];
        int e = 0;
        #pragma unroll 1
        for (int i = 0; i < 6; i++) for (int j = i; j < 6; j++) H[i * 6 + j] += w * s[e++];
        R2 += w * s[21]; Q2 += w * s[22]; W += w * s[23];
        o->n_pairs[k] = (uint64_t)s[23];
    }
    #pragma unroll 1
    for (int i = 1; i < 6; i++) for (int j = 0; j < i; j++) H[i * 6 + j] = H[j * 6 + i];
    for (int i = 0; i < 36; i++) o->information[i] = H[i];
    o->residual_sq_sum = R2; o->weight_sum = W;
    o->sigma2 = W > 6.0 ? R2 / (W - 6.0) : qnan;
    if (!(W > 0.0)) {                                              // no pairs: nothing is known
        for (int i = 0; i < 36; i++) { o->eigenvectors[i] = 0.0; o->covariance[i] = qnan; }
        for (int i = 0; i < 6; i++) o->eigenvalues[i] = 0.0;
        o->length_scale = 0.0; o->n_degenerate = 6; o->degenerate_mask = 0x3f;
        return;
    }
    double L = sqrt(Q2 / W);
    if (!(L > 0.0)) L = 1.0;
    const double sc[6] = {1.0, 1.0, 1.0, 1.0 / L, 1.0 / L, 1.0 / L};
    double A[36], V[36], total = 0.0;
    #pragma unroll 1
    for (int i = 0; i < 6; i++) for (int j = 0; j < 6; j++) { A[i * 6 + j] = sc[i] * H[i * 6 + j] * sc[j]; V[i * 6 + j] = i == j ? 1.0 : 0.0; }
    for (int i = 0; i < 36; i++) total += A[i] * A[i];
    // cyclic Jacobi: rotation (p, q) zeroes A[p][q] (theta = (a_qq - a_pp) / (2 a_pq), t = tan of the smaller angle); at most 32 sweeps, until the
    // off-diagonal sum of squares is at most 1e-30 of the whole (an off-diagonal entry 1e-15 of the norm)
    #pragma unroll 1
    for (int sweep = 0; sweep < 32; sweep++) {
        double off = 0.0;
        #pragma unroll 1
        for (int p = 0; p < 5; p++) for (int q = p + 1; q < 6; q++) off += A[p * 6 + q] * A[p * 6 + q];
        if (!(off > 1e-30 * total)) break;
        #pragma unroll 1
        for (int p = 0; p < 5; p++) for (int q = p + 1; q < 6; q++) {
            const double apq = A[p * 6 + q];
            if (apq == 0.0) continue;
            const double theta = (A[q * 6 + q] - A[p * 6 + p]) / (2.0 * apq);
            const double t = (theta >= 0.0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
            const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
            for (int k = 0; k < 6; k++) { const double x = A[k * 6 + p], y = A[k * 6 + q]; A[k * 6 + p] = c * x - s * y; A[k * 6 + q] = s * x + c * y; }
            for (int k = 0; k < 6; k++) { const double x = A[p * 6 + k], y = A[q * 6 + k]; A[p * 6 + k] = c * x - s * y; A[q * 6 + k] = s * x + c * y; }
            for (int k = 0; k < 6; k++) { const double x = V[k * 6 + p], y = V[k * 6 + q]; V[k * 6 + p] = c * x - s * y; V[k * 6 + q] = s * x + c * y; }
            A[p * 6 + q] = 0.0; A[q * 6 + p] = 0.0;
        }
    }
    int idx[6] = {0, 1, 2, 3, 4, 5};
    #pragma unroll 1
    for (int a = 0; a < 5; a++) for (int b = a + 1; b < 6; b++) if (A[idx[b] * 7] < A[idx[a] * 7]) { const int t = idx[a]; idx[a] = idx[b]; idx[b] = t; }
    double lam[6], ev[36];
    #pragma unroll 1
    for (int i = 0; i < 6; i++) {
        lam[i] = A[idx[i] * 7];
        int m = 0;
        for (int k = 1; k < 6; k++) if (fabs(V[k * 6 + idx[i]]) > fabs(V[m * 6 + idx[i]])) m = k;
        const double sg = V[m * 6 + idx[i]] < 0.0 ? -1.0 : 1.0;
        for (int k = 0; k < 6; k++) ev[i * 6 + k] = sg * V[k * 6 + idx[i]];
    }
    double Cs[36];
    for (int i = 0; i < 36; i++) Cs[i] = 0.0;
    uint32_t mask = 0, n_deg = 0;
    #pragma unroll 1
    for (int i = 0; i < 6; i++) {
        const bool deg = lam[i] <= tau * lam[5];
        if (deg) { mask |= 1u << i; n_deg++; }
        const double f = deg ? degenerate_variance : o->sigma2 / lam[i];
        #pragma unroll 1
        for (int a = 0; a < 6; a++) for (int b = 0; b < 6; b++) Cs[a * 6 + b] += f * (ev[i * 6 + a] * ev[i * 6 + b]);
    }
    for (int a = 0; a < 6; a++) for (int b = 0; b < 6; b++) o->covariance[a * 6 + b] = sc[a] * Cs[a * 6 + b] * sc[b];
    for (int i = 0; i < 6; i++) o->eigenvalues[i] = lam[i];
    for (int i = 0; i < 36; i++) o->eigenvectors[i] = ev[i];
    o->length_scale = L; o->n_degenerate = n_deg; o->degenerate_mask = mask;
}

#if defined(__CUDACC__)
// One launch over all sensors; blocks [blk0, blk0 + nblk) read sensor k's pairs with k_p2l_reduce's loads and gate.  Block partials go to
// `partials`; the last block to finish sums them per sensor in a fixed order (repeated calls give the same bytes) and writes the record.
__global__ void __launch_bounds__(B2_COV_BLOCK) k_micp_information(const __grid_constant__ MicpCovLaunch L, double* __restrict__ partials,
                                                                   unsigned int* __restrict__ ticket, b2_micp_covariance* __restrict__ out)
{
    constexpr int NW = B2_COV_BLOCK / 32, NG = B2_COV_BLOCK / B2_COV_NACC;
    __shared__ double smem[B2_COV_NACC][NW];
    __shared__ double s_grp[NG][B2_COV_NACC];
    __shared__ double s_sum[B2_COV_SENSORS][B2_COV_NACC];
    __shared__ bool is_last;
    double acc[B2_COV_NACC];
    #pragma unroll
    for (int j = 0; j < B2_COV_NACC; j++) acc[j] = 0.0;
    for (uint32_t k = 0; k < L.n_sensors; k++) {
        const MicpCovSensor& S = L.s[k];
        if (blockIdx.x < S.blk0 || blockIdx.x >= S.blk0 + S.nblk) continue;
        const Tf Tpre = tf_from_pod(S.Tpre);
        const uint32_t stride = S.nblk * B2_COV_BLOCK;
        #pragma unroll 1
        for (uint32_t i = (blockIdx.x - S.blk0) * B2_COV_BLOCK + threadIdx.x; i < S.n; i += stride) {
            const uint8_t dm = S.dmask[i], mm = S.mmask[i];
            const V3 d = mk3(S.dpts[3 * i], S.dpts[3 * i + 1], S.dpts[3 * i + 2]);
            const V3 I = mk3(S.mpts[3 * i], S.mpts[3 * i + 1], S.mpts[3 * i + 2]);
            const V3 N = mk3(S.mnrm[3 * i], S.mnrm[3 * i + 1], S.mnrm[3 * i + 2]);
            V3 D, M;
            if ((dm > 0) && (mm > 0) && p2l_pair(Tpre, d, I, N, S.max_dist, D, M)) micp_cov_add_pair(acc, S.U, S.RN, d, N, v_dot(v_sub(I, D), N));
        }
    }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    #pragma unroll
    for (int j = 0; j < B2_COV_NACC; j++) {
        double v = acc[j];
        #pragma unroll
        for (int off = 16; off > 0; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
        if (lane == 0) smem[j][warp] = v;
    }
    __syncthreads();
    if (threadIdx.x < B2_COV_NACC) {
        double x = 0.0;
        #pragma unroll
        for (int w = 0; w < NW; w++) x += smem[threadIdx.x][w];
        partials[(size_t)blockIdx.x * B2_COV_NACC + threadIdx.x] = x;
        __threadfence();
    }
    __syncthreads();
    if (threadIdx.x == 0) is_last = atomicAdd(ticket, 1u) == gridDim.x - 1;
    __syncthreads();
    if (!is_last) return;
    __threadfence();
    // per sensor: thread (g, i) adds value i of blocks blk0 + g, blk0 + g + NG, ...; then the NG group sums in order
    for (uint32_t k = 0; k < L.n_sensors; k++) {
        const MicpCovSensor& S = L.s[k];
        if (threadIdx.x < NG * B2_COV_NACC) {
            const uint32_t i = threadIdx.x % B2_COV_NACC, g = threadIdx.x / B2_COV_NACC;
            double a = 0.0;
            for (uint32_t b = S.blk0 + g; b < S.blk0 + S.nblk; b += NG) a += __ldcg(partials + (size_t)b * B2_COV_NACC + i);
            s_grp[g][i] = a;
        }
        __syncthreads();
        if (threadIdx.x < B2_COV_NACC) {
            double a = 0.0;
            #pragma unroll
            for (int g = 0; g < NG; g++) a += s_grp[g][threadIdx.x];
            s_sum[k][threadIdx.x] = a;
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        double w[B2_COV_SENSORS];
        for (uint32_t k = 0; k < L.n_sensors; k++) w[k] = L.s[k].weight;
        micp_cov_finalize(&s_sum[0][0], w, L.n_sensors, L.tau, L.degenerate_variance, out);
        *ticket = 0u;
    }
}
#endif

#include "icp_loop.cuh"
