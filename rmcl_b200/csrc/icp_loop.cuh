// icp_loop.cuh -- the inner iterations of MICPLocalizationNode::correctOnce (rmcl_ros/src/nodes/micp_localization.cpp:915-964) for up to
// B2_MAX_SENSORS sensors in ONE kernel (included at the end of kernels.cuh).
//
//   per iteration (reference, per sensor s):  T_bnew_bold = ~Tbo_s * T_onew_oold * Tbo_s                    :926
//                                             Cs_b = sensor.computeCrossStatistics(T_bnew_bold, cp)          :928  (MICPSensor.hpp:158-184)
//                                             Cs_o = Tbo_s * Cs_b;  weighted copy n_meas *= merge_weight     :931-934 (u32 *= double truncates, quirk D3)
//                                             Cmerged_o += Cs_o;  Cmerged_weighted_o += Cs_weighted_o        :936-937
//                                           T_inner = umeyama_transform(Cmerged_weighted_o)                  :952-953
//                                           T_onew_oold = T_onew_oold * T_inner                              :963
//
// Shape: one 512-thread block per SM; the blocks are split among the sensors in proportion to their pair counts.  Every thread
// owns a fixed set of (dataset, model) pairs for the whole kernel -- two in registers, the next ones in shared memory, anything beyond
// streamed from L2 -- so that after the first pass an iteration touches no global memory except the exchange of the block sums.
// Per iteration:  P2L pass (FP32 per-pair math identical to the oracle, FP64 sums) -> reduce-scatter warp reduction -> block sums ->
// grid-wide exchange (64-bit fixed-point atomics, see below; FP64 slots behind a grid sync in the cooperative variant) -> warp 0 of EVERY
// block turns the sums into the per-sensor statistics (15 elements on 15 lanes) and runs the rest of the serial tail redundantly (no
// broadcast hop).  The result leaves through mapped pinned host memory in 16-byte chunks that each carry the sequence number of the call,
// so the host needs no separate completion flag and the kernel no system-wide fence.
#pragma once

#define B2_MAX_SENSORS 4
#define B2_ICP_BLOCK 512
#define B2_ICP_REG_PAIRS 2                     // pairs per thread kept in registers
#define B2_ICP_MAX_GRID 160                    // re-sum: 32 groups x 5 predicated loads

struct IcpSensor {
    const float* dpts; const uint8_t* dmask;                   // dataset (sensor frame)
    const float* mpts; const float* mnrm; const uint8_t* mmask; // model buffers written by find (sensor frame)
    const float* zc_ranges;                                     // != nullptr: the scan is unpacked HERE (MICPSphericalSensorCPU.cpp:181-233) from ...
    const unsigned int* zc_flag;                                //   != nullptr: ... the handle's device buffer, which a copy engine fills from the caller's pinned
                                                                //   buffer while find runs; the copy is complete when *zc_flag == zc_seq (written by a second copy
                                                                //   behind it on the same stream).  nullptr: ... the caller's pinned host buffer itself, over PCIe
    const float* zc_dirs; const float* zc_origs;                // results mirrored into the handle's buffers:
    float* dpts_out; uint8_t* dmask_out; float* ranges_out;
    double merge_weight;                                        // MICPSensor.hpp:103, applied at micp_localization.cpp:934
    b2_transform Tos, Tso;                                      // Tos = Tbo * Tsb (sensor -> odom), Tso = ~Tos, composed once on the host
    float Ros[9];                                               // rotation matrix of Tos, row-major
    float max_dist, range_min, range_max;
    uint32_t n, blk0, nblk, zc_n_origs, smem_u;                 // pairs; blocks [blk0, blk0+nblk); pairs per thread kept in shared memory
    uint32_t zc_seq;
    const uint32_t* tile_cost; uint16_t* tile_perm;             // != nullptr: the idle warps of this sensor's first block turn the tile durations of the find
    uint32_t n_tiles;                                           //   kernel into the tile order of the NEXT find (kernels.cuh: tile schedule)
    float max_dist_min;                                         // chain steps only: adaptive_max_dist_min (Correspondences.hpp:23); max_dist is then params.max_dist
};
// Device state of a chain of corrections (b2_micp_correct): what step k+1 reads from step k, so that the host is not involved between them.
struct alignas(16) IcpChainState {
    IcpState find[B2_MAX_SENSORS];     // Tom (the pose of the next find, written by block 0 of each loop) and Tbo of sensor k; the find kernels' `icp` argument
    double cp;                         // convergence_progress_ after the last completed step (micp_localization.cpp:988-1007)
    uint32_t valid, total;             // stats.valid_measurements / total_measurements over all sensors (:866-871): mask ones, dataset sizes
    uint32_t done, pad_;               // steps completed
};
struct IcpLaunch {
    IcpSensor s[B2_MAX_SENSORS];
    b2_transform Tom;
    uint32_t n_sensors, iterations, seq, smem_u_max;
    IcpChainState* chain;              // != nullptr: one step of a chain -- Tom and the progress come from here and block 0 writes the step's outcome back
    b2_micp_step* step_out;            //   the record of this step
    uint32_t adaptive, pad_;           //   adaptive_max_dist_ (micp_localization.hpp:157)
};
struct IcpResult { b2_transform Tom_new, T_onew_oold; b2_cross_stats Cmerged_o; };                  // 128 bytes
static_assert(sizeof(IcpResult) == 128, "IcpResult must be 128 bytes");
#define B2_ICP_RESULT_CHUNKS 11                // 32 payload words, 3 per 16-byte chunk + the sequence number

// make PROFILE=1: SM-clock stamps inside the serial tail (scripts/exp_step.py prints them); compiled out of the product build
#if defined(B2_ICP_PROFILE) && defined(__CUDA_ARCH__)
#define B2_TAIL_STAMP(st, i) do { if (st) (st)[i] = clock64(); } while (0)
#else
#define B2_TAIL_STAMP(st, i) do { } while (0)
#endif

// ---------------------------------------------------------------------------------------------------------------------
// serial tail of one inner iteration (one thread; host+device so that tests/emul runs the same code)
// ---------------------------------------------------------------------------------------------------------------------
B2_DEV double b2_rcp_u32(uint32_t n)
{
    const double d = (double)n;
    double x = (double)b2_rcp_approx((float)n);
    x = x * (2.0 - d * x); x = x * (2.0 - d * x);              // two Newton steps: full double precision without the software division
    return x;
}

// sums (n, S_d, S_m, S_md^T in FP64) -> CrossStatistics in FP32 (like acc_finalize, without the FP64 division), one element at a time so that
// the device can spread the elements over the lanes of a warp: element 0..2 dataset mean, 3..5 model mean, 6..14 covariance [c*3+r]
B2_DEV float icp_finalize_elem(double vi, double vm /* S_m[r] */, double vd /* S_d[c] */, double inv, int i)
{
    if (i < 6) return (float)(vi * inv);
    return (float)(vi * inv - (vm * inv) * (vd * inv));
}
// Tos * stats in rotation-matrix form (means as points, C -> R C R^T), explicit FMAs, one element from what it reads: rows r and j of R
// (icp_odom_rows), t[r], the point p (dm or mm) and C.  Element i < 6: (R p + t)[r];  i >= 6: o.C[j*3 + r] = sum_l (R C)[r][l] * R[j][l]
B2_DEV void icp_odom_rows(int i, int& r, int& j)
{
    if (i < 6) { r = i < 3 ? i : i - 3; j = 0; }
    else { j = (i - 6) / 3; r = (i - 6) - 3 * j; }
}
B2_DEV float icp_to_odom_rows(const float* Rr, const float* Rj, float tr, const float* p, const float* C, int i)
{
    if (i < 6) return fma_rn(Rr[2], p[2], fma_rn(Rr[1], p[1], fma_rn(Rr[0], p[0], tr)));
    float RC[3];
    #pragma unroll
    for (int l = 0; l < 3; l++) RC[l] = fma_rn(Rr[2], C[l * 3 + 2], fma_rn(Rr[1], C[l * 3 + 1], mul(Rr[0], C[l * 3 + 0])));
    return fma_rn(RC[2], Rj[2], fma_rn(RC[1], Rj[1], mul(RC[0], Rj[0])));
}
// the same over a whole statistics record s = {dm, mm, C} as 15 floats, same element numbering
B2_DEV float icp_to_odom_elem(const float* R, const float* t, const float* s, int i)
{
    int r, j;
    icp_odom_rows(i, r, j);
    return icp_to_odom_rows(R + r * 3, R + j * 3, t[r], s + (i < 3 ? 0 : 3), s + 6, i);
}
// per-sensor statistics in the odom frame from the reduced sums: serial form (host emulation; k_icp_loop spreads the elements over lanes)
B2_DEV uint32_t icp_sensor_stats(const IcpSensor& S, const double* v, float* o /* 16 */)
{
    const uint32_t n = (uint32_t)(v[B2_NACC] + 0.5);
    const double inv = n ? b2_rcp_u32(n) : 0.0;
    float e[15];
    for (int i = 0; i < 15; i++) e[i] = icp_finalize_elem(v[i], i >= 6 ? v[3 + (i - 6) % 3] : 0.0, i >= 6 ? v[(i - 6) / 3] : 0.0, inv, i);
    const float t[3] = {S.Tos.t.x, S.Tos.t.y, S.Tos.t.z};
    for (int i = 0; i < 15; i++) o[i] = icp_to_odom_elem(S.Ros, t, e, i);
    o[15] = 0.f;
    return n;
}

// One Newton step of the polar iteration, X <- a X + b X^-T with X^-T = Cf / det; Frobenius-scaled in the first three steps.  Returns
// |X_k+1 - X_k|^2; `ok` drops when det <= 1e-12 (reflection, singular, NaN).
B2_DEV float icp_polar_step(float* X, bool scaled, bool& ok)
{
    float Cf[9];
    Cf[0] = fma_rn(X[4], X[8], -mul(X[5], X[7])); Cf[1] = fma_rn(X[5], X[6], -mul(X[3], X[8])); Cf[2] = fma_rn(X[3], X[7], -mul(X[4], X[6]));
    Cf[3] = fma_rn(X[2], X[7], -mul(X[1], X[8])); Cf[4] = fma_rn(X[0], X[8], -mul(X[2], X[6])); Cf[5] = fma_rn(X[1], X[6], -mul(X[0], X[7]));
    Cf[6] = fma_rn(X[1], X[5], -mul(X[2], X[4])); Cf[7] = fma_rn(X[2], X[3], -mul(X[0], X[5])); Cf[8] = fma_rn(X[0], X[4], -mul(X[1], X[3]));
    const float det = fma_rn(X[2], Cf[2], fma_rn(X[1], Cf[1], mul(X[0], Cf[0])));
    ok = ok && det > 1e-12f;
    float a, b;
    if (scaled) {
        // g = (|X^-1|_F / |X|_F)^(1/2) with X^-1 = Cf^T / det:  a = g / 2,  b = 1 / (2 g det).  Three short FMA chains per norm; the
        // reciprocal roots of det and |X|^2 do not wait for the cofactor norm, so only two special-function results are chained.
        const float nx = add(add(fma_rn(X[2], X[2], fma_rn(X[1], X[1], mul(X[0], X[0]))), fma_rn(X[5], X[5], fma_rn(X[4], X[4], mul(X[3], X[3])))),
                             fma_rn(X[8], X[8], fma_rn(X[7], X[7], mul(X[6], X[6]))));
        const float nc = add(add(fma_rn(Cf[2], Cf[2], fma_rn(Cf[1], Cf[1], mul(Cf[0], Cf[0]))), fma_rn(Cf[5], Cf[5], fma_rn(Cf[4], Cf[4], mul(Cf[3], Cf[3])))),
                             fma_rn(Cf[8], Cf[8], fma_rn(Cf[7], Cf[7], mul(Cf[6], Cf[6]))));
        const float rd = b2_rsqrt_approx(det), rx = b2_rsqrt_approx(nx);          // det^-1/2, |X|_F^-1
        const float ratio = mul(mul(nc, b2_rsqrt_approx(nc)), rx);                 // |Cf|_F / |X|_F
        const float rr = b2_rsqrt_approx(ratio);
        b = mul(mul(0.5f, rr), rd);                                                // 1 / (2 g det),  g = ratio^1/2 det^-1/2
        a = mul(mul(ratio, rr), mul(0.5f, rd));
    } else { a = 0.5f; b = mul(0.5f, b2_rcp_approx(det)); }
    float d2[3] = {0.f, 0.f, 0.f};
    #pragma unroll
    for (int i = 0; i < 9; i++) { const float y = fma_rn(b, Cf[i], mul(a, X[i])); const float d = sub(y, X[i]); d2[i / 3] = fma_rn(d, d, d2[i / 3]); X[i] = y; }
    return add(add(d2[0], d2[1]), d2[2]);
}

// Orthogonal polar factor of C (det > 0) by the Frobenius-scaled Newton iteration, everything in registers: FP32 iterations, one FP64
// polishing step whose 1/det is a Newton reciprocal around 1.  Returns false for reflections / singular / non-converged input (the caller
// then takes the Jacobi SVD).  Same mathematics as polar_newton3, minus the call, the stack frame and the software divisions.
// Converged after step k (k >= 2): |X_k+1 - X_k| < 3e-4 -- the step after it is at FP32 rounding level, and the FP64 step squares what is
// left.  The cross-covariance of an ICP scan converges after three or four steps, so those four run as one straight chain: the fourth is
// computed before the test of the third (and dropped if the third converged), the rest of the 40 only if the fourth has not.
B2_DEV bool icp_polar(const float* C /* column-major, like CStats::C */, float* Rf /* row-major */, long long* st = nullptr)
{
    float X[9];
    #pragma unroll
    for (int r = 0; r < 3; r++)
        #pragma unroll
        for (int c = 0; c < 3; c++) X[r * 3 + c] = C[c * 3 + r];
    float fro = 0.0f;
    #pragma unroll
    for (int i = 0; i < 9; i++) fro = fma_rn(X[i], X[i], fro);
    if (!(fro > 1e-30f)) return false;
    const float inv_n = b2_rsqrt_approx(fro);
    #pragma unroll
    for (int i = 0; i < 9; i++) X[i] = mul(X[i], inv_n);
    bool ok = true, ok3 = true;
    icp_polar_step(X, true, ok);
    icp_polar_step(X, true, ok);
    const float s2 = icp_polar_step(X, true, ok);
    float X3[9];
    #pragma unroll
    for (int i = 0; i < 9; i++) X3[i] = X[i];
    const float s3 = icp_polar_step(X3, false, ok3);
    if (!ok) return false;
    bool conv = s2 < 1e-7f;
    if (!conv) {
        if (!ok3) return false;
        #pragma unroll
        for (int i = 0; i < 9; i++) X[i] = X3[i];
        conv = s3 < 1e-7f;
        for (int it = 4; it < 40 && !conv; it++) {
            const float s = icp_polar_step(X, false, ok);
            if (!ok) return false;
            conv = s < 1e-7f;
        }
        if (!conv) return false;
    }
    B2_TAIL_STAMP(st, 3);
    double Y[9];
    #pragma unroll
    for (int i = 0; i < 9; i++) Y[i] = (double)X[i];
    double Cf[9];
    Cf[0] = Y[4] * Y[8] - Y[5] * Y[7]; Cf[1] = Y[5] * Y[6] - Y[3] * Y[8]; Cf[2] = Y[3] * Y[7] - Y[4] * Y[6];
    Cf[3] = Y[2] * Y[7] - Y[1] * Y[8]; Cf[4] = Y[0] * Y[8] - Y[2] * Y[6]; Cf[5] = Y[1] * Y[6] - Y[0] * Y[7];
    Cf[6] = Y[1] * Y[5] - Y[2] * Y[4]; Cf[7] = Y[2] * Y[3] - Y[0] * Y[5]; Cf[8] = Y[0] * Y[4] - Y[1] * Y[3];
    const double det = Y[0] * Cf[0] + Y[1] * Cf[1] + Y[2] * Cf[2];
    const double e = 1.0 - det;                                   // |e| ~ 1e-6 after the FP32 iterations: 1/det = 1 + e + e^2 + O(e^3)
    const double b = 0.5 * (1.0 + e + e * e);
    #pragma unroll
    for (int i = 0; i < 9; i++) Rf[i] = (float)(0.5 * Y[i] + b * Cf[i]);
    return true;
}

// 1/sqrt(x) to FP32 rounding level: special-function seed + one Newton step (no IEEE division / square root on the loop's critical path)
B2_DEV float icp_rsqrt(float x)
{
    const float r = b2_rsqrt_approx(x);
    return mul(r, fma_rn(mul(-0.5f, x), mul(r, r), 1.5f));
}
// rotation matrix (row-major, orthogonal to double precision) -> unit quaternion; same branches as the tail of umeyama_dev
B2_DEV Q4 icp_mat_to_quat(const float* R)
{
    float q[4];
    const float tr = R[0] + R[4] + R[8];
    if (tr > 0.0f) {
        const float s = tr + 1.0f, h = mul(0.5f, icp_rsqrt(s));                            // h = 1 / (2 sqrt(s))
        q[3] = mul(s, h); q[0] = mul(R[7] - R[5], h); q[1] = mul(R[2] - R[6], h); q[2] = mul(R[3] - R[1], h);
    } else if (R[0] > R[4] && R[0] > R[8]) {
        const float s = 1.0f + R[0] - R[4] - R[8], h = mul(0.5f, icp_rsqrt(s));
        q[3] = mul(R[7] - R[5], h); q[0] = mul(s, h); q[1] = mul(R[1] + R[3], h); q[2] = mul(R[2] + R[6], h);
    } else if (R[4] > R[8]) {
        const float s = 1.0f + R[4] - R[0] - R[8], h = mul(0.5f, icp_rsqrt(s));
        q[3] = mul(R[2] - R[6], h); q[0] = mul(R[1] + R[3], h); q[1] = mul(s, h); q[2] = mul(R[5] + R[7], h);
    } else {
        const float s = 1.0f + R[8] - R[0] - R[4], h = mul(0.5f, icp_rsqrt(s));
        q[3] = mul(R[3] - R[1], h); q[0] = mul(R[2] + R[6], h); q[1] = mul(R[5] + R[7], h); q[2] = mul(s, h);
    }
    const float rn = icp_rsqrt(add(add(mul(q[0], q[0]), mul(q[1], q[1])), add(mul(q[2], q[2]), mul(q[3], q[3]))));
    Q4 qq; qq.x = mul(q[0], rn); qq.y = mul(q[1], rn); qq.z = mul(q[2], rn); qq.w = mul(q[3], rn);
    return qq;
}

// rm::umeyama_transform on the critical path of the loop: polar fast path inline, SVD fallback out of line
B2_DEV Tf icp_umeyama(const CStats& s, long long* st = nullptr)
{
    if (s.n == 0) return tf_identity();
    float Rf[9];
    if (!icp_polar(s.C, Rf, st)) return umeyama_dev(s);
    B2_TAIL_STAMP(st, 4);
    Tf out;
    out.R = icp_mat_to_quat(Rf);
    out.t = v_sub(s.mm, q_rot(out.R, s.dm));
    B2_TAIL_STAMP(st, 5);
    return out;
}

// Sensor k's statistics in the odom frame (o = Tbo * (Tsb * stats_s), :931) into the merged statistics, in sensor order; merged / merged_w
// start as cs_identity().  One sensor: merging with the empty identity is an exact no-op, so the sensor's statistics are taken as they are.
B2_DEV void icp_merge_sensor(const IcpLaunch& L, uint32_t k, const CStats& o, CStats& merged, CStats& merged_w)
{
    CStats w = o;
    if (L.s[k].merge_weight != 1.0) w.n = (uint32_t)((double)o.n * L.s[k].merge_weight);              // :933-934 (u32 *= double; exact no-op for weight 1)
    if (L.n_sensors == 1) { merged = o; merged_w = w; }
    else { merged = cs_merge(merged, o); merged_w = cs_merge(merged_w, w); }                          // :936-937
}

// One inner iteration after the merged statistics are known.  T_onew_oold is updated in place, Tpre_out[s] receives the pre-transform of sensor s
// for the NEXT pass (T_snew_sold = Tso * T_onew_oold * Tos: MICPSensor.hpp:178 with the constant frame chain pre-composed) for the sensors
// [k0, k1) -- on the device lane k of the warp computes sensor k --, `res` is filled after the last iteration (micp_localization.cpp:972-984).
B2_DEV void icp_tail_rest(const IcpLaunch& L, const b2_transform& Tom_pod, const CStats& merged, const CStats& merged_w, Tf& T_onew_oold, Tf* Tpre_out, uint32_t k0, uint32_t k1,
                          bool last, IcpResult* res, long long* st = nullptr)
{
    B2_TAIL_STAMP(st, 2);
    const Tf T_inner = icp_umeyama(merged_w, st);                                                     // :952-953
    T_onew_oold = tf_mul(T_onew_oold, T_inner);                                                       // :963
    B2_TAIL_STAMP(st, 6);
    for (uint32_t k = k0; k < k1; k++) Tpre_out[k] = tf_mul(tf_mul(tf_from_pod(L.s[k].Tso), T_onew_oold), tf_from_pod(L.s[k].Tos));
    B2_TAIL_STAMP(st, 7);
    if (last && res) {
        const Tf Tom = tf_from_pod(Tom_pod);
        Tf Tn = tf_mul(Tom, T_onew_oold);                                                             // :972
        if (merged.n > 0) Tn.R = q_normalize(Tn.R); else Tn = Tom;                                    // :974-984
        tf_store(&res->Tom_new, Tn); tf_store(&res->T_onew_oold, T_onew_oold); cs_store(&res->Cmerged_o, merged);
    }
}
// the whole serial tail from the reduced sums (host emulation: tests/emul)
B2_DEV void icp_tail(const IcpLaunch& L, const double (*sums)[B2_NACC + 1], Tf& T_onew_oold, Tf* Tpre_out, bool last, IcpResult* res)
{
    CStats merged = cs_identity(), merged_w = cs_identity();
    for (uint32_t k = 0; k < L.n_sensors; k++) {
        float odo[16];
        CStats o; o.n = icp_sensor_stats(L.s[k], sums[k], odo);
        o.dm = mk3(odo[0], odo[1], odo[2]); o.mm = mk3(odo[3], odo[4], odo[5]);
        for (int q = 0; q < 9; q++) o.C[q] = odo[6 + q];
        icp_merge_sensor(L, k, o, merged, merged_w);
    }
    icp_tail_rest(L, L.Tom, merged, merged_w, T_onew_oold, Tpre_out, 0, L.n_sensors, last, res);
}

// ---------------------------------------------------------------------------------------------------------------------
// Between two corrections (host+device so that tests/emul runs the same code)
// ---------------------------------------------------------------------------------------------------------------------
// params.max_dist interpolated towards adaptive_max_dist_min by the progress (CorrespondencesCPU.cpp:21-23): float * double + float * double
// in double, rounded to float -- the host's expression (api.cu: adaptive_max_dist), so that a chain step gates exactly like a host-fed call
B2_DEV float icp_adaptive_max_dist(float max_dist, float max_dist_min, double cp)
{
    return (float)((double)max_dist * (1.0 - cp) + (double)max_dist_min * cp);
}
// convergence_progress_ after one correctOnce (micp_localization.cpp:988-1007), with the reference's types statement by statement.  T_onew_map =
// Tom * T_onew_oold before the normalisation of :983 (:972); valid = stats.valid_measurements (:870).  Quirk: trans_force is the norm of the
// ABSOLUTE translation of T_odom_map, so the progress is about 0 unless the odom origin lies within ~0.3 m of the map origin (SURVEY.md D12).
B2_DEV double micp_progress(const b2_transform& Tom, const b2_transform& T_onew_oold, uint32_t n_meas, uint32_t valid, bool adaptive)
{
    if (n_meas == 0 || !adaptive) return 0.0;                                                        // :988-991
    const Tf T = tf_mul(tf_from_pod(Tom), tf_from_pod(T_onew_oold));                                 // :972
    const float trans_force = v_l2norm(T.t);                                                         // :994
    const float trans_progress = (float)(1.0 / exp(10.0 * (double)trans_force));                     // :995
    const float qscalar = add(add(add(mul(T.R.x, 0.0f), mul(T.R.y, 0.0f)), mul(T.R.z, 0.0f)), mul(T.R.w, 1.0f));   // :997-998, R.dot(Identity)
    const float rot_progress = mul(qscalar, qscalar);                                                // :999
    const double match_ratio = (double)n_meas / (double)valid;                                       // :1001
    const float adaption_rate = (float)((double)mul(trans_progress, rot_progress) * match_ratio);   // :1002
    return (double)adaption_rate;                                                                    // :1006
}

#if defined(__CUDACC__)
// ---------------------------------------------------------------------------------------------------------------------
// Grid-wide exchange of the block partial sums without a barrier object: every block publishes its 16 FP64 partials as 16-byte slots
// {low word | tag << 32, high word | tag << 32}; every block then reads ALL slots and simply re-reads the ones whose tag is not yet this
// iteration's.  Each 8-byte half validates itself (single-copy atomic, relaxed), so no fence, no arrival counter and no second round trip:
// one store, one (repeated) load.  Tags grow monotonically per handle across launches and iterations; two slot buffers alternate by
// iteration parity -- a block can publish iteration i+2 only after it has read every block's i+1, i.e. after all of them finished reading i.
// Needs all blocks co-resident: one block per SM, and the host never lets two such kernels overlap on a device (api.cu: per-device ordering
// of the loop launches); blocks of ordinary kernels only delay residency.  A thread that waits longer than ~2 s raises the abort word: a
// scheduling surprise ends in a re-run through the cooperative launch, never in a hung GPU.
// ---------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void slot_store(ulonglong2* p, double x, unsigned int tag)
{
    const unsigned long long u = (unsigned long long)__double_as_longlong(x), t = (unsigned long long)tag << 32;
    asm volatile("st.relaxed.gpu.global.v2.u64 [%0], {%1, %2};" ::"l"(p), "l"((u & 0xffffffffull) | t), "l"((u >> 32) | t) : "memory");
}
__device__ __forceinline__ bool slot_load(const ulonglong2* p, unsigned int tag, double& x)
{
    unsigned long long a, b;
    asm volatile("ld.relaxed.gpu.global.v2.u64 {%0, %1}, [%2];" : "=l"(a), "=l"(b) : "l"(p) : "memory");
    x = __longlong_as_double((long long)((a & 0xffffffffull) | (b << 32)));
    return (unsigned int)(a >> 32) == tag && (unsigned int)(b >> 32) == tag;
}

// reduce-scatter warp reduction: afterwards smem[warp * 16 + value] holds each warp's total of the 16 values (15 = count; warp-major: the
// 16 lanes that read one warp's values hit 16 different banks); ends with a block barrier
template <int BLOCK>
__device__ __forceinline__ void block_reduce_to_smem(P2LAcc& a, double* smem)
{
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    static_assert(BLOCK % 32 == 0, "whole warps");
    double v[16];
    #pragma unroll
    for (int i = 0; i < B2_NACC; i++) v[i] = a.v[i];
    v[15] = (double)a.n;                                           // counts <= 2^32 are exact in FP64
    rs_step<8>(v, 16, (lane & 16) != 0);
    rs_step<4>(v, 8, (lane & 8) != 0);
    rs_step<2>(v, 4, (lane & 4) != 0);
    rs_step<1>(v, 2, (lane & 2) != 0);
    const double tot = v[0] + __shfl_xor_sync(0xffffffffu, v[0], 1);
    const int vidx = ((lane >> 4) & 1) * 8 + ((lane >> 3) & 1) * 4 + ((lane >> 2) & 1) * 2 + ((lane >> 1) & 1);
    if ((lane & 1) == 0) smem[warp * 16 + vidx] = tot;
    __syncthreads();
}

// ---------------------------------------------------------------------------------------------------------------------
// The default exchange: 64-bit integer atomics.  Every sum is published as two fixed-point limbs (integer part, 40 fractional bits), each
// added with ONE fire-and-forget `red` to a grid-wide accumulator word that lives in its own 128-byte line:
//     word += (limb << 8) + 1
// The low 8 bits count arrivals (fewer than 256 blocks per sensor), the upper 56 bits carry the sum modulo 2^56.  The accumulators are
// never reset: a reader knows the word's value before this round (`prev`), waits until the arrival count has advanced by the number of
// contributing blocks and takes the difference.  No flag, no fence, no bulk read: one atomic out, one 8-byte load back per lane, and integer
// addition makes the result independent of the arrival order (bit-reproducible).  Two accumulator sets alternate by iteration parity (a block
// can contribute to round i+2 only after it has read round i+1 complete, i.e. after every block finished reading round i); block 0 leaves
// the final words in `base` for the next launch.  Doubles with |x| >= 4096 convert without loss, smaller ones to 2^-40; a block partial
// beyond +-2^46 (or non-finite) raises abort code 2 and the call runs again through the cooperative FP64 variant below.
// ---------------------------------------------------------------------------------------------------------------------
static_assert(B2_ICP_MAX_GRID < 256, "the arrival count of an accumulator word has 8 bits");
#define B2_ICP_ACC_STRIDE 16                   // u64 words per accumulator (one 128-byte line each)
#define B2_ICP_ACC_WORDS (2 * B2_MAX_SENSORS * 32 * B2_ICP_ACC_STRIDE)      // [parity][sensor][32 limbs] accumulators ...
#define B2_ICP_BASE_WORDS (2 * B2_MAX_SENSORS * 32)                          // ... followed by the dense `base` copy
#define B2_ICP_SLOT_WORDS (2 * 2 * B2_ICP_MAX_GRID * (B2_NACC + 1))          // ... followed by the FP64 slots of the cooperative variant (ulonglong2 each = 2 words)
__device__ __forceinline__ void acc_red(unsigned long long* p, unsigned long long v) { asm volatile("red.relaxed.gpu.global.add.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory"); }
__device__ __forceinline__ unsigned long long acc_ld(const unsigned long long* p)
{
    unsigned long long v; asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory"); return v;
}

// The tile order of the next find (kernels.cuh: tile schedule) computed by warps 1..15 of one block while warp 0 is busy with the exchange and
// the serial tail: tiles grouped into 16 duration classes relative to the slowest one, slowest class first, raster order inside a class
// (only the slow tail of the distribution has to start early; the bulk may stay where it is: scripts/exp_find_sched*.py).  The work is
// split over the idle windows of the first THREE iterations so that none outlasts its window: (0) durations -> shared memory, maximum;
// (1) per-(class, warp) counts, prefix sums; (2) scatter.  No atomics on hot counters (most tiles share two or three classes): the lanes of a
// warp that hold the same class are found with match.any and their lowest lane updates the warp's counter.  `t` = 0..479; the group
// synchronises on named barrier 1, so the block's own barrier 0 is untouched.
#define B2_PERM_GROUP (B2_ICP_BLOCK - 32)
#define B2_PERM_WARPS (B2_PERM_GROUP / 32)
#define B2_PERM_PT 24                                               // tiles per thread
#define B2_PERM_MAX_TILES (B2_PERM_PT * B2_PERM_GROUP)              // 11 520 tiles = 368 640 rays; s_cost takes 2 bytes per tile of dynamic shared memory
__device__ __forceinline__ void perm_group_sync() { asm volatile("bar.sync 1, %0;" ::"n"(B2_PERM_GROUP) : "memory"); }
__device__ __forceinline__ uint32_t perm_class(uint32_t v16, float scale) { return min(15u, (uint32_t)((float)v16 * scale)); }
__device__ __forceinline__ void tile_perm_load(const uint32_t* __restrict__ cost, uint32_t n_tiles, uint16_t* s_cost, uint32_t* s_bin /* 1 + 16 * 15 */, uint32_t t)
{
    const uint32_t lane = t & 31u, w = t >> 5, iters = (n_tiles + B2_PERM_GROUP - 1) / B2_PERM_GROUP;
    uint32_t* s_off = s_bin + 1;                                   // [(15 - class) * 15 + warp]: slowest class first, then by warp
    if (t == 0) s_bin[0] = 0u;
    if (lane < 16u) s_off[(15u - lane) * B2_PERM_WARPS + w] = 0u;
    perm_group_sync();
    uint32_t m = 0;
    #pragma unroll 8
    for (uint32_t k = 0; k < iters; k++) {                         // one coalesced pass over the durations (SM cycles / 64, 16 bits)
        const uint32_t i = t + k * B2_PERM_GROUP;
        if (i < n_tiles) { const uint32_t v = min(65535u, __ldcg(cost + i) >> 6); s_cost[i] = (uint16_t)v; m = max(m, v); }
    }
    #pragma unroll
    for (int off = 16; off; off >>= 1) m = max(m, __shfl_xor_sync(0xffffffffu, m, off));
    if (lane == 0) atomicMax(&s_bin[0], m);
}
__device__ __forceinline__ void tile_perm_count(uint32_t n_tiles, const uint16_t* s_cost, uint32_t* s_bin, uint32_t t)
{
    const uint32_t lane = t & 31u, w = t >> 5, iters = (n_tiles + B2_PERM_GROUP - 1) / B2_PERM_GROUP;
    uint32_t* s_off = s_bin + 1;
    const float scale = 16.0f / ((float)s_bin[0] + 1.0f);
    #pragma unroll 4
    for (uint32_t k = 0; k < iters; k++) {                         // counts per (class, warp): one shared-memory add per class present in the warp
        const uint32_t i = t + k * B2_PERM_GROUP;
        const uint32_t cls = i < n_tiles ? perm_class(s_cost[i], scale) : 16u;
        const uint32_t grp = __match_any_sync(0xffffffffu, cls);
        if (cls < 16u && lane == (uint32_t)__ffs((int)grp) - 1u) atomicAdd(&s_off[(15u - cls) * B2_PERM_WARPS + w], (uint32_t)__popc(grp));
    }
    perm_group_sync();
    if (w == 0) {                                                  // exclusive prefix over the 240 counts: 8 per lane, then across the lanes
        constexpr uint32_t PER = (16u * B2_PERM_WARPS + 31u) / 32u;
        uint32_t sum = 0;
        for (uint32_t j = 0; j < PER; j++) { const uint32_t e = lane * PER + j; if (e < 16u * B2_PERM_WARPS) sum += s_off[e]; }
        uint32_t incl = sum;
        for (uint32_t off = 1; off < 32u; off <<= 1) { const uint32_t v = __shfl_up_sync(0xffffffffu, incl, off); if (lane >= off) incl += v; }
        uint32_t run = incl - sum;
        for (uint32_t j = 0; j < PER; j++) { const uint32_t e = lane * PER + j; if (e < 16u * B2_PERM_WARPS) { const uint32_t cc = s_off[e]; s_off[e] = run; run += cc; } }
    }
}
__device__ __forceinline__ void tile_perm_scatter(uint32_t n_tiles, const uint16_t* s_cost, uint32_t* s_bin, uint16_t* __restrict__ perm, uint32_t t)
{
    const uint32_t lane = t & 31u, w = t >> 5, iters = (n_tiles + B2_PERM_GROUP - 1) / B2_PERM_GROUP;
    uint32_t* s_off = s_bin + 1;                                   // [class, warp] = next free position of the class for this warp
    const float scale = 16.0f / ((float)s_bin[0] + 1.0f);
    #pragma unroll 4
    for (uint32_t k = 0; k < iters; k++) {
        const uint32_t i = t + k * B2_PERM_GROUP;
        const uint32_t cls = i < n_tiles ? perm_class(s_cost[i], scale) : 16u;
        const uint32_t grp = __match_any_sync(0xffffffffu, cls);
        const uint32_t lead = (uint32_t)__ffs((int)grp) - 1u;
        uint32_t base = 0;
        if (cls < 16u && lane == lead) base = atomicAdd(&s_off[(15u - cls) * B2_PERM_WARPS + w], (uint32_t)__popc(grp));      // the group's block of positions
        base = __shfl_sync(0xffffffffu, base, lead);
        if (cls < 16u) perm[base + (uint32_t)__popc(grp & ((1u << lane) - 1u))] = (uint16_t)i;
    }
}

// The kernel.  COOP: cooperative launch + cg grid sync in front of the slot reads (fallback when co-residency cannot be guaranteed);
// otherwise an ordinary launch, normally with programmatic stream serialization behind the last find kernel.
template <bool COOP>
__global__ void __launch_bounds__(B2_ICP_BLOCK) k_icp_loop(const __grid_constant__ IcpLaunch L, unsigned long long* __restrict__ xbuf, IcpResult* __restrict__ res_dev,
                                                          uint4* host_out, unsigned int tag_base, unsigned int* bar_abort, unsigned long long* __restrict__ dbg)
{
    namespace cg = cooperative_groups;
    extern __shared__ float s_pairs[];                             // [smem_u][9][B2_ICP_BLOCK]
    __shared__ double smem[16 * (B2_ICP_BLOCK / 32)];
    __shared__ double s_part[B2_MAX_SENSORS][B2_ICP_BLOCK / 32][B2_NACC + 1];
    __shared__ float s_Rt[B2_MAX_SENSORS][12];                     // Ros (9) + translation of Tos (3): lane-indexed reads in the tail
    __shared__ unsigned long long s_prev[2][B2_MAX_SENSORS][32];   // accumulator words before the current round, per parity
    __shared__ uint32_t s_bin[1 + 16 * 15];                        // tile schedule of the next find (first block of each sensor)
    __shared__ Tf s_Tpre[B2_MAX_SENSORS];
    __shared__ b2_transform s_Tom;                                 // Tom of this correctOnce (micp_localization.cpp:860)
    __shared__ IcpResult s_res;
    const long long k0 = clock64();
    const unsigned long long g0 = globaltimer_ns();
    const uint32_t tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5;
    // a chain step behind a step that gave up (abort word still set) does nothing: the host re-runs the chain from the first step without a record
    if (L.chain && __syncthreads_or(tid == 0u && *reinterpret_cast<volatile unsigned int*>(bar_abort) != 0u)) return;
    uint32_t si = 0;
    for (uint32_t k = 1; k < L.n_sensors; k++) if (blockIdx.x >= L.s[k].blk0) si = k;
    const IcpSensor& S = L.s[si];
    const uint32_t stride = S.nblk * B2_ICP_BLOCK, lid = (blockIdx.x - S.blk0) * B2_ICP_BLOCK + tid, n = S.n, smem_u = S.smem_u;
    const uint32_t n_cached = B2_ICP_REG_PAIRS + smem_u;           // pairs per thread that never touch global memory again
    if (tid < L.n_sensors) {
        // pre-transform of the first pass: T_onew_oold = I  ->  Tso * I * Tos with the same individually rounded ops as later iterations
        s_Tpre[tid] = tf_mul(tf_mul(tf_from_pod(L.s[tid].Tso), tf_identity()), tf_from_pod(L.s[tid].Tos));
        if (tid == 0) s_Tom = L.chain ? L.chain->find[0].Tom : L.Tom;
    }
    if (tid >= 32u && tid < 32u + 12u * L.n_sensors) {
        const uint32_t k = (tid - 32u) / 12u, e = (tid - 32u) - 12u * k;
        s_Rt[k][e] = e < 9u ? L.s[k].Ros[e] : (e == 9u ? L.s[k].Tos.t.x : (e == 10u ? L.s[k].Tos.t.y : L.s[k].Tos.t.z));
    }
    const float qnan = u2f(0x7fc00000u);
    V3 c_d[B2_ICP_REG_PAIRS], c_I[B2_ICP_REG_PAIRS], c_N[B2_ICP_REG_PAIRS];
    // ---- everything that does not depend on the find kernel: with the programmatic launch this overlaps find's tail ----
    if (S.zc_ranges) {
        if (S.zc_flag) {                                           // wait for the copy engine (long done in practice: the copy started before find)
            bool arrived = true;
            if (tid == 0) {
                const long long t0 = clock64();
                unsigned int v, spins = 0;
                while (true) {
                    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(S.zc_flag) : "memory");
                    if (v == S.zc_seq) break;
                    if ((++spins & 0x3ffu) == 0u && (clock64() - t0 > 4000000000ll || *reinterpret_cast<volatile unsigned int*>(bar_abort) != 0u)) { arrived = false; atomicCAS(bar_abort, 0u, 1u); break; }
                }
            }
            if (__syncthreads_or(!arrived)) return;
        }
        for (uint32_t u = 0; u < n_cached; u++) {
            const uint32_t i = lid + u * stride;
            const bool in = i < n;
            const uint32_t j = in ? i : 0u, oj = S.zc_n_origs == 1 ? 0u : j;
            const float r = S.zc_flag ? __ldcg(S.zc_ranges + j) : __ldcs(S.zc_ranges + j);
            const V3 dir = mk3(S.zc_dirs[3 * j], S.zc_dirs[3 * j + 1], S.zc_dirs[3 * j + 2]), org = mk3(S.zc_origs[3 * oj], S.zc_origs[3 * oj + 1], S.zc_origs[3 * oj + 2]);
            V3 d = mk3(add(mul(dir.x, r), org.x), add(mul(dir.y, r), org.y), add(mul(dir.z, r), org.z));
            const bool valid = !(r < S.range_min || r > S.range_max);
            if (in) {      // keep the handle's dataset / scan buffers coherent for datasetView(), computeCrossStatistics(), segment()
                S.dpts_out[3 * j] = d.x; S.dpts_out[3 * j + 1] = d.y; S.dpts_out[3 * j + 2] = d.z;
                S.dmask_out[j] = valid ? 1 : 0; if (!S.zc_flag) S.ranges_out[j] = r;
            }
            if (!(in && valid)) d.x = qnan;
            if (u < B2_ICP_REG_PAIRS) { if (u == 0) c_d[0] = d; else c_d[1] = d; }
            else { float* p = s_pairs + (size_t)(u - B2_ICP_REG_PAIRS) * 9 * B2_ICP_BLOCK + tid; p[0] = d.x; p[B2_ICP_BLOCK] = d.y; p[2 * B2_ICP_BLOCK] = d.z; }
        }
    } else {
        // the dataset half of this thread's pairs (written before the find was launched), with its own validity folded in.  Each block first
        // pulls one slice of its sensor's whole dataset into L2: a block that becomes resident early behind the find then warms the pairs of
        // the block that lands last (on the SM the find leaves last), whose loads are on the critical path.
        if (tid == 0u) bulk_prefetch_slice(S.dpts, 12ull * n, blockIdx.x - S.blk0, S.nblk);
        else if (tid == 32u) bulk_prefetch_slice(S.dmask, n, blockIdx.x - S.blk0, S.nblk);
        for (uint32_t u = 0; u < n_cached; u++) {
            const uint32_t i = lid + u * stride;
            const bool in = i < n;
            const uint32_t j = in ? i : 0u;
            V3 d = mk3(S.dpts[3 * j], S.dpts[3 * j + 1], S.dpts[3 * j + 2]);
            if (!(in && (S.dmask[j] > 0))) d.x = qnan;
            if (u < B2_ICP_REG_PAIRS) { if (u == 0) c_d[0] = d; else c_d[1] = d; }
            else { float* p = s_pairs + (size_t)(u - B2_ICP_REG_PAIRS) * 9 * B2_ICP_BLOCK + tid; p[0] = d.x; p[B2_ICP_BLOCK] = d.y; p[2 * B2_ICP_BLOCK] = d.z; }
        }
    }
    unsigned long long* const acc_w = xbuf;
    unsigned long long* const base_w = xbuf + B2_ICP_ACC_WORDS;
    ulonglong2* const slots = reinterpret_cast<ulonglong2*>(xbuf + B2_ICP_ACC_WORDS + B2_ICP_BASE_WORDS);
    // written by block 0 of the previous launch, which completed before the find this launch follows was started
    if (!COOP && tid < 2u * B2_MAX_SENSORS * 32u) (&s_prev[0][0][0])[tid] = __ldcg(base_w + tid);
    if (!COOP) asm volatile("griddepcontrol.wait;" ::: "memory");
    // ---- the model half of this thread's pairs, from the find: validity is folded into the dataset point (NaN fails the P2L gate like a masked pair) ----
    // Slots beyond the sensor's pairs read pair 0 (and are then masked): every sensor that is given blocks has at least one pair (api.cu: loop_layout).
    for (uint32_t u = 0; u < n_cached; u++) {
        const uint32_t i = lid + u * stride;
        const uint32_t j = i < n ? i : 0u;
        V3 d;
        if (u < B2_ICP_REG_PAIRS) d = (u == 0) ? c_d[0] : c_d[1];
        else { const float* p = s_pairs + (size_t)(u - B2_ICP_REG_PAIRS) * 9 * B2_ICP_BLOCK + tid; d = mk3(p[0], p[B2_ICP_BLOCK], p[2 * B2_ICP_BLOCK]); }
        if (!(S.mmask[j] > 0)) d.x = qnan;
        const V3 I = mk3(S.mpts[3 * j], S.mpts[3 * j + 1], S.mpts[3 * j + 2]), N = mk3(S.mnrm[3 * j], S.mnrm[3 * j + 1], S.mnrm[3 * j + 2]);
        if (u < B2_ICP_REG_PAIRS) { if (u == 0) { c_d[0] = d; c_I[0] = I; c_N[0] = N; } else { c_d[1] = d; c_I[1] = I; c_N[1] = N; } }
        else {
            float* p = s_pairs + (size_t)(u - B2_ICP_REG_PAIRS) * 9 * B2_ICP_BLOCK + tid;
            p[0] = d.x; p[B2_ICP_BLOCK] = d.y; p[2 * B2_ICP_BLOCK] = d.z;
            p[3 * B2_ICP_BLOCK] = I.x; p[4 * B2_ICP_BLOCK] = I.y; p[5 * B2_ICP_BLOCK] = I.z;
            p[6 * B2_ICP_BLOCK] = N.x; p[7 * B2_ICP_BLOCK] = N.y; p[8 * B2_ICP_BLOCK] = N.z;
        }
    }
    __syncthreads();
    // a chain step gates with the progress the previous step left (written before this grid's find was launched)
    const float max_dist = L.chain ? icp_adaptive_max_dist(S.max_dist, S.max_dist_min, L.chain->cp) : S.max_dist;
    Tf T = tf_identity();                                          // T_onew_oold: the same value on every lane of warp 0
    const long long k1 = clock64();
    for (uint32_t it = 0; it < L.iterations; it++) {
        const long long c0 = clock64();
        const Tf Tpre = s_Tpre[si];
        P2LAcc acc; acc_zero(acc);
        #pragma unroll
        for (int u = 0; u < B2_ICP_REG_PAIRS; u++) {
            V3 D, M;
            if (p2l_pair(Tpre, c_d[u], c_I[u], c_N[u], max_dist, D, M)) acc_add_pair(acc, D, M);
        }
        for (uint32_t u = 0; u < smem_u; u++) {
            const float* p = s_pairs + (size_t)u * 9 * B2_ICP_BLOCK + tid;
            V3 D, M;
            if (p2l_pair(Tpre, mk3(p[0], p[B2_ICP_BLOCK], p[2 * B2_ICP_BLOCK]), mk3(p[3 * B2_ICP_BLOCK], p[4 * B2_ICP_BLOCK], p[5 * B2_ICP_BLOCK]),
                         mk3(p[6 * B2_ICP_BLOCK], p[7 * B2_ICP_BLOCK], p[8 * B2_ICP_BLOCK]), max_dist, D, M)) acc_add_pair(acc, D, M);
        }
        for (uint32_t i = lid + n_cached * stride; i < n; i += stride) {        // beyond registers + shared memory: streamed from L2 every iteration
            const uint8_t dm = S.dmask[i], mm = S.mmask[i];
            const V3 d = mk3(S.dpts[3 * i], S.dpts[3 * i + 1], S.dpts[3 * i + 2]);
            const V3 I = mk3(S.mpts[3 * i], S.mpts[3 * i + 1], S.mpts[3 * i + 2]), N = mk3(S.mnrm[3 * i], S.mnrm[3 * i + 1], S.mnrm[3 * i + 2]);
            V3 D, M;
            if ((dm > 0) && (mm > 0) && p2l_pair(Tpre, d, I, N, max_dist, D, M)) acc_add_pair(acc, D, M);
        }
        block_reduce_to_smem<B2_ICP_BLOCK>(acc, smem);
        const long long c1 = clock64();
        if (it < 3u && S.tile_perm && blockIdx.x == S.blk0 && warp >= 1u && L.iterations >= 3u) {
            uint16_t* s_cost = reinterpret_cast<uint16_t*>(s_pairs + (size_t)L.smem_u_max * 9 * B2_ICP_BLOCK);      // behind the pair cache
            if (it == 0) tile_perm_load(S.tile_cost, S.n_tiles, s_cost, s_bin, tid - 32u);          // the block barrier at the end of every iteration separates the phases
            else if (it == 1) tile_perm_count(S.n_tiles, s_cost, s_bin, tid - 32u);
            else tile_perm_scatter(S.n_tiles, s_cost, s_bin, S.tile_perm, tid - 32u);
        }
        constexpr int NW = B2_ICP_BLOCK / 32;
        const uint32_t par = (tag_base + it) & 1u;
        bool ok = true;
        if (COOP) {
            // ---- cooperative variant: FP64 slots {low word | tag, high word | tag}, grid sync, every block sums all slots in a fixed order ----
            const unsigned int tag = tag_base + it + 1u;
            ulonglong2* part = slots + (size_t)par * B2_ICP_MAX_GRID * (B2_NACC + 1);
            if (warp == 0 && lane < 16) {
                double x = 0.0;
                #pragma unroll
                for (int w = 0; w < NW; w++) x += smem[w * 16 + lane];     // fixed order
                slot_store(part + (size_t)blockIdx.x * (B2_NACC + 1) + lane, x, tag);
            }
            __threadfence(); cg::this_grid().sync();
            const uint32_t i = tid & 15u, g = tid >> 4;                    // thread = (group g of 32, value i of 16)
            for (uint32_t k = 0; k < L.n_sensors; k++) {
                const uint32_t b0 = L.s[k].blk0, b1 = b0 + L.s[k].nblk;
                double a[5];
                #pragma unroll
                for (int q = 0; q < 5; q++) { a[q] = 0.0; if (b0 + g + 32u * q < b1 && !slot_load(part + (size_t)(b0 + g + 32u * q) * (B2_NACC + 1) + i, tag, a[q])) ok = false; }
                double x = ((a[0] + a[1]) + (a[2] + a[3])) + a[4];
                x += __shfl_xor_sync(0xffffffffu, x, 16);          // the warp's two groups
                if (lane < 16) s_part[k][warp][lane] = x;
            }
            if (!ok) atomicExch(bar_abort, 3u);                    // cannot happen behind a grid sync; never continue on an incomplete sum
            __syncthreads();
        }
        const long long c2 = clock64();
        if (warp == 0) {
            const int e = (int)lane, cr = lane >= 6u && lane < 15u ? (int)lane - 6 : 0, rr = cr % 3, cc = cr / 3;
            if (!COOP) {
                // ---- publish this block's sums: lane = (limb, value); both halves of the warp add the 16 per-warp totals in the same order ----
                const uint32_t v = lane & 15u, limb = lane >> 4;
                double x = 0.0;
                #pragma unroll
                for (int w = 0; w < NW / 2; w++) x += smem[w * 16 + v];
                double y = 0.0;
                #pragma unroll
                for (int w = NW / 2; w < NW; w++) y += smem[w * 16 + v];
                x += y;
                if (!(fabs(x) < 70368744177664.0)) { ok = false; atomicExch(bar_abort, 2u); }      // 2^46 (also catches NaN / Inf)
                const double fl = floor(x);
                const long long q = limb ? __double2ll_rn((x - fl) * 1099511627776.0) : __double2ll_rn(fl);      // 2^40
                if (ok) acc_red(acc_w + ((size_t)(par * B2_MAX_SENSORS + si) * 32u + lane) * B2_ICP_ACC_STRIDE, ((unsigned long long)q << 8) + 1ull);
#if defined(B2_ICP_PROFILE)
                if (it == 1 && dbg && lane == 0) { dbg[16 + 4 * blockIdx.x] = globaltimer_ns(); dbg[16 + 4 * blockIdx.x + 2] = (unsigned long long)(clock64() - c1); }
#endif
            }
            // ---- per sensor: the grid-wide sums on lanes 0..15, then the 15 elements of the statistics on 15 lanes, moved between the lanes
            //      by shuffles: finalised (sensor frame) -> odom frame -> every lane's copy of the sensor's statistics -> merged ----
            int orow, ocol;                                         // the rows of Ros that this lane's odom-frame element reads
            icp_odom_rows(lane < 15u ? e : 0, orow, ocol);
            CStats merged = cs_identity(), merged_w = cs_identity();
            for (uint32_t k = 0; k < L.n_sensors; k++) {
                float Rr[3], Rj[3];
                #pragma unroll
                for (int q = 0; q < 3; q++) { Rr[q] = s_Rt[k][orow * 3 + q]; Rj[q] = s_Rt[k][ocol * 3 + q]; }
                const float tr = s_Rt[k][9 + orow];
                double x = 0.0;
                if (COOP) {
                    if (lane < 16u) {
                        #pragma unroll
                        for (int w = 0; w < NW; w++) x += s_part[k][w][lane];              // fixed order
                    }
                } else {
                    const unsigned long long prev = s_prev[par][k][lane], nb = L.s[k].nblk;
                    const unsigned long long* wp = acc_w + ((size_t)(par * B2_MAX_SENSORS + k) * 32u + lane) * B2_ICP_ACC_STRIDE;
                    unsigned long long w = 0;
                    long long t0 = 0;
                    for (uint32_t spins = 0; ok; spins++) {
                        w = acc_ld(wp);
                        if (((w - prev - nb) & 255ull) == 0ull) break;
                        if ((spins & 0x3ffu) == 0x3ffu) {
                            if (t0 == 0) t0 = clock64();
                            if (clock64() - t0 > 4000000000ll || *reinterpret_cast<volatile unsigned int*>(bar_abort) != 0u) { ok = false; atomicCAS(bar_abort, 0u, 1u); }
                        }
                    }
                    ok = __all_sync(0xffffffffu, ok);
#if defined(B2_ICP_PROFILE)
                    if (it == 1 && dbg && lane == 0 && k == 0) { dbg[16 + 4 * blockIdx.x + 1] = globaltimer_ns(); dbg[16 + 4 * blockIdx.x + 3] = (unsigned long long)(clock64() - c1); }
#endif
                    s_prev[par][k][lane] = w;
                    const double part = (double)((long long)(w - prev - nb) >> 8);                   // the sum of the limbs, modulo 2^56, sign-extended
                    const double lo = __shfl_down_sync(0xffffffffu, part, 16);
                    x = part + lo * 9.094947017729282379150390625e-13;                                // 2^-40
                }
                // the count first: its reciprocal is the longest chain here and does not wait for the value shuffles
                const double cnt = __shfl_sync(0xffffffffu, x, 15);
                const uint32_t nk = (uint32_t)(cnt + 0.5);
                const double inv = nk ? b2_rcp_u32(nk) : 0.0;
                const double vm = __shfl_sync(0xffffffffu, x, 3 + rr), vd = __shfl_sync(0xffffffffu, x, cc);
                const float fin = icp_finalize_elem(x, vm, vd, inv, e);                              // lanes 0..14 (the rest is not read)
                float p[3], Cs[9];
                #pragma unroll
                for (int q = 0; q < 3; q++) p[q] = __shfl_sync(0xffffffffu, fin, (lane < 3u ? 0 : 3) + q);
                #pragma unroll
                for (int q = 0; q < 9; q++) Cs[q] = __shfl_sync(0xffffffffu, fin, 6 + q);
                const float od = icp_to_odom_rows(Rr, Rj, tr, p, Cs, e);
                CStats o; o.n = nk;
                o.dm = mk3(__shfl_sync(0xffffffffu, od, 0), __shfl_sync(0xffffffffu, od, 1), __shfl_sync(0xffffffffu, od, 2));
                o.mm = mk3(__shfl_sync(0xffffffffu, od, 3), __shfl_sync(0xffffffffu, od, 4), __shfl_sync(0xffffffffu, od, 5));
                #pragma unroll
                for (int q = 0; q < 9; q++) o.C[q] = __shfl_sync(0xffffffffu, od, 6 + q);
                icp_merge_sensor(L, k, o, merged, merged_w);
            }
            const long long c3 = clock64();
            long long st[8] = {0, 0, 0, 0, 0, 0, 0, 0};
            const bool prof = it == 1 && blockIdx.x == 0 && dbg && lane == 0;
            const bool mine = lane < L.n_sensors;                                                    // lane k prepares sensor k's next pre-transform
            if (ok) icp_tail_rest(L, s_Tom, merged, merged_w, T, s_Tpre, mine ? lane : 0u, mine ? lane + 1u : 0u, it + 1 == L.iterations, lane == 0 ? &s_res : nullptr, prof ? st : nullptr);
            if (prof) {
                const long long c4 = clock64();
                dbg[0] = (unsigned long long)(c1 - c0); dbg[1] = (unsigned long long)(c2 - c1); dbg[2] = (unsigned long long)(c3 - c2); dbg[3] = (unsigned long long)(c4 - c3);
#if defined(B2_ICP_PROFILE)
                for (int q = 0; q < 8; q++) dbg[8 + q] = (unsigned long long)(st[q] - c3);
#endif
            }
        }
#if defined(B2_ICP_PROFILE)
        if (dbg && blockIdx.x == 0 && it == 0 && lane == 0) { if (warp == 0) dbg[641] = (unsigned long long)(clock64() - c1); else atomicMax(dbg + 642, (unsigned long long)(clock64() - c1)); }
#endif
        if (__syncthreads_or(!ok)) return;                         // gave up: the host finds the abort word set and re-runs the step cooperatively
    }
    if (!COOP && blockIdx.x == 0 && tid < 2u * B2_MAX_SENSORS * 32u) base_w[tid] = (&s_prev[0][0][0])[tid];      // the accumulators' state for the next launch
    if (blockIdx.x == 0) {
        // result: device copy + (spin path) mapped pinned host memory, 16-byte chunks {3 payload words, sequence number}: each chunk is one
        // store, the host accepts the result when every chunk carries this call's sequence number -- no flag, no system-wide fence
        const uint32_t* w = reinterpret_cast<const uint32_t*>(&s_res);
        if (tid < 32u) reinterpret_cast<uint32_t*>(res_dev)[tid] = w[tid];
        if (host_out && tid < B2_ICP_RESULT_CHUNKS) {
            uint4 c; c.x = w[3 * tid]; c.y = 3 * tid + 1 < 32u ? w[3 * tid + 1] : 0u; c.z = 3 * tid + 2 < 32u ? w[3 * tid + 2] : 0u; c.w = L.seq;
            asm volatile("st.volatile.global.v4.u32 [%0], {%1, %2, %3, %4};" ::"l"(host_out + tid), "r"(c.x), "r"(c.y), "r"(c.z), "r"(c.w) : "memory");
        }
        if (L.chain && tid == 0) {
            // chain step: the progress (micp_localization.cpp:988-1007), then the state the next step reads -- the next find's pose (Tom_ after
            // :983) and the progress its loop gates with -- and this step's record.  Every block has read the previous state before it
            // contributed to this grid's first exchange, so nothing reads what is overwritten here.
            IcpChainState* c = L.chain;
            const uint32_t valid = c->valid;
            const double cp = micp_progress(s_Tom, s_res.T_onew_oold, s_res.Cmerged_o.n_meas, valid, L.adaptive != 0u);
            for (uint32_t k = 0; k < L.n_sensors; k++) c->find[k].Tom = s_res.Tom_new;
            c->cp = cp;
            b2_micp_step* r = L.step_out;
            r->Tom_new = s_res.Tom_new; r->T_onew_oold = s_res.T_onew_oold; r->Cmerged_o = s_res.Cmerged_o;
            r->convergence_progress = cp; r->valid_measurements = valid; r->total_measurements = c->total;
            c->done++;
        }
        if (tid == 0 && dbg) { dbg[4] = (unsigned long long)(k1 - k0); dbg[5] = (unsigned long long)(clock64() - k0); dbg[6] = g0; dbg[7] = globaltimer_ns(); }
    }
}

// stats.valid_measurements of a chain (micp_localization.cpp:866-871): the mask ones of one sensor's dataset (mask > 0, as unpackMessage
// counts them), added to *out; once per sensor at the start of the chain, the dataset is fixed for the whole call
__global__ void k_mask_count(const uint8_t* __restrict__ mask, uint32_t n, uint32_t* __restrict__ out)
{
    uint32_t c = 0;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) c += mask[i] > 0 ? 1u : 0u;
    c = __reduce_add_sync(0xffffffffu, c);
    if ((threadIdx.x & 31u) == 0u && c) atomicAdd(out, c);
}
#endif
