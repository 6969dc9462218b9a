/* TEST INFRASTRUCTURE ONLY: reference for residual resampling (b2_pf_resample_residual).
 *
 * ResidualResamplerCPU::update (rmcl_ros/src/rmcl/ResidualResamplerCPU.cpp:55-202) restated in C with the library's keyed draws and its
 * decisions (SURVEY D31-D34, E5): draw j takes parent word j % 4 of Philox4x32-10 with counter (lo(j / 4), 4, step, hi(j / 4)) modulo n;
 * slot k takes its normals from counters (k, 5, step, 0 and 1); the loop stops at M filled slots or after D_max = 16 max(n, M) draws; an
 * invalid weight sum fills nothing.  The oracle's source is compiled into this file, so its Philox, Box-Muller constants, Euler conversions
 * and Transform product are the ones used here, not copies.  Plain float ops, compiled with -ffp-contract=off: each is individually rounded. */
#include "../../oracle/oracle.c"

#define ORC_RES_DRAW_TAG 4u
#define ORC_RES_NOISE_TAG 5u

/* the parents of draws d0 .. d0+count-1 among n particles */
void orc_residual_parents(uint64_t seed, uint32_t step, uint64_t d0, uint64_t count, uint32_t n, uint32_t* out)
{
    const uint32_t key[2] = {(uint32_t)seed, (uint32_t)(seed >> 32)};
    for (uint64_t i = 0; i < count; i++) {
        const uint64_t j = d0 + i, b = j >> 2;
        const uint32_t c[4] = {(uint32_t)b, ORC_RES_DRAW_TAG, step, (uint32_t)(b >> 32)};
        uint32_t r[4];
        orc_philox4x32_10(c, key, r);
        out[i] = r[j & 3u] % n;
    }
}

static void normals_one(uint64_t seed, uint32_t step, uint32_t k, float N[6])
{
    const uint32_t key[2] = {(uint32_t)seed, (uint32_t)(seed >> 32)};
    const uint32_t c0[4] = {k, ORC_RES_NOISE_TAG, step, 0u}, c1[4] = {k, ORC_RES_NOISE_TAG, step, 1u};
    uint32_t r[8];
    orc_philox4x32_10(c0, key, r); orc_philox4x32_10(c1, key, r + 4);
    for (int p = 0; p < 3; p++) {                                      /* Box-Muller on (r0, r1), (r2, r3), (r4, r5) */
        const float u1 = u01_open(r[2 * p]), u2 = u01_open(r[2 * p + 1]);
        const float rad = sqrtf(-2.0f * logf(u1)), ang = 6.283185307179586f * u2;
        N[2 * p] = rad * cosf(ang);
        N[2 * p + 1] = rad * sinf(ang);
    }
}

/* the (count, 6) normals of slots first .. first+count-1: tx, ty, tz, roll, pitch, yaw */
void orc_residual_normals(uint64_t seed, uint32_t step, uint32_t first, uint32_t count, float* out)
{
    #pragma omp parallel for schedule(static)
    for (int64_t i = 0; i < (int64_t)count; i++) normals_one(seed, step, first + (uint32_t)i, out + 6 * i);
}

/* weight_sum (sequential, as :78-84 sums), the minimum from DBL_MAX and the maximum from 0.0 of likelihood.mean in double */
void orc_residual_stats(uint32_t n, const orc_particle_attr* attrs, double out[3])
{
    double s = 0.0, mn = 1.7976931348623157e308, mx = 0.0;
    for (uint32_t i = 0; i < n; i++) {
        const double v = attrs[i].likelihood.mean;
        s += v;
        mx = (mx < v) ? v : mx;                                            /* std::max(weight_max, v) */
        mn = (v < mn) ? v : mn;                                            /* std::min(weight_min, v) */
    }
    out[0] = s; out[1] = mn; out[2] = mx;
}

/* one copy of the parent (:129-177) */
void orc_residual_copy(orc_transform pose, orc_particle_attr a, double L_max, const float N[6], const orc_gladiator_config* cfg, orc_transform* out_p,
                       orc_particle_attr* out_a)
{
    const double Lmn = (double)a.likelihood.mean / L_max;                 /* L_max_normed */
    const float s[6] = {(float)(cfg->min_noise_tx / Lmn), (float)(cfg->min_noise_ty / Lmn), (float)(cfg->min_noise_tz / Lmn),
                        (float)(cfg->min_noise_roll / Lmn), (float)(cfg->min_noise_pitch / Lmn), (float)(cfg->min_noise_yaw / Lmn)};
    orc_transform pn = pose;
    pn.t.x += N[0] * s[0]; pn.t.y += N[1] * s[1]; pn.t.z += N[2] * s[2];
    float roll, pitch, yaw; quat_to_euler(pn.R, &roll, &pitch, &yaw);
    roll += N[3] * s[3]; pitch += N[4] * s[4]; yaw += N[5] * s[5];
    pn.R = euler_to_quat(roll, pitch, yaw);
    const orc_transform d = T_mul(T_inv(pose), pn);                       /* ~pose * pose_new */
    const float trans_dist = d.t.x * d.t.x + d.t.y * d.t.y + d.t.z * d.t.z;                               /* l2normSquared */
    const float rot_dist = sqrtf(((d.R.x * d.R.x + d.R.y * d.R.y) + d.R.z * d.R.z) + d.R.w * d.R.w);     /* Quaternion::l2norm */
    const float f = (float)(pow((double)cfg->likelihood_forget_per_meter, (double)trans_dist) * pow((double)cfg->likelihood_forget_per_radian, (double)rot_dist));
    a.likelihood.n_meas = (uint32_t)((float)a.likelihood.n_meas * f);     /* uint *= float */
    pn.stamp = pose.stamp;
    *out_p = pn; *out_a = a;
}

/* The loop over M = n_new slots, with the statistics given (S, L_min, L_max).  Writes the slots in [first, first + n_local) that get filled
 * to poses_new[k - first] / attrs_new[k - first]; normals (n_new x 6) replace the keyed draws when given.  The first trace_cap draws' parents
 * and insertions go to parents_out / ins_out (may be NULL).  res[0] = n_particles, res[1] = draws. */
void orc_pf_resample_residual(uint32_t n, const orc_transform* poses, const orc_particle_attr* attrs, uint32_t n_new, double S, double L_min, double L_max,
                              const orc_gladiator_config* cfg, uint64_t seed, uint32_t step, const float* normals, uint32_t first, uint32_t n_local,
                              orc_transform* poses_new, orc_particle_attr* attrs_new, uint32_t* parents_out, uint64_t* ins_out, uint64_t trace_cap,
                              uint64_t res[2])
{
    const uint64_t M = n_new, d_max = 16 * (uint64_t)(n > n_new ? n : n_new);
    uint64_t fill = 0, j = 0;
    if (isfinite(S) && S > 0.0 && L_min >= 0.0) {
        while (fill < M && j < d_max) {
            uint32_t p;
            orc_residual_parents(seed, step, j, 1, n, &p);
            const double c = (double)attrs[p].likelihood.mean / S * (double)M;
            const uint64_t cnt = c >= (double)M ? M : (uint64_t)c, left = M - fill, ins = cnt <= left ? cnt : left;
            for (uint64_t k = fill; k < fill + ins; k++) {
                if (k < first || k >= (uint64_t)first + n_local) continue;
                float N[6];
                if (normals) { for (int e = 0; e < 6; e++) N[e] = normals[6 * k + e]; }
                else normals_one(seed, step, (uint32_t)k, N);
                orc_residual_copy(poses[p], attrs[p], L_max, N, cfg, poses_new + (k - first), attrs_new + (k - first));
            }
            if (j < trace_cap) { if (parents_out) parents_out[j] = p; if (ins_out) ins_out[j] = ins; }
            fill += ins; j++;
        }
    }
    res[0] = fill; res[1] = j;
}
