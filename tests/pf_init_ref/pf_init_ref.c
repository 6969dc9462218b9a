/* TEST INFRASTRUCTURE ONLY: reference for the particle set initialisers (b2_pf_init_uniform, b2_pf_init_gaussian).
 *
 * RmclNode::initSamplesUniform (rmcl_ros/src/nodes/rmcl_localization.cpp:277-342) and RmclNode::initSamples(PoseWithCovarianceStamped)
 * (:165-275) restated in C with the draws of the library: Philox4x32-10, counter (global particle index, tag, 0, block), key = seed; tag 1
 * uniform, tag 2 Gaussian.  The oracle's source is compiled into this file, so its Philox, Box-Muller constants, euler_to_quat and Transform
 * product are the ones used here, not copies.  Plain float ops, compiled with -ffp-contract=off: each is individually rounded. */
#include "../../oracle/oracle.c"

#define ORC_INIT_TAG_UNIFORM 1u
#define ORC_INIT_TAG_GAUSSIAN 2u

/* rm::chol (Cholesky-Banachiewicz in float, sums over k in order) of the 36 doubles narrowed to float, lower triangle only, with the
 * library's rule for zero pivots: a zero pivot whose column numerators are all exactly 0 gives a zero column; a negative or NaN pivot, a
 * zero pivot with a non-zero numerator, a non-finite entry or a non-finite factor is refused.  Returns 0, or 1 + the offending column. */
int orc_pf_chol6(const double cov[36], float L[36])
{
    float A[36];
    for (int i = 0; i < 36; i++) { A[i] = (float)cov[i]; L[i] = 0.0f; }
    for (int i = 0; i < 6; i++)
        for (int j = 0; j <= i; j++)
            if (!isfinite(A[6 * i + j])) return 1 + j;
    for (int i = 0; i < 6; i++) {                                  /* row by row, as Banachiewicz; column j's pivot is row j's diagonal */
        for (int j = 0; j <= i; j++) {
            float s = 0.0f;
            for (int k = 0; k < j; k++) s += L[6 * i + k] * L[6 * j + k];
            const float num = A[6 * i + j] - s;
            if (i == j) {
                if (!(num >= 0.0f) || !isfinite(num)) return 1 + j;
                L[6 * i + i] = sqrtf(num);
            } else if (L[6 * j + j] == 0.0f) {
                if (num != 0.0f) return 1 + j;
            } else {
                L[6 * i + j] = num / L[6 * j + j];
                if (!isfinite(L[6 * i + j])) return 1 + j;
            }
        }
    }
    return 0;
}

static void init_words(uint64_t seed, uint32_t gidx, uint32_t tag, uint32_t r[8])
{
    const uint32_t key[2] = {(uint32_t)seed, (uint32_t)(seed >> 32)};
    const uint32_t c0[4] = {gidx, tag, 0u, 0u}, c1[4] = {gidx, tag, 0u, 1u};
    orc_philox4x32_10(c0, key, r); orc_philox4x32_10(c1, key, r + 4);
}

static void init_attr(orc_particle_attr* a)
{
    a->likelihood.mean = 1.0f; a->likelihood.sigma = 0.0f; a->likelihood.n_meas = 0u;
    for (int k = 0; k < 6; k++) a->state_sigma[k] = 0.0f;
}

/* lo / hi: the box narrowed to float (x, y, z, roll, pitch, yaw).  v = min(lo + (hi - lo) u, hi), u = (r >> 8) 2^-24 in [0, 1) */
void orc_pf_init_uniform(uint32_t first, uint32_t n, const float lo[6], const float hi[6], uint64_t seed, orc_transform* poses, orc_particle_attr* attrs)
{
    #pragma omp parallel for schedule(static)
    for (int64_t i = 0; i < (int64_t)n; i++) {
        uint32_t r[8];
        init_words(seed, first + (uint32_t)i, ORC_INIT_TAG_UNIFORM, r);
        float v[6];
        for (int k = 0; k < 6; k++) {
            const float u = (float)(r[k] >> 8) * 5.9604644775390625e-08f;
            v[k] = fminf(lo[k] + (hi[k] - lo[k]) * u, hi[k]);
        }
        orc_transform T;
        T.t = v3(v[0], v[1], v[2]); T.R = euler_to_quat(v[3], v[4], v[5]); T.stamp = 0;
        poses[i] = T;
        init_attr(attrs + i);
    }
}

/* the N(0, I6) draws of one particle: Box-Muller on (r0, r1), (r2, r3), (r4, r5) as in orc_pf_gladiator_randoms */
static void init_normals_one(uint64_t seed, uint32_t gidx, float N[6])
{
    uint32_t r[8];
    init_words(seed, gidx, ORC_INIT_TAG_GAUSSIAN, r);
    for (int p = 0; p < 3; p++) {
        const float u1 = u01_open(r[2 * p]), u2 = u01_open(r[2 * p + 1]);
        const float rad = sqrtf(-2.0f * logf(u1)), ang = 6.283185307179586f * u2;
        N[2 * p] = rad * cosf(ang);
        N[2 * p + 1] = rad * sinf(ang);
    }
}

void orc_pf_init_normals(uint32_t first, uint32_t n, uint64_t seed, float* normals)
{
    #pragma omp parallel for schedule(static)
    for (int64_t i = 0; i < (int64_t)n; i++) init_normals_one(seed, first + (uint32_t)i, normals + 6 * i);
}

/* L: orc_pf_chol6's factor.  normals (n x 6) may be NULL (drawn here) or given, to isolate the arithmetic from the generator.
 * x = L N (rm::Matrix_ product: a = 0, a += L(i,k) N(k) for k = 0..5), pose = Tlm * Transform{EulerAngles{x3, x4, x5}, {x0, x1, x2}} */
void orc_pf_init_gaussian(uint32_t first, uint32_t n, const float L[36], const orc_transform* Tlm, uint64_t seed, const float* normals,
                          orc_transform* poses, orc_particle_attr* attrs)
{
    #pragma omp parallel for schedule(static)
    for (int64_t i = 0; i < (int64_t)n; i++) {
        float N[6], x[6];
        if (normals) { for (int k = 0; k < 6; k++) N[k] = normals[6 * i + k]; }
        else init_normals_one(seed, first + (uint32_t)i, N);
        for (int r = 0; r < 6; r++) {
            float a = 0.0f;
            for (int k = 0; k < 6; k++) a += L[6 * r + k] * N[k];
            x[r] = a;
        }
        orc_transform Pl;
        Pl.t = v3(x[0], x[1], x[2]); Pl.R = euler_to_quat(x[3], x[4], x[5]); Pl.stamp = 0;
        orc_transform T = T_mul(*Tlm, Pl);
        T.stamp = 0;
        poses[i] = T;
        init_attr(attrs + i);
    }
}
