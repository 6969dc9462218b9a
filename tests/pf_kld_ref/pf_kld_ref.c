/* TEST INFRASTRUCTURE ONLY: reference for KLD-sampling (b2_pf_resample_kld; Fox, IJRR 2003; SURVEY appendix G).
 *
 * A sequential C restatement of the resampler: integer weights and their prefix, draw j's 64-bit uniform from words 2(j % 2), 2(j % 2) + 1 of
 * Philox4x32-10 with counter (lo(j / 2), 6, step, hi(j / 2)), the parent by the prefix, the bin key of the parent's pose (the yaw sector
 * counted boundary by boundary, not searched), a set of the keys drawn so far, Fox's bound and the stop rule, then residual's copy of each
 * drawn parent.  The residual restatement's source is compiled into this file (and through it the oracle's), so Philox, the normals and the
 * copy are the ones used there, not copies.  Plain float / double ops, compiled with -ffp-contract=off: each is individually rounded. */
#include "../pf_residual_ref/pf_residual_ref.c"

#include <stdlib.h>

#define ORC_KLD_DRAW_TAG 6u
#define ORC_KLD_PI 3.14159265358979323846

typedef struct { float res_xy, res_z, res_yaw; uint32_t n_min; double epsilon, z; } orc_kld_config;

/* K = ceil(2 pi / res_yaw (1 - 2^-20)); 0 when outside [1, 32768] */
uint32_t orc_kld_sectors(float res_yaw)
{
    const double K = ceil(2.0 * ORC_KLD_PI / (double)res_yaw * (1.0 - 0x1p-20));
    return (K >= 1.0 && K <= 32768.0) ? (uint32_t)K : 0u;
}

/* the K boundary vectors (cos, sin) of theta_k = -pi + 2 pi k / K, as floats */
void orc_kld_table(uint32_t K, float* cs)
{
    for (uint32_t k = 0; k < K; k++) {
        const double th = -ORC_KLD_PI + 2.0 * ORC_KLD_PI * (double)k / (double)K;
        cs[2 * k] = (float)cos(th); cs[2 * k + 1] = (float)sin(th);
    }
}

static float cell(float v, float res, float half)
{
    float c = floorf(v / res);
    if (c < -half) c = -half;
    if (c > half - 1.0f) c = half - 1.0f;
    return c;
}

static int finite_f(float v) { return isfinite(v); }

/* the number of boundaries k in [1, K) at or before phi(h), counted one by one */
uint32_t orc_kld_sector(float hx, float hy, const float* cs, uint32_t K)
{
    if (hx == 0.0f && hy == 0.0f) return 0u;
    const int lower = hy < 0.0f || (hy == 0.0f && hx < 0.0f);
    uint32_t s = 0;
    for (uint32_t k = 1; k < K; k++) {
        const int b_lower = 2 * k < K;
        if (b_lower != lower) { s += b_lower; continue; }          /* a lower boundary lies before every upper heading */
        const double c = (double)cs[2 * k] * (double)hy - (double)cs[2 * k + 1] * (double)hx;
        s += c >= 0.0;
    }
    return s;
}

uint64_t orc_kld_key(orc_transform p, float res_xy, float res_z, const float* cs, uint32_t K)
{
    if (!(finite_f(p.t.x) && finite_f(p.t.y) && finite_f(p.t.z) && finite_f(p.R.x) && finite_f(p.R.y) && finite_f(p.R.z) && finite_f(p.R.w)))
        return ~0ull;
    const float ix = cell(p.t.x, res_xy, 524288.0f), iy = cell(p.t.y, res_xy, 524288.0f);
    const float iz = res_z > 0.0f ? cell(p.t.z, res_z, 128.0f) : 0.0f;
    const float x = p.R.x, y = p.R.y, z = p.R.z, w = p.R.w;
    const float hx = 1.0f - 2.0f * (y * y + z * z);
    const float hy = 2.0f * (x * y + w * z);
    const uint64_t sec = orc_kld_sector(hx, hy, cs, K);
    return (uint64_t)((int64_t)ix + 524288) << 44 | (uint64_t)((int64_t)iy + 524288) << 24 | (uint64_t)((int64_t)iz + 128) << 16 | sec;
}

void orc_kld_keys(const orc_transform* poses, uint64_t count, float res_xy, float res_z, const float* cs, uint32_t K, uint64_t* out)
{
    #pragma omp parallel for schedule(static)
    for (int64_t i = 0; i < (int64_t)count; i++) out[i] = orc_kld_key(poses[i], res_xy, res_z, cs, K);
}

uint64_t orc_kld_bound(uint64_t k, double epsilon, double z, uint32_t n_min)
{
    if (k <= 1) return n_min;
    const double km1 = (double)(k - 1);
    const double a = 2.0 / (9.0 * km1);
    const double x = (1.0 - a) + sqrt(a) * z;
    const double v = (km1 / (2.0 * epsilon)) * ((x * x) * x);
    if (!(v > 0.0)) return 0;
    const double c = ceil(v);
    return c >= 18446744073709551616.0 ? ~0ull : (uint64_t)c;
}

void orc_kld_bounds(const uint64_t* k, uint64_t count, double epsilon, double z, uint32_t n_min, uint64_t* out)
{
    for (uint64_t i = 0; i < count; i++) out[i] = orc_kld_bound(k[i], epsilon, z, n_min);
}

/* the integer weights' inclusive prefix W */
void orc_kld_prefix(uint32_t n, const orc_particle_attr* attrs, double L_max, uint64_t* W)
{
    uint64_t s = 0;
    for (uint32_t i = 0; i < n; i++) {
        s += (uint64_t)((double)attrs[i].likelihood.mean / L_max * 4294967296.0);
        W[i] = s;
    }
}

/* the parents of draws d0 .. d0+count-1 over the prefix W of n weights: the smallest i with W[i] > mulhi64(u, W[n-1]) */
void orc_kld_parents(uint64_t seed, uint32_t step, uint64_t d0, uint64_t count, const uint64_t* W, uint32_t n, uint32_t* out)
{
    const uint32_t key[2] = {(uint32_t)seed, (uint32_t)(seed >> 32)};
    #pragma omp parallel for schedule(static)
    for (int64_t i = 0; i < (int64_t)count; i++) {
        const uint64_t j = d0 + (uint64_t)i, b = j >> 1;
        const uint32_t c[4] = {(uint32_t)b, ORC_KLD_DRAW_TAG, step, (uint32_t)(b >> 32)};
        uint32_t r[4];
        orc_philox4x32_10(c, key, r);
        const uint64_t u = (uint64_t)r[2 * (j & 1u) + 1] << 32 | r[2 * (j & 1u)];
        const uint64_t x = (uint64_t)(((unsigned __int128)u * W[n - 1]) >> 64);
        uint32_t lo = 0, hi = n - 1;
        while (lo < hi) { const uint32_t mid = lo + (hi - lo) / 2; if (W[mid] > x) hi = mid; else lo = mid + 1; }
        out[i] = lo;
    }
}

/* a set of 64-bit keys: open addressing over a power-of-two table with a separate occupancy byte */
typedef struct { uint64_t* k; uint8_t* used; uint64_t mask, size; } keyset;
static int keyset_insert(keyset* s, uint64_t key)                         /* 1 iff the key is new */
{
    uint64_t h = key * 0x9e3779b97f4a7c15ull;
    for (uint64_t i = (h ^ (h >> 29)) & s->mask;; i = (i + 1) & s->mask) {
        if (!s->used[i]) { s->used[i] = 1; s->k[i] = key; s->size++; return 1; }
        if (s->k[i] == key) return 0;
    }
}

/* The whole resampler with the statistics given (S, L_min, L_max).  Writes the slots in [first, first + n_local) below n_particles to
 * poses_new[k - first] / attrs_new[k - first].  The parents and keys of the draws made go to parents_out / keys_out (n_max entries, may be
 * NULL).  res[0] = n_particles, res[1] = bins. */
void orc_pf_resample_kld(uint32_t n, const orc_transform* poses, const orc_particle_attr* attrs, uint32_t n_max, double S, double L_min, double L_max,
                         const orc_gladiator_config* cfg, const orc_kld_config* kc, uint64_t seed, uint32_t step, uint32_t first, uint32_t n_local,
                         orc_transform* poses_new, orc_particle_attr* attrs_new, uint32_t* parents_out, uint64_t* keys_out, uint64_t res[2])
{
    res[0] = res[1] = 0;
    if (!(isfinite(S) && S > 0.0 && L_min >= 0.0)) return;
    const uint32_t K = orc_kld_sectors(kc->res_yaw);
    float* cs = malloc(sizeof(float) * 2 * K);
    uint64_t* W = malloc(sizeof(uint64_t) * n);
    uint32_t* par = malloc(sizeof(uint32_t) * n_max);
    orc_kld_table(K, cs);
    orc_kld_prefix(n, attrs, L_max, W);
    orc_kld_parents(seed, step, 0, n_max, W, n, par);                     /* keyed by index: drawing them all first changes nothing */
    keyset s = {0};
    uint64_t T = 1;
    while (T < 2 * (uint64_t)n_max) T <<= 1;
    s.k = malloc(sizeof(uint64_t) * T); s.used = calloc(T, 1); s.mask = T - 1;
    uint64_t j = 0;
    for (;; j++) {
        const uint64_t key = orc_kld_key(poses[par[j]], kc->res_xy, kc->res_z, cs, K);
        keyset_insert(&s, key);
        if (parents_out) parents_out[j] = par[j];
        if (keys_out) keys_out[j] = key;
        const uint64_t b = orc_kld_bound(s.size, kc->epsilon, kc->z, kc->n_min);
        if (j + 1 >= (b > kc->n_min ? b : kc->n_min) || j + 1 == n_max) break;
    }
    const uint64_t np = j + 1;
    #pragma omp parallel for schedule(static)
    for (int64_t k = first; k < (int64_t)first + n_local; k++) {
        if ((uint64_t)k >= np) continue;
        float N[6];
        normals_one(seed, step, (uint32_t)k, N);
        orc_residual_copy(poses[par[k]], attrs[par[k]], L_max, N, cfg, poses_new + (k - first), attrs_new + (k - first));
    }
    res[0] = np; res[1] = s.size;
    free(cs); free(W); free(par); free(s.k); free(s.used);
}
