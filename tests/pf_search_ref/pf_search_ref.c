/* pf_search_ref.c -- TEST HARNESS ONLY: a C restatement of the global search's candidates, peak rule, ranking and separation pass
 * (b2_pf_global_search; SURVEY appendix M), written from the definition, independently of the product's kernels.cuh.
 * Compiled with -ffp-contract=off, so every float operation is rounded on its own as the product's are. */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define PI 3.14159265358979323846

typedef struct { float x, y, z, w; float tx, ty, tz; uint32_t stamp; } tf_t;   /* b2_transform */

static double psi_of(uint32_t k, uint32_t K) { return -PI + 2.0 * PI * (double)k / (double)K; }
static float coord(float o, uint32_t i, float step) { float a = (float)i * step; return o + a; }

/* the n = nx ny K candidate poses in c order (before any surface rule) */
void ref_search_poses(float x0, float y0, float z0, float step, uint32_t nx, uint32_t ny, uint32_t K, tf_t* out)
{
    for (uint32_t k = 0; k < K; k++) {
        const double half = psi_of(k, K) / 2.0;
        const float s = (float)sin(half), c = (float)cos(half);
        for (uint32_t j = 0; j < ny; j++)
            for (uint32_t i = 0; i < nx; i++) {
                tf_t* T = out + ((size_t)k * ny + j) * nx + i;
                T->x = 0.0f; T->y = 0.0f; T->z = s; T->w = c;
                T->tx = coord(x0, i, step); T->ty = coord(y0, j, step); T->tz = z0; T->stamp = 0u;
            }
    }
}

/* the peak flags of a score array (score < 0: invalid); -> the number of peaks, *n_valid the valid candidates */
uint64_t ref_search_peaks(const float* s, uint32_t nx, uint32_t ny, uint32_t K, uint8_t* peak, uint64_t* n_valid)
{
    const uint64_t n = (uint64_t)nx * ny * K;
    uint64_t np = 0, nv = 0;
    #pragma omp parallel for reduction(+ : np, nv) schedule(static)
    for (int64_t c = 0; c < (int64_t)n; c++) {
        peak[c] = 0;
        if (!(s[c] >= 0.0f)) continue;
        nv++;
        const int64_t i = c % nx, j = c / nx % ny, k = c / nx / ny;
        int ok = 1;
        for (int dk = -1; dk <= 1 && ok; dk++)
            for (int dj = -1; dj <= 1 && ok; dj++)
                for (int di = -1; di <= 1 && ok; di++) {
                    const int64_t ii = i + di, jj = j + dj, kk = ((k + dk) % (int64_t)K + K) % K;
                    if (ii < 0 || jj < 0 || ii >= nx || jj >= ny) continue;
                    const int64_t m = (kk * ny + jj) * nx + ii;
                    if (m == c || !(s[m] >= 0.0f)) continue;
                    if (!(s[m] < s[c] || (s[m] == s[c] && m > c))) ok = 0;
                }
        if (ok) { peak[c] = 1; np++; }
    }
    *n_valid = nv;
    return np;
}

static const float* g_scores;
static int by_rank(const void* a, const void* b)
{
    const uint32_t x = *(const uint32_t*)a, y = *(const uint32_t*)b;
    if (g_scores[x] != g_scores[y]) return g_scores[x] > g_scores[y] ? -1 : 1;
    return x < y ? -1 : (x > y ? 1 : 0);
}

/* rank the m peaks `list` (sorted in place: score descending, c ascending) and keep greedily; -> the number kept (<= max_records) */
uint32_t ref_search_records(const float* s, uint32_t* list, uint64_t m, float x0, float y0, float step, uint32_t nx, uint32_t ny, uint32_t K,
                            uint32_t max_records, float sep_xy, float sep_yaw, uint32_t* kept)
{
    g_scores = s;
    qsort(list, m, sizeof(uint32_t), by_rank);
    uint32_t n_kept = 0;
    for (uint64_t q = 0; q < m && n_kept < max_records; q++) {
        const uint32_t c = list[q];
        const double x = coord(x0, c % nx, step), y = coord(y0, c / nx % ny, step), p = psi_of(c / nx / ny, K);
        int keep = 1;
        for (uint32_t r = 0; r < n_kept && keep; r++) {
            const uint32_t o = kept[r];
            const double dx = x - coord(x0, o % nx, step), dy = y - coord(y0, o / nx % ny, step);
            double dp = fabs(p - psi_of(o / nx / ny, K));
            if (2.0 * PI - dp < dp) dp = 2.0 * PI - dp;
            if (sqrt(dx * dx + dy * dy) < (double)sep_xy && dp < (double)sep_yaw) keep = 0;
        }
        if (keep) kept[n_kept++] = c;
    }
    return n_kept;
}
