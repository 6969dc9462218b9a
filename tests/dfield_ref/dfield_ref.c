/* TEST INFRASTRUCTURE ONLY: reference for the distance field (b2_dfield_*; no reference implementation).
 *
 * A node's value restated over the oracle's closest point (orc_closest_point, brute force or through the oracle's own binary BVH): the
 * distance clamped at trunc, trunc where no face counts.  The oracle's source is compiled into this file. */
#include "../../oracle/oracle.c"

/* out[i] = min(d(p_i), trunc), trunc without a counting face */
void orc_df_values(const orc_scene* s, const float* pts, uint32_t n, float trunc, int brute, float* out)
{
    #pragma omp parallel for schedule(dynamic, 256)
    for (int64_t i = 0; i < (int64_t)n; i++) {
        float d;
        out[i] = orc_closest_point(s, pts + 3 * i, brute, &d, NULL, NULL, NULL) ? (d < trunc ? d : trunc) : trunc;
    }
}

/* out[i] = d(p_i), +inf without a counting face */
void orc_df_dist(const orc_scene* s, const float* pts, uint32_t n, int brute, float* out)
{
    #pragma omp parallel for schedule(dynamic, 256)
    for (int64_t i = 0; i < (int64_t)n; i++) {
        float d;
        out[i] = orc_closest_point(s, pts + 3 * i, brute, &d, NULL, NULL, NULL) ? d : INFINITY;
    }
}
