/* TEST INFRASTRUCTURE ONLY: reference for the surface constraint (b2_pf_project_to_surface; docs/RMCL.md:72, no reference implementation).
 *
 * The rule of SURVEY appendix F restated in C over the oracle's closest hit (orc_intersect: the hit definition of the product's tracer, by
 * brute force or through the oracle's own binary BVH): a ray from probe_above over the particle straight down, closest hit in (0, tfar];
 * ground iff the unit normal turned towards the ray origin has n.z >= cos_max; on ground the particle goes base_height over the hit, along z or,
 * with align, along n with the smallest rotation of its z-axis onto n; otherwise it keeps its pose and gets the likelihood {0, 0, 10000}.
 * The oracle's source is compiled into this file, so its vector and quaternion operations (rmagine's, in their order) are the ones used here.
 * Plain float ops, compiled with -ffp-contract=off: each is individually rounded. */
#include "../../oracle/oracle.c"

typedef struct { float probe_above, probe_below, base_height, max_slope; int32_t align; } ref_surface_config;

void orc_pf_surface(const orc_scene* s, uint32_t n, orc_transform* poses, orc_particle_attr* attrs, const ref_surface_config* c, int brute)
{
    const float cos_max = (float)cos((double)c->max_slope);
    const float tfar = c->probe_above + c->probe_below;
    #pragma omp parallel for schedule(dynamic, 64)
    for (int64_t i = 0; i < (int64_t)n; i++) {
        orc_transform T = poses[i];
        const float o[3] = {T.t.x, T.t.y, T.t.z + c->probe_above}, d[3] = {0.0f, 0.0f, -1.0f};
        float th = 0.0f, ng[3] = {0.0f, 0.0f, 0.0f};
        uint32_t face = 0;
        int ground = 0;
        orc_vec3 nv = v3(0.0f, 0.0f, 0.0f);
        const int finite_R = isfinite(T.R.x) && isfinite(T.R.y) && isfinite(T.R.z) && isfinite(T.R.w);
        if (finite_R && orc_intersect(s, o, d, tfar, brute, &th, &face, ng)) {       /* a non-finite position hits nothing */
            nv = v3_normalize(v3(ng[0], ng[1], ng[2]));
            if (nv.z < 0.0f) nv = v3_neg(nv);
            ground = nv.z >= cos_max;                                  /* false for a NaN normal */
        }
        if (!ground) {
            attrs[i].likelihood.mean = 0.0f; attrs[i].likelihood.sigma = 0.0f; attrs[i].likelihood.n_meas = 10000u;
            continue;
        }
        const orc_vec3 g = v3(T.t.x, T.t.y, o[2] - th);
        if (c->align) {
            const orc_vec3 a = q_rot(T.R, v3(0.0f, 0.0f, 1.0f));
            const float w = 1.0f + v3_dot(a, nv);
            orc_quat q;
            if (w < 1e-6f) {
                const orc_vec3 ex = q_rot(T.R, v3(1.0f, 0.0f, 0.0f));
                q.x = ex.x; q.y = ex.y; q.z = ex.z; q.w = 0.0f;
            } else {
                q.x = a.y * nv.z - a.z * nv.y; q.y = a.z * nv.x - a.x * nv.z; q.z = a.x * nv.y - a.y * nv.x; q.w = w;
            }
            T.R = q_normalize(q_mul(q_normalize(q), T.R));
            T.t = v3_add(g, v3_scale(nv, c->base_height));
        } else {
            T.t = v3(g.x, g.y, g.z + c->base_height);
        }
        poses[i] = T;                                                  /* the stamp is T's */
    }
}
