/* TEST INFRASTRUCTURE ONLY: reference for the recovery's injection (b2_pf_recovery_inject; Augmented MCL, no reference implementation).
 *
 * Decision, candidates and acceptance restated in C: particle g is chosen iff (double)word0 of Philox4x32-10 with counter (g, 7, step, 0)
 * times 2^-32 is below p; try t maps words 0-3 of block 1 + 2t and 0-1 of block 2 + 2t into the box as the uniform initialiser does
 * (pf_init_ref.c); without a surface the first candidate is taken, with one a candidate is taken iff the surface rule of pf_surface_ref.c
 * (over the oracle's closest hit) finds ground under it, as that rule moved it.  A taken candidate gets stamp 0 and the attributes {0, 0, 0},
 * state_sigma 0; a particle whose tries all fail is left as it was.  The surface rule and the oracle (Philox, euler_to_quat) are compiled
 * into this file, not copied.  Plain float ops, compiled with -ffp-contract=off: each is individually rounded. */
#include "../pf_surface_ref/pf_surface_ref.c"

#define ORC_RECOVERY_TAG 7u

static void recovery_words(uint64_t seed, uint32_t g, uint32_t step, uint32_t block, uint32_t r[4])
{
    const uint32_t key[2] = {(uint32_t)seed, (uint32_t)(seed >> 32)}, ctr[4] = {g, ORC_RECOVERY_TAG, step, block};
    orc_philox4x32_10(ctr, key, r);
}

/* s == NULL: no surface.  counts[0] += replaced, counts[1] += failed */
void orc_pf_recovery(const orc_scene* s, const ref_surface_config* c, uint32_t first, uint32_t n, double p, const float lo[6], const float hi[6],
                     uint32_t max_tries, uint64_t seed, uint32_t step, orc_transform* poses, orc_particle_attr* attrs, uint64_t counts[2])
{
    uint64_t n_rep = 0, n_fail = 0;
    #pragma omp parallel for schedule(dynamic, 256) reduction(+ : n_rep, n_fail)
    for (int64_t i = 0; i < (int64_t)n; i++) {
        const uint32_t g = first + (uint32_t)i;
        uint32_t r[8];
        recovery_words(seed, g, step, 0u, r);
        if (!((double)r[0] * 0x1p-32 < p)) continue;
        int taken = 0;
        for (uint32_t t = 0; t < max_tries && !taken; t++) {
            recovery_words(seed, g, step, 1u + 2u * t, r);
            recovery_words(seed, g, step, 2u + 2u * t, r + 4);
            float v[6];
            for (int k = 0; k < 6; k++) {
                const float u = (float)(r[k] >> 8) * 5.9604644775390625e-08f;
                v[k] = fminf(lo[k] + (hi[k] - lo[k]) * u, hi[k]);
            }
            orc_transform T;
            T.t = v3(v[0], v[1], v[2]); T.R = euler_to_quat(v[3], v[4], v[5]); T.stamp = 0;
            if (s) {
                orc_particle_attr a;
                memset(&a, 0, sizeof a);
                orc_pf_surface(s, 1, &T, &a, c, 0);
                if (a.likelihood.n_meas == 10000u) continue;                 /* the rule's mark: no ground under the candidate */
            }
            poses[i] = T;
            memset(attrs + i, 0, sizeof(orc_particle_attr));
            taken = 1;
        }
        if (taken) n_rep++; else n_fail++;
    }
    counts[0] += n_rep; counts[1] += n_fail;
}
