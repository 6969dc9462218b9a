// stein_slice_emul.cu -- TEST HARNESS ONLY: one rank's session of the sharded Stein steps (b2_pf_stein_slice_*, SURVEY L14) on the CPU,
// launch by launch, over the product's functions (rmcl_b200/csrc/kernels.cuh).  It is the emulator library (tests/emul/emul.cu, whose
// emul_stein_bandwidth is the whole-set bandwidth and whose emul_stein_update is the whole-set reference) plus the slice score and the
// slice move below, built into a library of its own by tests/pf_stein_sharded_ref.py.
#include "../emul/emul.cu"

// The score of J's references [j_first, j_first + j_count), as k_pf_stein_score with its j_first offset: snap[r - j_first]
EMUL_API void emul_stein_slice_score(const float* lo, const float* hi, float h, float trunc, const uint32_t* index, const float* bricks, const b2_transform* poses_all,
                                     uint32_t n_all, uint32_t j_first, uint32_t j_count, uint32_t n_ref, uint64_t seed, uint32_t step, uint32_t it,
                                     const b2_transform* Tsb_val, const b2_range_meas* beams, uint32_t n_beams, float dist_sigma, float w_rand, SteinRef* snap)
{
    const DfieldView f = field_of(lo, hi, h, trunc, index, bricks);
    const Tf Tsb = tf_from_pod(*Tsb_val);
    const float sigma2 = mul(dist_sigma, dist_sigma);
    #pragma omp parallel for schedule(dynamic, 16)
    for (int64_t r = 0; r < (int64_t)j_count; r++) {
        std::vector<float> terms(3 * (size_t)n_beams);
        const Tf T = tf_from_pod(poses_all[stein_ref_index(j_first + (uint32_t)r, n_all, n_ref, seed, step, it)]);
        const Tf Tsm = tf_mul(T, Tsb);
        for (uint32_t b = 0; b < n_beams; b++) {
            const b2_range_meas& q = beams[b];
            const PfBeam pb{q.orig.x, q.orig.y, q.orig.z, q.dir.x, q.dir.y, q.dir.z, q.range, b};
            stein_beam_term(f, Tsm, T.t, pb, sigma2, w_rand, terms.data() + 3 * (size_t)b);
        }
        snap[r] = stein_ref_entry(T, terms.data(), n_beams);
    }
}
// The move of the slice [first, first + n_local) of poses_all into out (n_local; out == poses_all + first is in place), as k_pf_stein_move
// with first and its output pointer: v (n_local x 3) the slice's RMSProp state; rec's n_blocked is added to, its step count and sums set
// (the step sums in est_grid_reduce's order over the slice's blocks, grid_reduce of stein_emul.cu).  An empty slice launches nothing on
// the device, so it leaves rec.
EMUL_API void emul_stein_slice_move(void* scene, const b2_transform* poses_all, uint32_t first, uint32_t n_local, const SteinRef* snap, uint32_t m, uint32_t it,
                                    float step_t, float step_r, float* v, const float* h, b2_transform* out, b2_stein_slice_result* rec)
{
    if (n_local == 0) return;
    const BvhView bvh = view_of(scene);
    float ih2[3];
    stein_inv_h2(h, ih2);
    std::vector<double> per((size_t)n_local * B2_STEIN_NMV, 0.0);
    uint64_t blocked = 0;
    #pragma omp parallel for schedule(static) reduction(+ : blocked)
    for (int64_t i = 0; i < (int64_t)n_local; i++) {
        const b2_transform* src = poses_all + first + i;
        const Tf T = tf_from_pod(*src);
        if (out + i != src) out[i] = *src;
        float ci[3];
        stein_chart(T, ci);
        if (!stein_finite3(ci)) continue;
        float a[3] = {0.0f, 0.0f, 0.0f};
        for (uint32_t j = 0; j < m; j++) if (snap[j].x == snap[j].x) stein_pair(ci, snap[j], ih2, a);
        blocked += stein_move_one(bvh, out + i, T, v + 3 * i, a, m, it, step_t, step_r, per.data() + (size_t)i * B2_STEIN_NMV);
    }
    double tot[B2_STEIN_NMV];
    grid_reduce(per, B2_STEIN_NMV, n_local, tot);
    rec->n_blocked += (uint32_t)blocked;
    rec->n_steps = (uint32_t)tot[0];
    rec->sum_step_t2 = tot[1];
    rec->sum_step_r2 = tot[2];
}
