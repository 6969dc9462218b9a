// cov_emul.cu -- TEST HARNESS ONLY: the product's pieces of b2_micp_pose_covariance (rmcl_b200/csrc/kernels.cuh: micp_cov_finalize, the
// pre-transform and the P2L gate the kernel applies) compiled for the CPU, so that they can be compared with numpy in a container without a GPU.
// Included into the emulator library (tests/emul/emul.cu).

EMUL_API void emul_micp_cov_finalize(const double* sums, const double* weights, uint32_t n_sensors, double tau, double degenerate_variance,
                                     b2_micp_covariance* out)
{
    micp_cov_finalize(sums, weights, n_sensors, tau, degenerate_variance, out);
}
// T_snew_sold = Tso * T_onew_oold * Tos with Tos = Tbo * Tsb, as b2_micp_pose_covariance and the ICP loop compose it
EMUL_API void emul_micp_cov_pretransform(const b2_transform* Tbo, const b2_transform* Tsb, const b2_transform* T_onew_oold, b2_transform* out)
{
    const Tf Tos = tf_mul(tf_from_pod(*Tbo), tf_from_pod(*Tsb));
    tf_store(out, tf_mul(tf_mul(tf_inv(Tos), tf_from_pod(*T_onew_oold)), Tos));
}
// the accepted pairs (dataset mask, model hit, p2l_pair) and their residuals r = (I - Tpre d) . N
EMUL_API void emul_micp_cov_gate(const b2_transform* Tpre, uint32_t n, const float* d, const uint8_t* dmask, const float* I, const float* N,
                                 const uint8_t* hits, float max_dist, uint8_t* ok, float* r)
{
    const Tf T = tf_from_pod(*Tpre);
    for (uint32_t i = 0; i < n; i++) {
        const V3 dd = mk3(d[3 * i], d[3 * i + 1], d[3 * i + 2]), II = mk3(I[3 * i], I[3 * i + 1], I[3 * i + 2]), NN = mk3(N[3 * i], N[3 * i + 1], N[3 * i + 2]);
        V3 D, M;
        ok[i] = (dmask[i] > 0) && (hits[i] > 0) && p2l_pair(T, dd, II, NN, max_dist, D, M);
        r[i] = ok[i] ? v_dot(v_sub(II, D), NN) : 0.0f;
    }
}
