// estimate_emul.cu -- TEST HARNESS ONLY: the product's building blocks of the pose estimate (rmcl_b200/csrc/kernels.cuh: sym4_top_eigvec, the
// Markley mean's 4x4 eigen solver, and pf_deviation, the 6-vector of a particle about the mean) compiled for the CPU, so that they can be
// compared with numpy in a container without a GPU.  Built by tests/pf_estimate_ref.py with the flags of tests/chain_ref (host code with
// -ffp-contract=off: plain float ops rounded like __fmul_rn / __fadd_rn).
#include "../../rmcl_b200/csrc/kernels.cuh"

extern "C" {
__attribute__((visibility("default"))) void emul_sym4_top_eigvec(const double* A16, double* v4, double* lambda) { sym4_top_eigvec(A16, v4, lambda); }
__attribute__((visibility("default"))) void emul_pf_deviation(const b2_transform* Tbm, const b2_transform* poses, uint32_t n, float* v6)
{
    const Tf Tinv = tf_inv(tf_from_pod(*Tbm));
    for (uint32_t i = 0; i < n; i++) pf_deviation(Tinv, tf_from_pod(poses[i]), v6 + 6 * (size_t)i);
}
}
