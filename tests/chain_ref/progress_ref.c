/* progress_ref.c -- TEST INFRASTRUCTURE ONLY: C restatement of MICPLocalizationNode::correctOnce's convergence progress
 * (rmcl_ros/src/nodes/micp_localization.cpp:988-1007), statement by statement in the reference's types, independent of the product's code.
 * T_onew_map = Tom * T_onew_oold (:972) comes from the oracle's Transform product (oracle/: orc_transform_mul).  Built by tests/chain_ref.py
 * with the oracle's flags (-ffp-contract=off: every operation rounded on its own, as in the reference's scalar code). */
#include <math.h>
#include <stdint.h>

typedef struct { float x, y, z, w; } ref_quat;
typedef struct { ref_quat R; float t[3]; uint32_t stamp; } ref_transform;     /* rm::Transform, 32 B */

double ref_micp_progress(const ref_transform* T_onew_map, uint32_t n_meas, uint32_t valid_measurements, int adaptive_max_dist)
{
    if (n_meas == 0 || !adaptive_max_dist) return 0.0;                                             /* :988-991 */
    const float trans_force = sqrtf(T_onew_map->t[0] * T_onew_map->t[0] + T_onew_map->t[1] * T_onew_map->t[1]
                                    + T_onew_map->t[2] * T_onew_map->t[2]);                        /* :994, Vector3::l2norm */
    const float trans_progress = 1.0 / exp(10.0 * trans_force);                                    /* :995 */
    const ref_quat qunit = {0.0f, 0.0f, 0.0f, 1.0f};                                               /* :997 */
    const float qscalar = T_onew_map->R.x * qunit.x + T_onew_map->R.y * qunit.y + T_onew_map->R.z * qunit.z
                          + T_onew_map->R.w * qunit.w;                                             /* :998, Quaternion::dot */
    const float rot_progress = qscalar * qscalar;                                                  /* :999 */
    const double match_ratio = (double)n_meas / (double)valid_measurements;                       /* :1001 */
    const float adaption_rate = trans_progress * rot_progress * match_ratio;                      /* :1002 */
    return adaption_rate;                                                                          /* :1006 */
}
