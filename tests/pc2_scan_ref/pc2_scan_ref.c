/* TEST INFRASTRUCTURE ONLY: reference for b2_rcc_set_cloud_spherical (PointCloud2 -> spherical scan + dataset).
 *
 * Pc2ToScanNode::convert (rmcl_ros/src/nodes/conversion/pc2_to_scan.cpp:105-213), fillEmpty (rmcl_ros/src/util/scan_operations.cpp:25-39)
 * and MICPSphericalSensorCUDA::unpackMessage (MICPSphericalSensorCUDA.cpp:176-235) restated in C, statement by statement.  The oracle's
 * source is compiled in, so `T * ps_s` is the oracle's Transform product.  Plain float ops, compiled with -ffp-contract=off: each is
 * individually rounded, as the reference's.  `flags` picks the elevation rule and the atan2 precision:
 *   0                    the product's rule: phi = atan2(z, sqrt(x^2 + y^2)), both angles FP64 atan2 rounded to float (SURVEY D21)
 *   REF_ELEV_3D          the reference's rule: phi = atan2(z, |p|)
 *   REF_ATAN2F           the angles with float atan2f (the reference's float path); with the product's rule sqrt(x^2 + y^2) is sqrtf
 * Points are read at row * row_step + col * point_step (D22; identical to the reference's i * point_step for dense clouds). */
#include "../../oracle/oracle.c"

#include <limits.h>

#define REF_ELEV_3D 1
#define REF_ATAN2F  2

/* b2_spherical_model / rmcl_msgs ScanInfo as converted by rmcl::convert (conversions.cpp:22-34) */
typedef struct { float phi_min, phi_inc; uint32_t phi_size; float theta_min, theta_inc; uint32_t theta_size; float range_min, range_max; } ref_spherical_model;

/* rm::SphericalModel::getDirection(vid, hid) as the library's set_model_spherical evaluates it on the host (libm cosf / sinf) */
void ref_spherical_dirs(const ref_spherical_model* m, float* dirs)
{
    for (uint32_t vid = 0; vid < m->phi_size; vid++) {
        const float phi = m->phi_min + (float)vid * m->phi_inc;
        const float cp = cosf(phi), sp = sinf(phi);
        for (uint32_t hid = 0; hid < m->theta_size; hid++) {
            const float theta = m->theta_min + (float)hid * m->theta_inc;
            float* d = &dirs[3 * ((size_t)vid * m->theta_size + hid)];
            d[0] = cp * cosf(theta); d[1] = cp * sinf(theta); d[2] = sp;
        }
    }
}

/* int id = ((angle - min) / inc) + 0.5 (:195-196): float subtraction and division, double + 0.5, truncation.  A double outside the range
 * of int (or NaN) makes the conversion undefined in C++; it is reported as outside the model, which is what the id test would say of any
 * value the conversion could give there except INT_MIN's neighbours.  A dimension of size 1 with increment 0 (0 / 0 in the reference:
 * D24) gives 0. */
static int bin_id(float a, float mn, float inc, uint32_t size, int* id)
{
    if (inc == 0.0f && size == 1) { *id = 0; return 1; }
    const double b = ((a - mn) / inc) + 0.5;
    if (!(b > (double)INT_MIN - 1.0 && b < (double)INT_MAX + 1.0)) return 0;
    *id = (int)b;
    return *id >= 0 && *id < (int)size;                    /* :198-199 */
}

/* data: the cloud's bytes; off: byte offsets of x, y, z; f64: FLOAT64 fields.  Out: ranges, points, mask of the model's cells; per point
 * (may be null): the cell it writes (a later point may overwrite it) or -1, and its float theta and phi (0 for skipped points). */
void ref_pc2_to_scan(const uint8_t* data, uint32_t width, uint32_t height, uint32_t point_step, uint64_t row_step, const uint32_t off[3], int f64,
                     const orc_transform* T, const ref_spherical_model* m, int flags, float* ranges, float* pts, uint8_t* mask,
                     int64_t* point_cell, float* point_theta, float* point_phi)
{
    const size_t n_cells = (size_t)m->phi_size * m->theta_size;
    for (size_t k = 0; k < n_cells; k++) ranges[k] = m->range_max + 1.0;       /* fillEmpty (scan_operations.cpp:35) */
    const size_t n_points = (size_t)width * height;
    for (size_t i = 0; i < n_points; i++) {                                     /* :160 */
        const size_t row = i / width, col = i - row * width;
        const uint8_t* data_ptr = data + row * row_step + col * point_step;    /* :162 (D22) */
        float x, y, z;
        if (!f64) {
            memcpy(&x, data_ptr + off[0], 4); memcpy(&y, data_ptr + off[1], 4); memcpy(&z, data_ptr + off[2], 4);
        } else {
            double dx, dy, dz;
            memcpy(&dx, data_ptr + off[0], 8); memcpy(&dy, data_ptr + off[1], 8); memcpy(&dz, data_ptr + off[2], 8);
            x = (float)dx; y = (float)dy; z = (float)dz;
        }
        if (point_cell) { point_cell[i] = -1; point_theta[i] = 0.0f; point_phi[i] = 0.0f; }
        if (isfinite(x) && isfinite(y) && isfinite(z)) {                       /* :186 */
            const float ps_s[3] = {x, y, z};
            float ps[3];
            orc_transform_point(T, ps_s, ps);                                   /* :188-189 */
            const float range_est = sqrtf(ps[0] * ps[0] + ps[1] * ps[1] + ps[2] * ps[2]);          /* :191, rm::Vector::l2norm */
            float theta_est, phi_est;
            if (flags & REF_ATAN2F) {
                theta_est = atan2f(ps[1], ps[0]);
                phi_est = (flags & REF_ELEV_3D) ? atan2f(ps[2], range_est) : atan2f(ps[2], sqrtf(ps[0] * ps[0] + ps[1] * ps[1]));
            } else {
                const double px = ps[0], py = ps[1], pz = ps[2];
                theta_est = (float)atan2(py, px);
                phi_est = (flags & REF_ELEV_3D) ? (float)atan2(pz, (double)range_est) : (float)atan2(pz, sqrt(px * px + py * py));
            }
            if (point_cell) { point_theta[i] = theta_est; point_phi[i] = phi_est; }
            int phi_id, theta_id;
            const int in_phi = bin_id(phi_est, m->phi_min, m->phi_inc, m->phi_size, &phi_id);
            const int in_theta = bin_id(theta_est, m->theta_min, m->theta_inc, m->theta_size, &theta_id);
            if (in_phi && in_theta) {
                if (range_est >= m->range_min && range_est <= m->range_max) {  /* model.range.inside */
                    const size_t p_id = (size_t)phi_id * m->theta_size + (size_t)theta_id;         /* getBufferId(phi_id, theta_id) */
                    ranges[p_id] = range_est;
                    if (point_cell) point_cell[i] = (int64_t)p_id;
                }
            }
        }
    }
    /* MICPSphericalSensorCUDA::unpackMessage (:202-222): point = dir * range + orig (orig 0), mask = range in [min, max] */
    float* dirs = (float*)malloc(sizeof(float) * 3 * (n_cells ? n_cells : 1));
    ref_spherical_dirs(m, dirs);
    for (uint32_t vid = 0; vid < m->phi_size; vid++)
        for (uint32_t hid = 0; hid < m->theta_size; hid++) {
            const size_t loc_id = (size_t)vid * m->theta_size + hid;
            const float real_range = ranges[loc_id];
            for (int c = 0; c < 3; c++) pts[3 * loc_id + c] = dirs[3 * loc_id + c] * real_range + 0.0f;
            mask[loc_id] = (real_range < m->range_min || real_range > m->range_max) ? 0 : 1;
        }
    free(dirs);
}
