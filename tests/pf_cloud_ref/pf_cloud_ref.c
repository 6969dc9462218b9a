/* TEST INFRASTRUCTURE ONLY: reference for the sensor update's beam sampling (b2_pf_sample_cloud).
 *
 * PCDSensorUpdaterOptix::update's sampling loop (rmcl_ros/src/rmcl/PCDSensorUpdaterOptix.cpp:227-311) restated in C with the draws of the
 * library: sample k makes up to 100 tries (max_tries, :267); try t reads point raw % n_points with raw = word t % 4 of Philox4x32-10, counter
 * (k, 3, step, t / 4), key = seed; a try is valid iff x, y and z are not NaN (:278); a valid sample is orig 0, range |p|, dir p / range
 * (:291-293), cov 0.1 I (:296-301); a NaN direction component is stored as 0x7fffffff.  Sampling stops at the 10th sample whose tries all
 * failed (max_invalids, :264-287).  Point i = row * width + col is read at row * row_step + col * point_step through the x, y, z offsets,
 * FLOAT32 as is, FLOAT64 narrowed to float.  The oracle's source is compiled into this file, so its Philox is the one used here.  Plain float
 * ops, compiled with -ffp-contract=off: each is individually rounded. */
#include "../../oracle/oracle.c"

#define ORC_BEAM_TAG 3u
#define ORC_BEAM_TRIES 100
#define ORC_BEAM_MAX_INVALIDS 10

static float read_coord(const uint8_t* p, int f64)
{
    if (f64) { double d; memcpy(&d, p, 8); return (float)d; }
    float f; memcpy(&f, p, 4); return f;
}

static float nan_canonical(float v)
{
    if (v == v) return v;
    const uint32_t u = 0x7fffffffu;
    memcpy(&v, &u, 4);
    return v;
}

/* sample k: 1 and *m from its first valid try, or 0 when all 100 tries read a NaN coordinate; width * height > 0 */
int ref_pf_sample_one(const uint8_t* cloud, uint32_t width, uint32_t height, uint64_t row_step, uint32_t point_step, const uint32_t off[3], int f64,
                      uint64_t seed, uint32_t step, uint32_t k, orc_range_meas* m)
{
    const uint32_t n_points = (uint32_t)((uint64_t)width * height);
    const uint32_t key[2] = {(uint32_t)seed, (uint32_t)(seed >> 32)};
    uint32_t words[4];
    for (uint32_t t = 0; t < ORC_BEAM_TRIES; t++) {
        if (t % 4 == 0) {
            const uint32_t ctr[4] = {k, ORC_BEAM_TAG, step, t / 4};
            orc_philox4x32_10(ctr, key, words);
        }
        const uint32_t i = words[t % 4] % n_points;
        const uint8_t* p = cloud + (uint64_t)(i / width) * row_step + (uint64_t)(i % width) * point_step;
        const float x = read_coord(p + off[0], f64), y = read_coord(p + off[1], f64), z = read_coord(p + off[2], f64);
        if (!(x == x && y == y && z == z)) continue;
        const float range = sqrtf(x * x + y * y + z * z);
        m->orig = v3(0.0f, 0.0f, 0.0f);
        m->dir = v3(nan_canonical(x / range), nan_canonical(y / range), nan_canonical(z / range));
        m->range = range;
        memset(&m->cov, 0, sizeof(m->cov));
        m->cov.m[0] = m->cov.m[4] = m->cov.m[8] = 0.1f;
        return 1;
    }
    return 0;
}

/* the beams of one update in sample order -> their count; beams has room for n_samples */
uint32_t ref_pf_sample_cloud(const uint8_t* cloud, uint32_t width, uint32_t height, uint64_t row_step, uint32_t point_step, const uint32_t off[3], int f64,
                             uint32_t n_samples, uint64_t seed, uint32_t step, orc_range_meas* beams)
{
    if ((uint64_t)width * height == 0) return 0;
    uint32_t n = 0;
    int max_invalids = ORC_BEAM_MAX_INVALIDS;
    for (uint32_t k = 0; k < n_samples && max_invalids > 0; k++) {
        orc_range_meas m;
        if (ref_pf_sample_one(cloud, width, height, row_step, point_step, off, f64, seed, step, k, &m)) beams[n++] = m;
        else max_invalids--;
    }
    return n;
}
