/*
 * rmcl_b200.h -- C ABI of the H100-native ray-casting-correspondence library (librmcl_b200.so).
 *
 * This is the drop-in boundary for ONE hot path of uos/rmcl (SURVEY.md section 8b): plain pointers and sizes, no C++
 * or torch types.  Every entry point cites the reference interface it replaces (paths relative to the rmcl repo).
 * The reference-side bindings a maintainer would add are shown in INTEGRATION.md; the C++ shim classes with the
 * reference's names live in include/rmcl_b200/ (C++ headers).
 *
 * Conventions
 *  - every function returns B2_OK (0) or a negative B2_ERR_*; b2_last_error() gives the thread-local message.
 *  - nothing here falls back to the CPU: if no CUDA device / kernel image is usable the call fails with B2_ERR_CUDA.
 *  - "device pointer" arguments are CUDA device addresses on the mesh's device; all work is enqueued on the handle's
 *    stream (b2_*_set_stream, default: the legacy default stream).  Calls that return data to HOST memory synchronise
 *    that stream; calls that take/return only device pointers do not.
 *  - layouts are byte-compatible with rmagine / rmcl (SURVEY.md Appendix B).
 */
#ifndef RMCL_B200_H
#define RMCL_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(_WIN32)
#define B2_API
#else
#define B2_API __attribute__((visibility("default")))
#endif

/* ---------------------------------------------------------------- POD types ---------------------------------- */
typedef struct { float x, y, z; } b2_vec3;                                   /* rmagine::Vector3f   (12 B) */
typedef struct { float x, y, z, w; } b2_quat;                                /* rmagine::Quaternion (16 B) */
typedef struct { b2_quat R; b2_vec3 t; uint32_t stamp; } b2_transform;       /* rmagine::Transform  (32 B) */
typedef struct { float m[9]; } b2_mat3;                                      /* rmagine::Matrix3x3, column-major */
typedef struct { b2_vec3 dataset_mean, model_mean; b2_mat3 covariance; uint32_t n_meas; } b2_cross_stats; /* rmagine::CrossStatistics (64 B) */
typedef struct { float mean, sigma; uint32_t n_meas; } b2_gaussian1d;        /* rmagine::Gaussian1D (12 B) */
typedef struct { b2_gaussian1d likelihood; float state_sigma[6]; } b2_particle_attr;  /* rmcl::ParticleAttributes, rmcl_ros/include/rmcl_ros/rmcl/ParticleAttributes.hpp:18-32 (36 B) */
typedef struct { b2_vec3 orig, dir; float range; b2_mat3 cov; } b2_range_meas;         /* rmcl::RangeMeasurement,  rmcl_ros/include/rmcl_ros/rmcl/RangeMeasurement.hpp:10-21 (64 B) */

/* rmagine::SphericalModel as filled at rmcl_ros/src/util/conversions.cpp:22-34 */
typedef struct { float phi_min, phi_inc; uint32_t phi_size; float theta_min, theta_inc; uint32_t theta_size; float range_min, range_max; } b2_spherical_model;
/* rmagine::PinholeModel as filled at rmcl_ros/src/util/conversions.cpp:48-60 */
typedef struct { uint32_t width, height; float fx, fy, cx, cy; float range_min, range_max; } b2_pinhole_model;

/* PCDSensorUpdaterEmbree config, rmcl_ros/src/rmcl/PCDSensorUpdaterEmbree.cpp:122-134 (defaults in comments) */
typedef struct {
    float dist_sigma;                 /* 2.0   */
    float real_hit_sim_miss_error;    /* 100.0 */
    float real_miss_sim_hit_error;    /* 100.0 */
    float real_miss_sim_miss_error;   /* 0.0   */
    float range_min, range_max;       /* sensor_range 0.05 .. 80.0 */
    int   ng_mode;                    /* 0: raw un-normalised geometric normal (Embree path, :57-68); 1: unit normal (OptiX path, BeamEvaluateProgram.cu:104-113) */
    int   correspondence_type;        /* 0: ray casting (evaluate_rcc, :18-86); 1: closest point (evaluate_cpc, :88-95; selected at :219-222) */
} b2_pf_params;

typedef struct {
    uint32_t n_faces, n_vertices, n_nodes, n_leaf_tris, max_depth;
    uint64_t bvh_bytes;               /* nodes + leaf triangle records resident in HBM */
    float    build_ms;                /* wall time of b2_mesh_create (host build + upload, or device build) */
    int      device;
    int      build_mode;
    float    sah_cost;
} b2_mesh_info;

typedef struct b2_mesh b2_mesh;       /* immutable map: triangle mesh + in-HBM BVH.  Stands in for rmagine::EmbreeMap / OptixMap */
typedef struct b2_rcc  b2_rcc;        /* one ray-casting-correspondence set == one rmcl::RCC..{Spherical,Pinhole,O1Dn,OnDn} object */
typedef struct b2_pf   b2_pf;         /* one particle-filter sensor updater == rmcl::PCDSensorUpdater{Embree,Optix} */

enum {
    B2_OK = 0,
    B2_ERR_INVALID = -1,      /* bad argument / call order (e.g. find before set_model) */
    B2_ERR_CUDA = -2,         /* CUDA runtime error (message in b2_last_error) */
    B2_ERR_NO_MAP = -3,       /* empty mesh: mirrors "NO MAP"/"EMPTY MAP" of PCDSensorUpdaterOptix.cpp:179-192 */
    B2_ERR_OOM = -4,
    B2_ERR_UNSUPPORTED = -5
};
enum { B2_BUILD_HOST_SAH = 0, B2_BUILD_DEVICE_LBVH = 1 };
/* correspondence type of a b2_rcc handle: ray casting (RCCEmbree*, default) or closest point (CPCEmbree) */
enum { B2_CORR_RCC = 0, B2_CORR_CPC = 1 };

B2_API const char* b2_last_error(void);
B2_API int         b2_version(void);
B2_API int         b2_device_count(int* n);

/* ---------------------------------------------------------------- map ---------------------------------------- */
/* replaces rm::import_embree_map + Embree scene commit (rmcl_ros/src/nodes/micp_localization.cpp:188,
 * rmcl_ros/src/rmcl/PCDSensorUpdaterEmbree.cpp:158): vertices/faces in HOST memory -> BVH resident in HBM of `device`.
 * Every vertex coordinate must be finite and at most 2^62 in magnitude (B2_ERR_INVALID otherwise): box extents then stay below 2^63, so the
 * builders' box half-areas (<= 3 * 2^126 < FLT_MAX), box centres and octant slot costs are finite.  Beyond that they overflow to inf / NaN,
 * and the tree would lose or misfile triangles; metric maps are many orders of magnitude smaller. */
B2_API int b2_mesh_create(const float* verts_xyz, uint32_t n_vertices, const uint32_t* faces_ijk, uint32_t n_faces,
                          int device, int build_mode, b2_mesh** out);
/* rm::import_embree_map(file) (rmcl_ros/src/nodes/micp_localization.cpp:188, rmcl_ros/src/rmcl/PCDSensorUpdaterEmbree.cpp:158): mesh file ->
 * map.  Self-contained readers (no assimp) for Stanford PLY (ascii / binary_little_endian), Wavefront OBJ and COLLADA .dae (geometry library +
 * visual-scene node transforms; the format of the reference's example maps, docs/MICPL.md:46-49); polygons are fan-triangulated. */
B2_API int b2_mesh_create_from_file(const char* path, int device, int build_mode, b2_mesh** out);
/* the import step alone (host only, no device needed): malloc'ed vertex / face arrays, released with b2_mesh_file_free */
B2_API int b2_mesh_file_load(const char* path, float** verts_xyz, uint32_t* nv, uint32_t** faces_ijk, uint32_t* nf);
B2_API void b2_mesh_file_free(float* verts_xyz, uint32_t* faces_ijk);
/* Dynamic maps (SURVEY.md 8f1): the vertices moved, faces unchanged -> refit the resident BVH instead of rebuilding it (the reference
 * re-commits its Embree scene and flags dependants `outdated`, Correspondences.hpp:26-31).  Maps built with B2_BUILD_DEVICE_LBVH only; the call
 * synchronises the device first, so no handle may be tracing concurrently from another thread.  Results afterwards equal a fresh build's.
 * Host vertices obey b2_mesh_create's bound (finite, |coordinate| <= 2^62); device vertices are not inspected. */
B2_API int b2_mesh_refit(b2_mesh* m, const float* verts_xyz, uint32_t nv, int src_is_device);
/* BVH blob (SURVEY.md 8b): the built map as one host buffer (header + nodes + leaf triangle records), so that a map is built once and
 * shipped to the other ranks (broadcast) or cached on disk; b2_mesh_create_from_blob validates the header and every index before uploading. */
B2_API int b2_mesh_blob_size(const b2_mesh* m, uint64_t* bytes);
B2_API int b2_mesh_export_blob(const b2_mesh* m, void* dst_host, uint64_t capacity);
B2_API int b2_mesh_create_from_blob(const void* blob_host, uint64_t bytes, int device, b2_mesh** out);
/* Drops the creator's reference.  b2_rcc / b2_pf handles created on the map hold their own references (the reference shares its map through
 * rm::EmbreeMapPtr, a shared_ptr, micp_localization.cpp:545), so map and handles may be destroyed in any order. */
B2_API int b2_mesh_destroy(b2_mesh* m);
B2_API int b2_mesh_get_info(const b2_mesh* m, b2_mesh_info* info);
/* closest hit for arbitrary rays (host arrays in, host arrays out): t in (0,tfar], tie -> smaller face id.
 * Replaces rtcIntersect1 as used at rmcl_ros/src/rmcl/PCDSensorUpdaterEmbree.cpp:30-47. Any output may be NULL. */
B2_API int b2_mesh_intersect(const b2_mesh* m, const float* origs_xyz, const float* dirs_xyz, uint32_t n, float tfar,
                             float* t_out, uint32_t* face_out, float* ng_out_xyz, uint8_t* hit_out);
/* traversal counters of the same rays (instrumented build of the same kernel): mean nodes visited / triangles tested per ray */
B2_API int b2_mesh_intersect_stats(const b2_mesh* m, const float* origs_xyz, const float* dirs_xyz, uint32_t n, float tfar,
                                   double* mean_nodes, double* mean_tris);

/* ---------------------------------------------------------------- MICP-L: RCC ------------------------------ */
/* ctor(map): rmcl/include/rmcl/registration/RCCEmbree.hpp:25-26 */
B2_API int b2_rcc_create(b2_mesh* map, b2_rcc** out);
B2_API int b2_rcc_destroy(b2_rcc* h);
B2_API int b2_rcc_set_stream(b2_rcc* h, void* cuda_stream);
/* Correspondences_::setTsb, rmcl/include/rmcl/registration/Correspondences.hpp:33-36 */
B2_API int b2_rcc_set_tsb(b2_rcc* h, const b2_transform* Tsb);
/* ModelSetter<ModelT>::setModel, rmcl/src/rmcl/registration/RCCEmbree.cpp:21-24,53-56,84-87,116-119 */
B2_API int b2_rcc_set_model_spherical(b2_rcc* h, const b2_spherical_model* model);
B2_API int b2_rcc_set_model_pinhole(b2_rcc* h, const b2_pinhole_model* model);
B2_API int b2_rcc_set_model_o1dn(b2_rcc* h, uint32_t width, uint32_t height, const float orig_xyz[3], const float* dirs_xyz, float range_min, float range_max);
B2_API int b2_rcc_set_model_ondn(b2_rcc* h, uint32_t width, uint32_t height, const float* origs_xyz, const float* dirs_xyz, float range_min, float range_max);
/* public fields params.max_dist / adaptive_max_dist_min, Correspondences.hpp:22-23 */
B2_API int b2_rcc_set_params(b2_rcc* h, float max_dist, float adaptive_max_dist_min);
/* public field dataset (points + mask), Correspondences.hpp:24; src_is_device != 0: pointers are device addresses */
B2_API int b2_rcc_set_dataset(b2_rcc* h, const float* points_xyz, const uint8_t* mask, uint32_t n, int src_is_device);
/* The same two members as CALLER-OWNED device memory, nothing copied: a subclass of rmcl::Correspondences_<rm::VRAM_CUDA> keeps the reference's public
 * `dataset` (rm::PointCloud_<VRAM_CUDA>, Correspondences.hpp:24) and protected `model_buffers_` (Correspondences.hpp:81-85) and binds their device
 * pointers here; find() then writes points / normals / hits straight into the bound buffers (capacity entries; grow and re-bind like
 * RCCOptix.cpp:36-40), the reductions read the bound dataset.  b2_rcc_set_dataset / set_ranges / correct_once_ranges switch back to the handle's
 * own dataset buffers; binding with capacity 0 unbinds the model buffers. */
B2_API int b2_rcc_bind_dataset(b2_rcc* h, const float* points_xyz_dev, const uint8_t* mask_dev, uint32_t n);
B2_API int b2_rcc_bind_model_buffers(b2_rcc* h, float* points_xyz_dev, float* normals_xyz_dev, uint8_t* hits_dev, uint32_t capacity);
/* MICP..Sensor..::unpackMessage (rmcl_ros/src/micpl/MICPSphericalSensorCPU.cpp:181-233) on the device: dataset = dir*range (+orig),
 * mask = range in [range.min, range.max].  Also the v1 setInputData(ranges) (lidar_corrector_embree_benchmark.cpp:118). */
B2_API int b2_rcc_set_ranges(b2_rcc* h, const float* ranges, uint32_t n, int src_is_device);
/* An organised sensor_msgs/PointCloud2 as the O1Dn sensor's scan.  b2_cloud_layout carries the message's geometry; the lookup of the fields
 * named x, y and z stays with the caller (rmcl_msgs_adapters.hpp does it), B2_CLOUD_NO_FIELD marks one that is missing.  datatype is the
 * PointField datatype of x, which decides how all three are read (7 FLOAT32, 8 FLOAT64 narrowed to float). */
#define B2_CLOUD_NO_FIELD 0xffffffffu
typedef struct {
    uint32_t width, height, point_step, row_step;
    uint32_t offset_x, offset_y, offset_z;
    uint8_t  datatype, is_bigendian, pad[2];
} b2_cloud_layout;                                                            /* 32 B */
/* the parameters of pc2_to_o1dn (rmcl_ros/src/nodes/conversion/pc2_to_o1dn.cpp:48-77, FilterOptions2D, scan_operations.h:59-66) */
typedef struct {
    uint32_t height_skip_begin, height_skip_end, height_increment;
    uint32_t width_skip_begin, width_skip_end, width_increment;
    float    range_min, range_max;
} b2_o1dn_cloud_filter;                                                       /* 32 B */
/* Pc2ToO1DnNode::convert + MICPO1DnSensor*::unpackMessage + setModel on the device: estimateModelAndData (rmcl_ros/src/util/conversions.cpp:869-1073),
 * filter (rmcl_ros/src/util/scan_operations.cpp:41-143), then the model and dataset of MICPO1DnSensorCUDA.cpp:142-148,171-230, in one kernel.
 * Output ray (i, j), i < H = (height - h_skip_begin - h_skip_end) / h_increment, j < W likewise, reads the point at byte
 * (i*h_inc + h_skip_begin) * row_step + (j*w_inc + w_skip_begin) * point_step.  A finite point p gives range = |p| and dir = p / range; any other
 * gives dir 0 and range 0 (valid when range_min <= 0).  A finite (0,0,0) gives NaN directions, as in the reference.  The model becomes O1Dn
 * W x H, orig 0, [range_min, range_max]; the dataset is point = dir*range, mask = range in [range_min, range_max], as b2_rcc_set_ranges.  A field
 * named `mask` is not read (the reference would store it as the range).  src_is_device != 0: `data` is a device address, read in place (it
 * must stay valid until the handle's stream has run the kernel); else the bytes up to the last point read are uploaded and the call
 * synchronises.  When the handle's previous model came from this call with the same W x H, find's tile schedule is kept; any other model
 * resets it.  Refused (B2_ERR_INVALID, no launch, handle unchanged): null pointers, a missing field, a datatype other than 7 / 8, is_bigendian,
 * an increment of 0, skips larger than the dimension, a field that ends beyond point_step, `bytes` short of the last point read, more rays
 * than any model may have.  On a closest-point handle the dataset is filled the same way (the ray table is not used there). */
B2_API int b2_rcc_set_cloud_o1dn(b2_rcc* h, const void* data, uint64_t bytes, const b2_cloud_layout* layout, const b2_o1dn_cloud_filter* filter,
                                 int src_is_device);
/* Pc2ToScanNode::convert + fillEmpty + MICPSphericalSensor*::unpackMessage on the device (rmcl_ros/src/nodes/conversion/pc2_to_scan.cpp:105-213,
 * rmcl_ros/src/util/scan_operations.cpp:25-39, MICPSphericalSensorCUDA.cpp:176-235): a sensor_msgs/PointCloud2 binned into the spherical model
 * the handle holds (b2_rcc_set_model_spherical) as its scan.  Point (row, col) is read at row * row_step + col * point_step.  A point with a
 * non-finite x, y or z is skipped; else p = T_sensor_cloud * (x, y, z), range = |p| (float), theta = atan2(p.y, p.x) and
 * phi = atan2(p.z, sqrt(p.x^2 + p.y^2)), both in FP64 rounded to float (the reference takes phi against the 3-D norm: SURVEY D21);
 * id = int((angle - min) / inc + 0.5) with the float division and the double + 0.5 of the reference (no wrap-around, D23); a dimension of
 * size 1 with increment 0 puts every point at 0 (D24).  A point inside the model with range in [range_min, range_max] writes its cell; the
 * last such point in index order wins.  Every other cell gets range_max + 1.  The dataset is point = dir * range, mask = range in
 * [range_min, range_max], as b2_rcc_set_ranges.  The model, its direction table and find's tile schedule stay as they are.
 * src_is_device != 0: `data` is a device address, read in place (valid until the handle's stream has run the kernels); else the bytes up to
 * the last point read are uploaded and the call synchronises.  `data` may be null for a cloud of no points.  Refused (B2_ERR_INVALID, no
 * launch, handle unchanged): null pointers, a missing field, a datatype other than 7 / 8, is_bigendian, a field that ends beyond point_step,
 * `bytes` short of the last point read, more than 2^32 - 2 points, a non-finite T_sensor_cloud, a handle whose current model is not
 * spherical, a model increment of 0 with a size above 1, a non-finite model parameter.  Works on a closest-point handle holding a spherical model. */
B2_API int b2_rcc_set_cloud_spherical(b2_rcc* h, const void* data, uint64_t bytes, const b2_cloud_layout* layout, const b2_transform* T_sensor_cloud,
                                      int src_is_device);
/* RCC..::find(Tbm_est), rmcl/src/rmcl/registration/RCCEmbree.cpp:26-36,58-68,89-99,121-131 */
B2_API int b2_rcc_find(b2_rcc* h, const b2_transform* Tbm_est);
/* The three semantics of rm::*SimulatorEmbree::simulate that SURVEY.md Appendix A.3 cannot settle without rmagine's source, as switches (all 0 = the
 * defaults stated there): tfar_mode 1: rays are traced to +inf instead of model.range.max; min_mode 1: a closest hit nearer than model.range.min is
 * reported as a miss; miss_fill 1: points / normals of a miss are zeros instead of NaN.  Affects b2_rcc_find, correct_once and correct_batch. */
B2_API int b2_rcc_set_sim_options(b2_rcc* h, int tfar_mode, int min_mode, int miss_fill);
/* CPCEmbree (rmcl/include/rmcl/registration/CPCEmbree.hpp:20-54, find at rmcl/src/rmcl/registration/CPCEmbree.cpp:17-43): with
 * B2_CORR_CPC, b2_rcc_find runs one closest-point query per DATASET point (mask not consulted, as in the reference) instead of tracing
 * the sensor model: Pm = Tsm*d_i; cp = map.closestPoint(Pm); hits = cp.d <= max_dist; points = Tms*cp.p; normals = Tms.R*cp.n.
 * No sensor model is needed; the model buffers get n_dataset entries (ranges = cp.d), so b2_rcc_cross_statistics and
 * b2_rcc_correct_once work unchanged.  b2_rcc_correct_once_ranges is refused in this mode. */
B2_API int b2_rcc_set_correspondence_type(b2_rcc* h, int type);
/* closest-point mode only.  skip_masked != 0: dataset points whose mask is 0 are not queried (their model entry reads hits = 0, NaN).  The reference
 * queries every point and never uses those entries (statistics_p2l tests dataset.mask); a dropped beam unpacked to range.max + 1 lies far outside the
 * map and its query is the most expensive of the scan.  Default 0 = the reference's literal behaviour. */
B2_API int b2_rcc_set_cpc_options(b2_rcc* h, int skip_masked);
/* Correspondences{CPU,CUDA}::computeCrossStatistics, rmcl/src/rmcl/registration/CorrespondencesCPU.cpp:10-39 (CUDA twin CorrespondencesCUDA.cpp:9-30) */
B2_API int b2_rcc_cross_statistics(b2_rcc* h, const b2_transform* T_snew_sold, double convergence_progress, b2_cross_stats* out_host);
/* Scan-vs-map segmentation (SURVEY.md 8f4): the classification of ScanMapSegmentationEmbreeNode::scanCB (rmcl_ros/src/nodes/filter/
 * scan_map_segmentation_embree.cpp:84-187).  Call after b2_rcc_set_ranges (the real scan) and b2_rcc_find(T_sensor_map with Tsb = identity,
 * or Tbm with the handle's Tsb): compares real and simulated ranges / normals per ray and returns the two outlier clouds in raster order
 * (HOST buffers of cap_* points x 3 floats; n_* receive the full counts even when the capacity is smaller) and optionally one label per
 * ray (0 none, 1 outlier_scan, 2 outlier_map). */
B2_API int b2_rcc_segment(b2_rcc* h, float min_dist_outlier_scan, float min_dist_outlier_map, float* outlier_scan_host, uint32_t cap_scan, uint32_t* n_scan,
                          float* outlier_map_host, uint32_t cap_map, uint32_t* n_map, uint8_t* labels_host);
/* modelView()/datasetView(), Correspondences.hpp:47-62: device pointers (points/normals packed xyz, hits/mask u8) + our extra face ids / ranges */
B2_API int b2_rcc_model_view(b2_rcc* h, float** points, float** normals, uint8_t** hits, uint32_t** face_ids, float** ranges, uint32_t* n);
B2_API int b2_rcc_dataset_view(b2_rcc* h, float** points, uint8_t** mask, uint32_t* n);
/* host copies of the model buffers (synchronises); any pointer may be NULL */
B2_API int b2_rcc_download_model(b2_rcc* h, float* points, float* normals, uint8_t* hits, uint32_t* face_ids, float* ranges);
B2_API int b2_rcc_download_dataset(b2_rcc* h, float* points, uint8_t* mask);

/* One MICPLocalizationNode::correctOnce for this sensor, entirely on the device
 * (rmcl_ros/src/nodes/micp_localization.cpp:899-984 + rmcl_ros/include/rmcl_ros/micpl/MICPSensor.hpp:146-184):
 * find(Tom*Tbo), then `iterations` x { P2L cross statistics -> frame changes -> Umeyama -> compose }.  Outputs to HOST (may be NULL). */
B2_API int b2_rcc_correct_once(b2_rcc* h, const b2_transform* Tom, const b2_transform* Tbo, uint32_t iterations,
                               double convergence_progress, b2_transform* Tom_new, b2_transform* T_onew_oold, b2_cross_stats* Cmerged_o);
/* same, but the scan arrives as HOST ranges and is uploaded inside the call (end-to-end entry point used by bench.py "e2e").  A pinned buffer
 * (cudaHostAlloc / cudaHostRegister) is moved by a copy engine while find runs and unpacked by the loop kernel; a pageable one is staged and
 * uploaded on a side stream.  The buffer must stay unchanged until the call returns. */
B2_API int b2_rcc_correct_once_ranges(b2_rcc* h, const float* ranges_host, uint32_t n, const b2_transform* Tom, const b2_transform* Tbo,
                                      uint32_t iterations, double convergence_progress, b2_transform* Tom_new, b2_transform* T_onew_oold,
                                      b2_cross_stats* Cmerged_o);

/* The same step split into enqueue / collect: _async launches the kernels on the handle's stream and returns at once, _wait blocks until the
 * result of the OLDEST call in flight has landed (mapped pinned memory, no stream synchronise) and hands it out.  Up to 8 calls may be in flight
 * per handle (exec mode 0: one); the synchronous entry points refuse to run while any is.  Lets a caller keep the GPU queue full (bench.py's
 * device-timed loop) or overlap its own host work with the correction.  The dataset must not be changed while calls are in flight. */
B2_API int b2_rcc_correct_once_async(b2_rcc* h, const b2_transform* Tom, const b2_transform* Tbo, uint32_t iterations, double convergence_progress);
B2_API int b2_rcc_correct_once_wait(b2_rcc* h, b2_transform* Tom_new, b2_transform* T_onew_oold, b2_cross_stats* Cmerged_o);
/* MICPLocalizationNode::correctOnce over ALL sensors of the node (rmcl_ros/src/nodes/micp_localization.cpp:899-984): per sensor k
 * find(Tom * Tbo[k]) (:900-908), then `iterations` x { per sensor: P2L cross statistics under T_bnew_bold = ~Tbo[k] * T_onew_oold * Tbo[k] (:926-929),
 * Cs_o = Tbo[k] * Cs_b (:931), weighted copy n_meas *= merge_weights[k] (u32 *= double, :933-934), Cmerged_o += Cs_o, Cmerged_weighted_o +=
 * Cs_weighted_o (:936-937) } -> umeyama(Cmerged_weighted_o) -> compose (:952-963).  1..4 sensors (RCC or CPC handles on one device); all inner
 * iterations of all sensors run in one kernel.  merge_weights NULL = all 1.0 (MICPSensor.hpp:103); ranges_host NULL or per-sensor NULL = use the
 * resident dataset, else that sensor's scan is uploaded / read zero-copy inside the call.  Outputs to HOST (may be NULL). */
B2_API int b2_micp_correct_once(b2_rcc* const* sensors, const b2_transform* Tbo, const double* merge_weights, const float* const* ranges_host, uint32_t n_sensors,
                                const b2_transform* Tom, uint32_t iterations, double convergence_progress,
                                b2_transform* Tom_new, b2_transform* T_onew_oold, b2_cross_stats* Cmerged_o);
/* What one correctOnce of a chain leaves behind: what MICPSensorStats needs per correction (micp_localization.cpp:1009-1015). */
typedef struct {
    b2_transform   Tom_new, T_onew_oold;     /* as b2_micp_correct_once */
    b2_cross_stats Cmerged_o;
    double         convergence_progress;     /* after this step (:988-1007) */
    uint32_t       valid_measurements;       /* mask ones of all sensors' datasets (MICPSensor.hpp:110, counted as unpackMessage counts them) */
    uint32_t       total_measurements;       /* sum of the dataset sizes (MICPSensor.hpp:109) */
} b2_micp_step;                              /* 144 B */
/* n_corrections x MICPLocalizationNode::correctOnce (micp_localization.cpp:856-1007) back to back on the RESIDENT datasets of 1..4 sensors
 * (upload the scans first: b2_rcc_set_ranges / set_dataset / bind_dataset); n_corrections = 3 is correct() (:847-854), and the body of
 * correctionLoop (:1086-1171) is one call per scan.  Every step traces at the Tom the previous one left in device memory and gates with the
 * max_dist its convergence progress gives (CorrespondencesCPU.cpp:21-23); the host is not involved between the steps.  At the end, one copy to
 * the host: *Tom_inout and *convergence_progress_inout are updated (Tom only when a step had n_meas > 0, :974-984) and steps_out (NULL or
 * n_corrections records) receives each step's outcome.  adaptive_max_dist == 0: the progress stays 0 (:988-990).  Arguments are checked as in
 * b2_micp_correct_once; refused while calls are in flight on the lead handle; handles in exec mode 0 run the chain through mode 1. */
B2_API int b2_micp_correct(b2_rcc* const* sensors, const b2_transform* Tbo, const double* merge_weights, uint32_t n_sensors,
                           b2_transform* Tom_inout, double* convergence_progress_inout, int adaptive_max_dist,
                           uint32_t n_corrections, uint32_t iterations, b2_micp_step* steps_out);
/* The covariance of a MICP-L correction, from the point-to-plane information of its final correspondences (the reference publishes a guess,
 * micp_localization.cpp:1053-1084; no reference implementation, SURVEY appendix I).  Inputs: the sensors, Tbo and merge weights w_k (NULL = all
 * 1.0) of a correction that just ran, its T_onew_oold and the convergence_progress it gated with, and the reference frame Tbo_ref (NULL = Tbo[0]).
 * The published pose is Tbm = Tom_new * Tbo_ref; the covariance is about it, in its body frame: Tbm' = Tbm * Exp(d), d = (x, y, z, roll, pitch,
 * yaw), the order and frame of PoseWithCovariance and of b2_pf_estimate_stats.
 *  - Pairs: sensor k's loop pre-transform T_k = Tso_k * T_onew_oold * Tos_k (Tos = Tbo * Tsb, float, as the ICP loop composes it).  Pair i is
 *    used iff dataset mask > 0, model hit > 0 and the P2L gate of b2_rcc_cross_statistics(T_k, convergence_progress) accepts it, so n_pairs[k]
 *    equals that call's n_meas.  Its residual r is the signed point-to-plane distance of the gate.
 *  - Jacobian: U_k = ~Tbo_ref * Tbo_k * Tsb_k (composed in double, rounded to float once), q = U_k d (the raw dataset point), n = R(U_k) R(T_k)^T N
 *    (the model normal), J = (n, q x n), all in float.
 *  - Sums in FP64, per sensor, then weighted: H = sum_k w_k sum_i J J^T, R2 = sum_k w_k sum_i r^2, Q2 = sum_k w_k sum_i |q|^2, W = sum_k w_k n_k.
 *    sigma2 = R2 / (W - 6) (NaN when W <= 6), L = sqrt(Q2 / W) (1 when that is not > 0).
 *  - Scaling S = diag(1, 1, 1, 1/L, 1/L, 1/L); S H S is decomposed by cyclic Jacobi in FP64 (at most 32 sweeps; stops when the off-diagonal sum of
 *    squares is <= 1e-30 times the matrix's), eigenvalues ascending, each eigenvector's largest-magnitude component positive (first one on ties).
 *    Direction i is degenerate iff eigenvalues[i] <= tau * eigenvalues[5].
 *  - covariance = S (sigma2 sum_nondeg v v^T / lambda + degenerate_variance sum_deg v v^T) S: a degenerate direction gets degenerate_variance m^2
 *    along translation and degenerate_variance / L^2 rad^2 along rotation.
 *  - W == 0 (no pairs): information and the eigen data are 0, covariance and sigma2 NaN, length_scale 0, all six directions degenerate; B2_OK.
 * To describe the last step of b2_micp_correct, pass steps[-1].T_onew_oold with the progress that step gated with: the input progress for one
 * step, else steps[-2].convergence_progress.  Reads each handle's current dataset and model buffers (own or bound) and writes nothing into any
 * handle.  One launch on the lead handle's stream, ordered against the other handles' streams as b2_micp_correct_once orders them, then one copy of
 * the record and a synchronise.  Works for ray-casting and closest-point handles in every exec mode.  Refused (B2_ERR_INVALID, no launch, nothing
 * written): null sensors, Tbo, T_onew_oold, cfg or out_host; n_sensors outside 1..4, a handle given twice, handles on different devices; a handle
 * with calls in flight, with no find yet, or whose dataset size differs from its model size; non-finite transforms; a negative or non-finite
 * weight; tau outside (0, 1); degenerate_variance not finite and > 0.  Suggested values (not tuned on data): tau 1e-3, degenerate_variance 1e2. */
typedef struct { double tau, degenerate_variance; } b2_micp_cov_config;                                          /* 16 B */
typedef char b2_micp_cov_config_is_16_bytes[sizeof(b2_micp_cov_config) == 16 ? 1 : -1];
typedef struct {
    double   information[36], covariance[36];   /* row-major, x y z roll pitch yaw, body frame of Tom_new * Tbo_ref */
    double   eigenvalues[6], eigenvectors[36];  /* of S H S, ascending; row i = unit eigenvector i (scaled coordinates) */
    double   sigma2, residual_sq_sum, weight_sum, length_scale;
    uint64_t n_pairs[4];                        /* gated pairs per sensor */
    uint32_t n_degenerate, degenerate_mask;     /* bit i: eigenvalues[i] <= tau * eigenvalues[5] */
} b2_micp_covariance;                                                                                            /* 984 B */
typedef char b2_micp_covariance_is_984_bytes[sizeof(b2_micp_covariance) == 984 ? 1 : -1];
B2_API int b2_micp_pose_covariance(b2_rcc* const* sensors, const b2_transform* Tbo, const double* merge_weights, uint32_t n_sensors,
                                   const b2_transform* T_onew_oold, double convergence_progress, const b2_transform* Tbo_ref,
                                   const b2_micp_cov_config* cfg, b2_micp_covariance* out_host);
/* How b2_rcc_correct_once* runs the inner iterations: 2 (default) one kernel for all of them, launched programmatically behind find; the block
 * sums cross the grid as 64-bit fixed-point atomics (every block must be co-resident: one block per SM).  1 the same kernel through a cooperative
 * launch, the sums as FP64 slots behind a grid sync.  0 one reduction launch per inner iteration in the reference's own frame-algebra order
 * (MICPSensor.hpp:178-182).  Results agree within float rounding.  The environment variable B2_FUSED sets the default of new handles.  A mode-2
 * call whose blocks cannot become co-resident, or whose sums leave the fixed-point range (|block partial| >= 2^46), is run again through mode 1
 * by the library itself. */
B2_API int b2_rcc_set_exec_mode(b2_rcc* h, int mode);

/* v1 {Sphere,Pinhole,O1Dn}Corrector{Embree,Optix}::correct(Tbm[N]) -> {Tdelta[N], Ncorr[N]}
 * (shape: rmcl_ros/src/benchmarks/lidar_corrector_embree_benchmark.cpp:86-133, ..._optix_benchmark.cpp:85-155):
 * fused trace -> P2L gate -> per-pose cross statistics -> batched Umeyama, one launch sequence for all poses.
 * poses_on_device / out_on_device select HOST or DEVICE pointers. Outputs may be NULL. */
B2_API int b2_rcc_correct_batch(b2_rcc* h, const b2_transform* Tbm, uint32_t n_poses, int poses_on_device,
                                b2_transform* Tdelta, uint32_t* ncorr, b2_cross_stats* stats_b, int out_on_device);
/* v1 corrector.benchmark(Tbm, Nruns) -> {sim, red, svd} seconds (rmcl_ros/src/benchmarks/lidar_corrector_optix_benchmark.cpp:143-155): the stages of
 * correct() run unfused (trace of all poses -> P2L reduction -> Umeyama) and timed separately with CUDA events, summed over n_runs.  Poses on the HOST. */
B2_API int b2_rcc_benchmark_batch(b2_rcc* h, const b2_transform* Tbm_host, uint32_t n_poses, uint32_t n_runs, double* sim_s, double* red_s, double* svd_s);
/* rm::umeyama_transform for n statistics (rmcl_ros/src/nodes/micp_localization.cpp:952-953) */
B2_API int b2_umeyama_batch(const b2_cross_stats* stats, uint32_t n, b2_transform* out, int on_device, int device, void* cuda_stream);

/* ---------------------------------------------------------------- particle filter ---------------------------- */
B2_API int b2_pf_create(b2_mesh* map, b2_pf** out);
B2_API int b2_pf_destroy(b2_pf* h);
B2_API int b2_pf_set_stream(b2_pf* h, void* cuda_stream);
/* How b2_pf_sensor_update maps rays to lanes (a schedule: results are bit-identical).  0: the 32 lanes of a warp trace 32 beams of ONE particle --
 * the reference's loop order seen from a particle (PCDSensorUpdaterEmbree.cpp:290-342) and the better choice for particle sets spread over the map.
 * 1: the lanes trace the SAME beam for 32 particles; 2: the same after sorting the particles by (heading, map cell) on the device, coherent and up to
 * 1.7x faster once the cloud has converged.  3 (default): 0 or 2, whichever was faster when last timed (both on the first two updates, the slower one
 * again every 64 updates).  The environment variable B2_PF_MAP sets the default of new handles. */
B2_API int b2_pf_set_mapping(b2_pf* h, int mode);
B2_API int b2_pf_get_mapping(b2_pf* h, int* mode, int* current);
/* ParticleUpdater<VRAM_CUDA>::update (rmcl_ros/include/rmcl_ros/rmcl/ParticleUpdater.hpp:39-43) with the hot loop of
 * PCDSensorUpdaterEmbree::update (rmcl_ros/src/rmcl/PCDSensorUpdaterEmbree.cpp:290-342): all beams x all particles in ONE launch,
 * per-particle likelihood merged in beam order, attrs read-modified-written once.  poses/attrs: DEVICE pointers; beams: HOST. */
B2_API int b2_pf_sensor_update(b2_pf* h, const b2_transform* poses_dev, b2_particle_attr* attrs_dev, uint32_t n_particles,
                               const b2_transform* Tsb, const b2_range_meas* beams_host, uint32_t n_beams, const b2_pf_params* params);
/* ParticleUpdater<RAM>::update: HOST poses/attrs; copies in, updates, copies attrs back (end-to-end entry point).  Sets of 32 768 particles and more
 * are processed in 8 chunks alternating between two streams: with pinned host arrays the transfers run under the kernel (C3: 5.2 ms for 5.13 ms of
 * kernel).  attrs_host is updated in place. */
B2_API int b2_pf_sensor_update_host(b2_pf* h, const b2_transform* poses_host, b2_particle_attr* attrs_host, uint32_t n_particles,
                                    const b2_transform* Tsb, const b2_range_meas* beams_host, uint32_t n_beams, const b2_pf_params* params);
/* PCDSensorUpdaterOptix::update's beam sampling (rmcl_ros/src/rmcl/PCDSensorUpdaterOptix.cpp:227-311): the beams of one sensor update drawn
 * from a sensor_msgs/PointCloud2, for b2_pf_sensor_update / b2_pf_sensor_update_host as they are.
 *  - Points are i = row * width + col, n_points = width * height; point i is read at row * row_step + col * point_step through the x, y and z
 *    fields of `layout` (FLOAT32 as is, FLOAT64 narrowed to float), as b2_rcc_set_cloud_o1dn reads them.
 *  - Sample k < n_samples makes up to 100 tries.  Try t takes raw = word t % 4 of Philox4x32-10 with counter (k, 3, step, t / 4) and key
 *    `seed`, and reads point raw % n_points.  The draws depend on (seed, step, k) only: every rank of a sharded particle set that passes the
 *    same seed and step gets the same beams.  Advance `step` per update.
 *  - A try is valid iff x == x && y == y && z == z (NaN fails, an infinite coordinate passes).  A valid sample is orig = 0, range = |p|,
 *    dir = p / range (float, individually rounded), cov = 0.1 I.  A finite (0,0,0) gives range 0 and NaN directions; an infinite coordinate
 *    gives range inf.  A NaN component is stored as 0x7fffffff.
 *  - Sampling stops at the 10th sample whose 100 tries all failed.  beams_host receives the valid samples before that point in sample order
 *    (their likelihood merge order), *n_beams their count.  n_points == 0 or n_samples == 0: no beams, B2_OK.
 * src_is_device != 0: `data` is a device address, read in place by one kernel on the handle's stream (one thread per sample); 68 B per
 * sample come back and the call synchronises the stream.  Else `data` is host memory and the same function runs on the host over the
 * points it draws; nothing is uploaded and nothing is launched.  Both give the same bytes.  Refused (B2_ERR_INVALID, no launch, nothing
 * written): null pointers, a missing x, y or z field, a datatype other than 7 / 8, is_bigendian, a field that ends beyond point_step,
 * `bytes` short of the end of the last point (any point may be drawn), more than 2^32 - 1 points.  The arguments are checked before the
 * handle. */
B2_API int b2_pf_sample_cloud(b2_pf* h, const void* data, uint64_t bytes, const b2_cloud_layout* layout, int src_is_device, uint32_t n_samples,
                              uint64_t seed, uint32_t step, b2_range_meas* beams_host, uint32_t* n_beams);

/* rest of the particle-filter cycle on the device (SURVEY.md 8f2), so that particles never leave HBM between stages:
 * TFMotionUpdaterGPU / particle_move_and_forget (rmcl_ros/src/rmcl/particle_motion.cu:11-46): pose = pose * T_bnew_bold, n_meas -= forget_rate * n_meas.
 * check_collision != 0 adds the wall check of the CPU updater (TFMotionUpdaterCPU.cpp:17-50,205-216): a ray from the old to the new position; a hit
 * sets the particle's likelihood to {0, 0, MAX_N_MEAS}. */
B2_API int b2_pf_motion_update(b2_pf* h, b2_transform* poses_dev, b2_particle_attr* attrs_dev, uint32_t n_particles, const b2_transform* T_bnew_bold, double forget_rate,
                               int check_collision);
/* compute_stats (rmcl_ros/src/rmcl/resampling.cu:41-92): sum and max (initial 0) of likelihood.mean over the LOCAL particles; with particles
 * sharded across GPUs the caller all-reduces the 8 bytes (SUM, MAX) -- the one exchange step of the cycle.  Results to HOST. */
B2_API int b2_pf_likelihood_stats(b2_pf* h, const b2_particle_attr* attrs_dev, uint32_t n_particles, float* sum_out, float* max_out);

/* GladiatorResamplerGPU / gladiator_resample (rmcl_ros/src/rmcl/resampling.cu:108-221; config GladiatorResamplerConfig.hpp:7-20): each
 * champion i draws a random opponent; if the opponent's likelihood.mean is larger, the champion's slot receives a perturbed copy of the
 * opponent (Gaussian noise on t and on the Euler angles) whose n_meas is reduced by the forget rate; else it keeps its own state.
 * poses/attrs hold ALL n_all particles (on one GPU: the local ones; sharded: the all-gathered set -- the one exchange step of this stage);
 * this call produces the champions first .. first+n_local-1 into poses_new/attrs_new (n_local entries; must not alias the inputs).
 * Draws come from Philox4x32-10 keyed by (seed, step, global particle index) unless raw_dev/normals_dev (n_local, n_local x 6) supply them. */
typedef struct {
    float min_noise_tx, min_noise_ty, min_noise_tz, min_noise_roll, min_noise_pitch, min_noise_yaw;
    float likelihood_forget_per_meter, likelihood_forget_per_radian;     /* reference defaults 0.3, 0.2 */
} b2_gladiator_config;
B2_API int b2_pf_resample_gladiator(b2_pf* h, const b2_transform* poses_dev, const b2_particle_attr* attrs_dev, uint32_t n_all, uint32_t first, uint32_t n_local,
                                    b2_transform* poses_new_dev, b2_particle_attr* attrs_new_dev, const b2_gladiator_config* cfg, uint64_t seed, uint32_t step,
                                    const uint32_t* raw_dev, const float* normals_dev);
/* The same resampling with the particles SHARDED over GPUs (one process per GPU) and no all-gather: every rank publishes its shard in a buffer
 * the other ranks map over NVLink (CUDA IPC); a champion reads its opponent's 4-byte likelihood from the owner's HBM and fetches the 68-byte
 * record only when the opponent wins (the reference draws opponents from all particles, resampling.cu:137).  Equal shard sizes; results equal the
 * single-GPU resampling of the concatenated set bit for bit.  init -> (exchange the 128-byte handles of all ranks) -> connect; per step:
 * publish, cross-rank barrier, resample_p2p, cross-rank barrier.  remote_bytes_out (may be NULL) receives the bytes read from other GPUs. */
B2_API int b2_pf_p2p_init(b2_pf* h, uint32_t n_per_rank, void* handles_out_128_bytes);
B2_API int b2_pf_p2p_connect(b2_pf* h, const void* all_handles_world_x_128, uint32_t world, uint32_t rank, uint32_t n_per_rank);
B2_API int b2_pf_p2p_publish(b2_pf* h, const b2_transform* poses_dev, const b2_particle_attr* attrs_dev, uint32_t n_local);
B2_API int b2_pf_resample_gladiator_p2p(b2_pf* h, b2_transform* poses_new_dev, b2_particle_attr* attrs_new_dev, const b2_gladiator_config* cfg, uint64_t seed, uint32_t step,
                                        uint64_t* remote_bytes_out);
/* test hook: several shards on one device (poses_all / attrs_all hold world * n_per_rank particles; this handle plays `rank`) */
B2_API int b2_pf_p2p_connect_local(b2_pf* h, const b2_transform* poses_all_dev, const b2_particle_attr* attrs_all_dev, uint32_t world, uint32_t rank, uint32_t n_per_rank);
/* the draws b2_pf_resample_gladiator would use (replaces init_curand / curand(), resampling.cu:13-30,134-143): raw u32 + 6 normals per particle */
B2_API int b2_pf_gladiator_randoms(b2_pf* h, uint64_t seed, uint32_t step, uint32_t first, uint32_t n, uint32_t* raw_dev, float* normals_dev);

/* Particle set initialisation on the device: writes particles first .. first+n-1 of the set into poses_dev / attrs_dev (n entries each; DEVICE
 * pointers) with likelihood {1, 0, 0} and state_sigma 0.  Draws are Philox4x32-10 keyed by (seed, global particle index), so initialising
 * [first, first+n) on each rank and concatenating equals one call for the whole set, bit for bit.  Launches on the handle's stream, no host
 * synchronisation; n == 0 launches nothing.  A bad box or covariance and first + n > 2^32 are refused before any launch.
 * RmclNode::initSamplesUniform (rmcl_ros/src/nodes/rmcl_localization.cpp:277-342): t and the Euler angles uniform in [bb_min, bb_max]
 * (x, y, z, roll, pitch, yaw; doubles narrowed to float; min == max gives exactly that value; min > max or non-finite is refused). */
B2_API int b2_pf_init_uniform(b2_pf* h, b2_transform* poses_dev, b2_particle_attr* attrs_dev, uint32_t first, uint32_t n, const double bb_min[6], const double bb_max[6],
                              uint64_t seed);
/* RmclNode::initSamples(PoseWithCovarianceStamped) (rmcl_localization.cpp:165-275): x = chol(C) N(0, I6) with C the message's 36 doubles
 * (row-major, narrowed to float, lower triangle read), pose = *pose * Transform{EulerAngles{x3, x4, x5}, {x0, x1, x2}} -- the covariance
 * acts in the pose frame.  A zero variance whose covariances are zero gives that component no noise; a negative or NaN pivot, or a zero
 * variance with a non-zero covariance, is refused with a message naming the column. */
B2_API int b2_pf_init_gaussian(b2_pf* h, b2_transform* poses_dev, b2_particle_attr* attrs_dev, uint32_t first, uint32_t n, const b2_transform* pose,
                               const double cov_rowmajor[36], uint64_t seed);

/* rmcl_msgs/ParticleStats (rmcl_msgs/msg/ParticleStats.msg) with its LikelihoodStats and PoseWithCovariance flattened. */
typedef struct { double min, max, mean, sigma; } b2_likelihood_stats;
typedef struct {
    double position[3];                        /* pose.pose.position: x y z */
    double orientation[4];                     /* pose.pose.orientation: x y z w */
    double covariance[36];                     /* pose.covariance, row-major: x y z roll pitch yaw */
    double shift;
    double trans_bb_min[3], trans_bb_max[3];
    b2_likelihood_stats likelihood;
    uint64_t nparticles;
} b2_particle_stats;                           /* 440 B */
typedef char b2_particle_stats_is_440_bytes[sizeof(b2_particle_stats) == 440 ? 1 : -1];      /* static assert, valid C and C++ */
/* RmclNode::estimateStats (rmcl_ros/src/nodes/rmcl_localization.cpp:642-731) on the device: the statistics of the first n particles (the
 * caller passes n = min(n_particles, max_induction_particles), as the node slices poses(0, k)); poses/attrs are DEVICE pointers, out_host a
 * HOST record.  Two read passes on the handle's stream, then one copy of the record to the host and a synchronise.
 *  - likelihood: sum, sum of squares, min (from DBL_MAX), max (from 0.0) of likelihood.mean in double; mean = sum / n, sigma = sqrt(sum_sq / n
 *    - mean^2), 0 when rounding alone makes the variance negative; shift = min.  trans_bb_min/max: the float AABB of the translations.
 *  - pose: the weighted Markley mean with w_i = L_i / sum: t = sum w_i t_i, R = the eigenvector of the largest eigenvalue of sum w_i q_i q_i^T
 *    (sign: w >= 0), rounded to a float Transform Tbm.
 *  - covariance: sum w_i v_i v_i^T with v_i = (d.t, roll, pitch, yaw of d.R), d = ~Tbm * pose_i, about Tbm (no re-centring).
 * When the likelihood sum is not > 0 or not finite (every likelihood 0), the pose and covariance are NaN, as the reference's division by zero
 * gives them, and the rest is filled in; the call still returns B2_OK.  n == 0 and null pointers are refused before any launch. */
B2_API int b2_pf_estimate_stats(b2_pf* h, const b2_transform* poses_dev, const b2_particle_attr* attrs_dev, uint32_t n, b2_particle_stats* out_host);

/* ResidualResamplerCPU::update (rmcl_ros/src/rmcl/ResidualResamplerCPU.cpp:55-202; config and defaults :35-47, the fields of Gladiator's) on
 * the device.  Resamples the n particles poses_dev / attrs_dev into an output set of M = n_new slots; the set may grow (the node passes its
 * whole max_particles buffer).
 *  - S = weight_sum and weight_max = max(0, L_i) of likelihood.mean in double, in the order of b2_pf_estimate_stats: S / n and weight_max
 *    equal its likelihood.mean and .max bit for bit for the same n.
 *  - Draw j = 0, 1, ... picks parent word j % 4 of Philox4x32-10 with counter (lo(j / 4), 4, step, hi(j / 4)) and key `seed`, modulo n, and
 *    inserts min((uint64)(L / S * M), slots left) copies.  Draws that insert nothing are consumed.  The draws stop when all M slots are
 *    filled, or after D_max = 16 * max(n, M) draws (the reference's loop need not end); the slots filled by then are the result.
 *  - The copy in slot k takes its six normals from Box-Muller on words 0-5 of the counters (k, 5, step, 0) and (k, 5, step, 1): t += N *
 *    (float)(min_noise / (L / weight_max)) for x, y, z, then roll, pitch, yaw of R likewise; n_meas *= (float)(pow(forget_per_meter,
 *    |d.t|^2) * pow(forget_per_radian, |d.R|)) with d = ~pose * pose_new, truncated; the rest, the stamp included, is the parent's.
 *  - S not finite, S <= 0 or a likelihood below 0: 0 slots, nothing written, B2_OK (the node skips resampling below 10 particles).
 * poses_new_dev / attrs_new_dev hold n_local entries: entry i is slot first + i.  The call writes the entries whose slot is below
 * n_particles and leaves the others untouched, so ranks of a sharded set that pass the same (all-gathered) input and disjoint slices
 * [first, first + n_local) together write the one global result.  Runs on the handle's stream and synchronises it: one read-back after the
 * statistics and one per chunk of draws (chunks double from max(2n, 2^16) up to 2 max(n, M)).  Refused (B2_ERR_INVALID, no launch, nothing
 * written): null pointers, n == 0, n_new == 0, first + n_local > n_new, an output range overlapping an input range or the other output. */
typedef b2_gladiator_config b2_residual_config;
typedef struct { uint64_t n_particles, draws; double weight_sum, weight_max; } b2_residual_result;
B2_API int b2_pf_resample_residual(b2_pf* h, const b2_transform* poses_dev, const b2_particle_attr* attrs_dev, uint32_t n, uint32_t n_new,
                                   uint32_t first, uint32_t n_local, b2_transform* poses_new_dev, b2_particle_attr* attrs_new_dev,
                                   const b2_gladiator_config* cfg, uint64_t seed, uint32_t step, b2_residual_result* out_host);

/* KLD-sampling (Fox, "Adapting the sample size in particle filters through KLD-sampling", IJRR 2003; "reduce the number of particles more
 * intelligently", rmcl/docs/RMCL.md:80-83, listed as missing; SURVEY appendix G): resamples the n particles poses_dev / attrs_dev into an
 * output set of at most n_max slots (the node passes its whole max_particles buffer), as many as the spread of the drawn set calls for.
 *  - S = weight_sum, L_min and weight_max = L_max of likelihood.mean as b2_pf_resample_residual takes them.  S not finite, S <= 0 or L_min < 0:
 *    0 particles, nothing written, B2_OK.
 *  - Weights w_i = (uint64)((double)L_i / L_max * 2^32), inclusive prefix W (exact in 64 bits).  Draw j takes u = words 2(j % 2) (low) and
 *    2(j % 2) + 1 (high) of Philox4x32-10 with counter (lo(j / 2), 6, step, hi(j / 2)) and key `seed`; its parent is the smallest i with
 *    W[i] > mulhi64(u, W[n-1]).  A zero weight is never drawn.
 *  - The bin of a draw is its parent's ix = floor(t.x / res_xy), iy likewise, iz with res_z (res_z = 0: z not binned), clamped to [-2^19, 2^19)
 *    and [-2^7, 2^7), and the yaw sector of the heading h = (1 - 2(y^2 + z^2), 2(xy + wz)) among K = ceil(2 pi / res_yaw (1 - 2^-20)) sectors with
 *    boundaries -pi + 2 pi k / K; roll and pitch are not binned.  A non-finite pose is its own bin.
 *  - Stop at the first draw j with j + 1 >= max(n_min, bound(k_j)) or j + 1 = n_max, k_j the number of bins among draws 0 .. j and
 *    bound(k) = ceil((k - 1) / (2 epsilon) x^3), x = 1 - 2 / (9(k - 1)) + sqrt(2 / (9(k - 1))) z, bound(k <= 1) = n_min.  z is the upper
 *    standard normal quantile of the bound's confidence, used as given.  n_particles = j + 1, bins = k_j.
 *  - Slot j is a copy of draw j's parent as b2_pf_resample_residual copies it (normals keyed by the slot with tag 5, noise scaled by
 *    L_max / L, forget factors, the parent's stamp), with the Gladiator config `cfg`.
 * poses_new_dev / attrs_new_dev hold n_local entries: entry i is slot first + i.  Only slots below n_particles are written, so ranks that pass
 * the same (all-gathered) input and disjoint slices together write the one global result.  Runs on the handle's stream and synchronises it:
 * one read-back after the statistics and one per chunk of draws (chunks double from max(n_min, 2^16) up to n_max; at most n_max draws).
 * The handle keeps a hash set of at least 2 n_max slots (12 B each) and 24 B per draw of the largest chunk.  Refused (B2_ERR_INVALID, no
 * launch, nothing written): null pointers, n == 0, n_max == 0, n_min == 0, n_min > n_max, first + n_local > n_max, an output range overlapping
 * an input range or the other output, res_xy or epsilon not finite and > 0, res_z not finite and >= 0, z not finite, K outside [1, 32768].
 * Suggested values (AMCL's defaults but res_z; AMCL passes its kld_z of 0.99 as the quantile itself): res_xy 0.5 m, res_z 0, res_yaw 10 deg
 * (K = 36), epsilon 0.01, z 0.99, n_min 100. */
typedef struct { float res_xy, res_z, res_yaw; uint32_t n_min; double epsilon, z; } b2_kld_config;            /* 32 B */
typedef char b2_kld_config_is_32_bytes[sizeof(b2_kld_config) == 32 ? 1 : -1];
typedef struct { uint64_t n_particles, bins; double weight_sum, weight_max; } b2_kld_result;                  /* 32 B */
typedef char b2_kld_result_is_32_bytes[sizeof(b2_kld_result) == 32 ? 1 : -1];
B2_API int b2_pf_resample_kld(b2_pf* h, const b2_transform* poses_dev, const b2_particle_attr* attrs_dev, uint32_t n, uint32_t n_max, uint32_t first,
                              uint32_t n_local, b2_transform* poses_new_dev, b2_particle_attr* attrs_new_dev, const b2_gladiator_config* cfg,
                              const b2_kld_config* kld, uint64_t seed, uint32_t step, b2_kld_result* out_host);

/* The filter's pose hypotheses: the clusters of the particle set, heaviest first, each with the estimate b2_pf_estimate_stats would give of
 * it alone.  What AMCL publishes is the mean of its heaviest cluster (pf_cluster_stats); the reference reports one mean over the whole set,
 * which during global localisation lies between the modes (no reference implementation; SURVEY appendix H).  poses_dev / attrs_dev are DEVICE
 * pointers to n particles, records_host a HOST array of cfg->max_records records, labels_dev a DEVICE array of n labels or null.
 *  - S = weight_sum, L_min and weight_max = L_max of likelihood.mean as b2_pf_resample_kld takes them.  S not finite, S <= 0 or L_min < 0:
 *    0 clusters, nothing written but out_host, B2_OK.
 *  - Particle i is a member iff w_i = (uint64)((double)L_i / L_max * 2^32) > 0 and its pose is finite.  n_clustered counts the members,
 *    weight_total = sum w_i over them (exact in 64 bits).  A particle the wall check or the surface projection marked (L = 0) is in no
 *    cluster and joins none.
 *  - A member's bin is b2_pf_resample_kld's: the x, y, z cell (res_z = 0: z not binned) and the yaw sector among K = ceil(2 pi / res_yaw
 *    (1 - 2^-20)) sectors.  bins counts the occupied bins.
 *  - Two occupied bins touch iff their x, y and z cells each differ by at most 1 and their sectors by at most 1 modulo K: yaw wraps, while a
 *    cell clamped at +-2^19 (z: +-2^7) has no neighbour beyond the clamp.  With K <= 2 some of the 80 neighbours (26 when z is not binned)
 *    coincide; joining a pair twice changes nothing.  A cluster is a connected component of that graph.  Its key is its smallest bin key
 *    ((ix + 2^19) << 44 | (iy + 2^19) << 24 | (iz + 2^7) << 16 | sector), its weight_int the sum of its members' w_i, weight = weight_int /
 *    weight_total, bins its occupied bins.
 *  - Clusters are ranked by weight_int descending, ties by the smaller key; rank 0 is the best hypothesis.  records_host[r], r < n_records =
 *    min(n_clusters, max_records), describes rank r: `stats` is byte for byte what b2_pf_estimate_stats returns for the cluster's members
 *    alone, in ascending particle index.  labels_dev[i] is the rank of particle i's cluster (any rank, recorded or not), 0xFFFFFFFF for a
 *    particle in none.
 *  - rounds: the labelling rounds run.  A round joins every touching pair with lock-free union-find hooks and ends in the fixed point, so
 *    this is 1; the call gives up with an error after 64.
 * Every sum that decides a result is an integer, so nothing depends on the order in which threads run.  Runs on the handle's stream and
 * synchronises it: one read-back after the statistics, one per round, one for the ranking, one for the records.  The handle shares
 * b2_pf_resample_kld's hash set (at least 2 n slots of 12 B) and adds 16 B per slot (weight, members, bins / rank), 20 B per particle (slot,
 * sort keys and indices) and 68 B per member of a recorded cluster.  Refused (B2_ERR_INVALID, no launch, nothing written): null h, poses_dev,
 * attrs_dev, cfg, records_host or out_host, n == 0 or n > 2^30, res_xy not finite and > 0, res_z not finite and >= 0, K outside [1, 32768],
 * max_records outside [1, 16].  Suggested values (AMCL's bin sizes): res_xy 0.5 m, res_z 0, res_yaw 10 deg, max_records 8. */
typedef struct { float res_xy, res_z, res_yaw; uint32_t max_records; } b2_cluster_config;                     /* 16 B */
typedef char b2_cluster_config_is_16_bytes[sizeof(b2_cluster_config) == 16 ? 1 : -1];
typedef struct { b2_particle_stats stats; double weight; uint64_t weight_int, bins, key; } b2_cluster_record; /* 472 B */
typedef char b2_cluster_record_is_472_bytes[sizeof(b2_cluster_record) == 472 ? 1 : -1];
typedef struct { uint64_t n_clusters, n_records, bins, n_clustered, weight_total, rounds; double weight_sum, weight_max; } b2_cluster_result;   /* 64 B */
typedef char b2_cluster_result_is_64_bytes[sizeof(b2_cluster_result) == 64 ? 1 : -1];
B2_API int b2_pf_cluster_stats(b2_pf* h, const b2_transform* poses_dev, const b2_particle_attr* attrs_dev, uint32_t n, const b2_cluster_config* cfg,
                               b2_cluster_record* records_host, uint32_t* labels_dev /* nullable */, b2_cluster_result* out_host);

/* The motion stage's surface constraint, "a MotionUpdater constrained to the mesh surface" (rmcl/docs/RMCL.md:72, listed as missing; no
 * reference implementation, SURVEY appendix F): keeps the particle set on the walkable surface of a mesh map (ramps, stairs, floors) after any
 * stage that moves it (init, motion, resampling).  Up is map +z (REP-103).  Per particle, with t, R its pose, in float arithmetic rounded in
 * the order written, cos_max = (float)cos((double)max_slope) and tfar = probe_above + probe_below:
 *  1. probe: the closest hit of the ray from (t.x, t.y, t.z + probe_above) along (0, 0, -1) with t_hit in (0, tfar], ties to the smaller face
 *     id (the rule of b2_mesh_intersect);
 *  2. ground iff n.z >= cos_max, n = normalize(Ng) of the hit triangle, negated if n.z < 0 (it faces the ray origin); a NaN normal is not ground;
 *  3. on ground: g = (t.x, t.y, (t.z + probe_above) - t_hit).  align 0: R' = R, t' = (g.x, g.y, g.z + base_height).  align 1: a = R e_z (the
 *     quaternion rotation), c = a . n, q = (R e_x, 0) if 1 + c < 1e-6 else (a x n, 1 + c), R' = normalize(normalize(q) * R) and
 *     t' = g + base_height * n: the smallest rotation that takes the body z-axis onto n, so the heading changes as little as possible.
 *     The stamp and the attributes are unchanged;
 *  4. off surface (no hit, a hit that is not ground, a non-finite t or R; a non-finite position hits nothing): the pose is unchanged and the likelihood
 *     becomes {0, 0, MAX_N_MEAS}, the wall check's mark (b2_pf_motion_update); state_sigma is unchanged.  The next resampling replaces it.
 * Limits: a probe_above larger than the clearance under a table or an upper floor lands the particle on top of it; with base_height 0 the wall
 * check's old -> new ray runs along the ground and can graze it on curved terrain (use base_height > 0 with check_collision).
 * In place on poses_dev / attrs_dev (DEVICE pointers), one thread per particle on the handle's stream, no synchronisation; n == 0 launches
 * nothing.  Refused (B2_ERR_INVALID, no launch, both buffers untouched): null h or cfg, null buffers with n > 0, a non-finite field,
 * probe_above < 0, probe_below < 0, tfar <= 0, base_height < 0, max_slope outside [0, pi/2], align other than 0 or 1.
 * Suggested values: probe_above 0.5, probe_below 1.0, base_height 0.0, max_slope 0.6 rad, align 1. */
typedef struct { float probe_above, probe_below, base_height, max_slope; int32_t align; } b2_surface_config;      /* 20 B */
B2_API int b2_pf_project_to_surface(b2_pf* h, b2_transform* poses_dev, b2_particle_attr* attrs_dev, uint32_t n_particles, const b2_surface_config* cfg);

/* Recovery from a kidnapping: Augmented MCL (Thrun, Burgard, Fox, Probabilistic Robotics, 8.3.5; AMCL's recovery_alpha_slow / _fast; no
 * reference implementation, SURVEY appendix J).  A converged set only copies and perturbs its own particles, so once the robot is lifted,
 * slips or its odometry jumps, nothing puts a particle where it really is.  These calls keep a slow and a fast average of the set's mean
 * likelihood and, when the fast one drops below the slow one, replace a fraction p = max(0, 1 - w_fast / w_slow) of the particles with
 * random poses.  One cycle: motion, sensor update, b2_pf_recovery_observe, resampling, b2_pf_recovery_inject, (surface projection).
 * The handle keeps a device-resident record {w_slow, w_fast, p_inject}, zero at creation.
 *
 * b2_pf_recovery_reset: sets the record to 0, enqueued on the handle's stream.  Call it after (re)initialising the set.
 *
 * b2_pf_recovery_observe: call it once after each sensor update, on the whole set (a sharded set passes the all-gathered set, as
 * b2_pf_resample_kld takes it, so every rank holds the same record).
 *  - w_avg = S / n, S the FP64 sum of likelihood.mean that b2_pf_resample_residual computes (bit-equal to b2_pf_estimate_stats' sum).
 *    likelihood.mean is the filter's running, forgotten fit, not the latest scan's likelihood: the recovery reacts at the pace the forget
 *    settings give the filter's memory.
 *  - w_avg not finite or below 0: the record is left unchanged.  Otherwise each average w of rate alpha becomes w_avg when w == 0, else
 *    w + alpha (w_avg - w); then p_inject = w_slow > 0 ? max(0, 1 - w_fast / w_slow) : 0, all in FP64.
 *  - One statistics pass and a one-thread update kernel that reads its result in device memory: no read-back.  state_host (may be NULL)
 *    receives {w_avg, w_slow, w_fast, p_inject} and the call synchronises; otherwise it only enqueues.
 *  Refused (B2_ERR_INVALID, no launch): null h, attrs_dev or cfg; n == 0; an alpha not finite or outside [0, 1]; alpha_slow > alpha_fast.
 *  Suggested values: alpha_slow 0.001, alpha_fast 0.1 (AMCL's recovery_alpha_slow / _fast).
 *
 * b2_pf_recovery_inject: call it after resampling.  In place on the slice [first, first + n_local) of the set (poses_dev / attrs_dev hold
 * n_local entries, DEVICE pointers), with p = p_inject read from the record on the device.  Particle g (global index), Philox4x32-10 with key
 * `seed` and counter (g, 7, step, block):
 *  1. replaced iff (double)word0 of block 0 * 2^-32 < p (p == 0: nothing is touched);
 *  2. try t < max_tries draws the six words 0-3 of block 1 + 2t and 0-1 of block 2 + 2t and maps them into the box [bb_min, bb_max] (x, y,
 *     z, roll, pitch, yaw) as b2_pf_init_uniform does;
 *  3. surface NULL: the first candidate is taken.  Otherwise a candidate is taken iff b2_pf_project_to_surface's rule finds ground under it,
 *     and it is taken as that rule moved it;
 *  4. a taken candidate overwrites the pose (stamp 0, as the initialiser writes it) and the attributes become {mean 0, sigma 0, n_meas 0},
 *     state_sigma 0: an unevaluated particle carries no weight in the estimates and resamplers until the next sensor update, whose merge
 *     takes the fresh likelihood alone.  (The wall check's mark is {0, 0, MAX_N_MEAS}.)
 *  5. no candidate taken within max_tries: the particle stays exactly as it was and counts as failed.
 * After the call, if p > 0, the record is reset to 0 (AMCL resets the averages after it injects, so that it does not spiral into complete
 * randomness).  out_host (may be NULL) receives {p used, n_replaced, n_failed} of the slice and the call synchronises; otherwise it only
 * enqueues.  Draws depend on (seed, step, g, try) only, so slices concatenate to the whole result bit for bit.  n_local == 0 launches nothing
 * and so leaves the record as it is: in a sharded set give every rank a non-empty slice (equal shards do), or a rank with an empty one keeps
 * p > 0 while the others reset, and their records differ from then on.
 * Limit: the surface test puts a candidate on walkable ground; it does not prove the robot fits there (under a table, say).
 *  Refused (B2_ERR_INVALID, no launch, buffers untouched): null h, bb_min or bb_max; the box refusals of b2_pf_init_uniform; the refusals
 *  of b2_pf_project_to_surface when surface is given; max_tries outside [1, 64]; null buffers with n_local > 0; first + n_local > 2^32.
 *  Suggested values: max_tries 16; the map's box with roll and pitch 0 and yaw [-pi, pi); b2_pf_project_to_surface's suggested config. */
typedef struct { double alpha_slow, alpha_fast; } b2_recovery_config;                                          /* 16 B */
typedef char b2_recovery_config_is_16_bytes[sizeof(b2_recovery_config) == 16 ? 1 : -1];
typedef struct { double w_avg, w_slow, w_fast, p_inject; } b2_recovery_state;                                  /* 32 B */
typedef char b2_recovery_state_is_32_bytes[sizeof(b2_recovery_state) == 32 ? 1 : -1];
typedef struct { double p_inject; uint64_t n_replaced, n_failed; } b2_recovery_result;                         /* 24 B */
typedef char b2_recovery_result_is_24_bytes[sizeof(b2_recovery_result) == 24 ? 1 : -1];
B2_API int b2_pf_recovery_reset(b2_pf* h);
B2_API int b2_pf_recovery_observe(b2_pf* h, const b2_particle_attr* attrs_dev, uint32_t n, const b2_recovery_config* cfg, b2_recovery_state* state_host /* nullable */);
B2_API int b2_pf_recovery_inject(b2_pf* h, b2_transform* poses_dev, b2_particle_attr* attrs_dev, uint32_t first, uint32_t n_local, const double bb_min[6],
                                 const double bb_max[6], const b2_surface_config* surface /* nullable */, uint32_t max_tries, uint64_t seed, uint32_t step,
                                 b2_recovery_result* out_host /* nullable */);

/* ---------------------------------------------------------------- distance field ----------------------------- */
/* Truncated distance field of the map and the particle filter's sensor update from it (no reference counterpart; AMCL's
 * laser_model_type likelihood_field; SURVEY appendix K).  The closest-point update (correspondence_type 1) walks the BVH once per
 * (particle, beam); the field is built once per map and each beam then costs one interpolated lookup, whatever the depth of the tree.
 *
 * Definition (origin, h, dims, trunc).  Node (i, j, k) sits at x = origin.x + (float)i * h (likewise y, z; each op rounded) and holds
 * min(d, trunc), d the closest-point distance of b2_rcc's closest-point correspondences at that position (a bounded query: same value).
 * Storage: a dense uint32 index over bricks of 8^3 cells (0xFFFFFFFF: not allocated) and, per allocated brick, its 9^3 nodes (z, y, x; x
 * fastest; the far face is shared with the next brick).  A brick is allocated iff the distance from its centre node is < trunc + 8h; every
 * node of an unallocated brick has value trunc.  Memory: 4 B per brick of the box plus 2916 B per allocated brick.
 * Lookup at p: g = (p - origin) * (1 / h) per axis; inside iff 0 <= g <= dims - 1; cell = min(floor(g), dims - 2); trilinear in the order
 * x, y, z.  Unallocated brick or finite point outside the box: trunc.  Non-finite point: +inf.  No texture filtering.
 * Accuracy: |field(p) - min(d_exact(p), trunc)| <= (sqrt(3) / 2) h plus float rounding.  Choose h from this bound.
 *
 * b2_dfield_create: builds the field on the map's device (classify bricks, scan, fill nodes) and synchronises.  params.bb_min / bb_max
 *  (both or neither, 3 floats each) give the box; NULL: the map's AABB grown by `truncation`.  The field keeps a reference to the map,
 *  which may be destroyed first.  It is a snapshot: after b2_mesh_refit it still describes the map as it was -- destroy and recreate it.
 *  Refused (B2_ERR_INVALID, nothing built, *out = NULL): null arguments, one of bb_min / bb_max null, resolution or truncation not finite
 *  and > 0, non-finite bounds, bb_min >= bb_max on an axis, more than 2^24 nodes on an axis (8 x bricks + 1, so that (float)i is exact),
 *  more than 2^32 - 2 bricks.  An empty map: B2_ERR_NO_MAP; allocation failure: B2_ERR_OOM.
 * b2_dfield_get_info: the grid, counts, bytes resident and the build's wall time.
 * b2_dfield_download: the raw layout (bricks_total uint32 index words, bricks_allocated x 729 floats), either pointer may be NULL.
 * b2_dfield_query: lookups of n points (xyz), synchronous.  src_is_device != 0: points and dist_out are device addresses on the field's
 *  device; otherwise host arrays.
 * b2_pf_sensor_update_field: b2_pf_sensor_update's contract (DEVICE poses / attrs, HOST beams, merge per particle in beam order with the
 *  MAX_N_MEAS clamp, attrs read-modified-written once, enqueued on the handle's stream) with the error e = field(orig + dir * range), the
 *  closest-point branch's point; params.correspondence_type is ignored.  Where e equals the closest-point distance the evaluation is bit-equal
 *  to correspondence_type 1.  Elsewhere each beam's likelihood differs from it by at most exp(-1/2) / (dist_sigma * denom) * (sqrt(3)/2) h
 *  while d < trunc - (sqrt(3)/2) h, denom = sqrt(2 pi dist_sigma^2); beyond trunc the clamp moves an evaluation by at most
 *  exp(-trunc^2 / (2 dist_sigma^2)) / denom (exp(-4.5) / denom for trunc = 3 dist_sigma).  Refused (B2_ERR_INVALID, no launch): null h,
 *  f, Tsb or params, null buffers with n > 0 or n_beams > 0, a field on another device than the handle. */
typedef struct b2_dfield b2_dfield;
typedef struct { float resolution, truncation; const float* bb_min; const float* bb_max; } b2_dfield_params;               /* 24 B */
typedef char b2_dfield_params_is_24_bytes[sizeof(b2_dfield_params) == 24 ? 1 : -1];
typedef struct {
    uint32_t dims[3], brick_dims[3];          /* nodes / bricks per axis */
    float origin[3], resolution, inv_resolution, truncation;
    uint64_t bricks_total, bricks_allocated, bytes;
    float build_ms;                           /* wall time of b2_dfield_create */
    int device;
} b2_dfield_info;                                                                                                         /* 80 B */
typedef char b2_dfield_info_is_80_bytes[sizeof(b2_dfield_info) == 80 ? 1 : -1];
B2_API int b2_dfield_create(b2_mesh* map, const b2_dfield_params* params, b2_dfield** out);
B2_API int b2_dfield_destroy(b2_dfield* f);
B2_API int b2_dfield_get_info(const b2_dfield* f, b2_dfield_info* info);
B2_API int b2_dfield_download(const b2_dfield* f, uint32_t* index_host, float* bricks_host);
B2_API int b2_dfield_query(b2_dfield* f, const float* points_xyz, uint32_t n, float* dist_out, int src_is_device);
B2_API int b2_pf_sensor_update_field(b2_pf* h, const b2_dfield* f, const b2_transform* poses_dev, b2_particle_attr* attrs_dev, uint32_t n_particles,
                                     const b2_transform* Tsb, const b2_range_meas* beams_host, uint32_t n_beams, const b2_pf_params* params);

/* b2_pf_stein_update: `iterations` Stein variational gradient descent steps (SVGD, Liu & Wang 2016; the MegaParticles TODO of the reference's
 * docs/RMCL.md) that move the n particles toward the beams' likelihood over the field, in place, on the handle's stream, with no host round
 * trip between iterations (SURVEY appendix L states every operation).  Chart c = (x, y, psi), psi the ZYX yaw; a step moves x, y and turns
 * the pose about the world z axis through the body origin; z, roll and pitch stay (call b2_pf_project_to_surface after it on maps with
 * ramps).  Target: sum over beams of log((1 - w_rand) exp(-e^2 / (2 dist_sigma^2)) + w_rand), e = the field at the point
 * b2_pf_sensor_update_field looks up.  Each iteration scores a reference set J of m particles (all n in index order when n_ref == 0 or
 * n_ref >= n; else n_ref draws with replacement keyed by (seed, step, iteration)), sets the kernel bandwidth from the spread of the set, moves
 * every particle by the RMSProp-scaled kernel-weighted mean over J of score plus repulsion, and keeps a particle's pose for that iteration
 * where the motion update's wall check (a ray from the old to the new position) hits the map.  Attributes are not touched.
 * The result record (nullable out_host: one 32-byte copy and a synchronise): the last iteration's bandwidth (x, y, psi) and RMS step over
 * the finite particles (m, rad), m, and the blocked steps summed over all iterations.  n == 0 or iterations == 0: B2_OK, nothing launched
 * (out_host zeroed).  n_beams == 0: the score is 0, the particles only repel each other.  Refused (B2_ERR_INVALID, no launch):
 * b2_pf_sensor_update_field's checks, null cfg, a step or bandwidth floor not finite and > 0, w_rand outside [0, 1), dist_sigma not
 * finite and > 0.  Non-finite particles keep their pose and take no part in J's sums or the bandwidth. */
typedef struct { uint32_t iterations, n_ref; float step_t, step_r, min_bandwidth_t, min_bandwidth_r, w_rand, pad; } b2_stein_config;       /* 32 B */
typedef struct { float bandwidth[3]; uint32_t n_ref, n_blocked; float rms_step_t, rms_step_r, pad; } b2_stein_result;                      /* 32 B */
typedef char b2_stein_config_is_32_bytes[sizeof(b2_stein_config) == 32 ? 1 : -1];
typedef char b2_stein_result_is_32_bytes[sizeof(b2_stein_result) == 32 ? 1 : -1];
B2_API int b2_pf_stein_update(b2_pf* h, const b2_dfield* f, b2_transform* poses_dev, uint32_t n, const b2_transform* Tsb,
                              const b2_range_meas* beams_host, uint32_t n_beams, const b2_pf_params* params,
                              const b2_stein_config* cfg, uint64_t seed, uint32_t step, b2_stein_result* out_host /* nullable */);

/* ---------------------------------------------------------------- introspection ------------------------------ */
/* CUDA-event timing of the kernels inside b2_rcc_correct_once*(): when enabled, events are recorded on the handle's stream around the
 * find kernel and around the reduction/Umeyama kernels; b2_rcc_last_timing returns the two durations of the most recent call (ms). */
B2_API int b2_rcc_enable_timing(b2_rcc* h, int enable);
B2_API int b2_rcc_last_timing(b2_rcc* h, float* find_ms, float* reduce_ms);
/* the calling thread's pending CUDA runtime error as text ("" if none), without clearing it: no entry point of this library leaves one behind */
B2_API const char* b2_peek_cuda_error(void);
/* memory-system micro-benchmark for bench.py's roofline denominators: read bandwidth (GB/s) of a `bytes` working set, 128-bit loads from all SMs,
 * `iters` timed launches after a warm-up.  Below the L2 capacity it measures the L2, far above it the HBM. */
B2_API int b2_debug_read_bandwidth(int device, uint64_t bytes, int iters, double* gbytes_per_s);
/* number of kernels this library has launched in this process (bench.py's gpu_launches) */
B2_API uint64_t b2_kernel_launch_count(void);

#ifdef __cplusplus
}
#endif
#endif /* RMCL_B200_H */
