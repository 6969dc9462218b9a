// rcc_b200.hpp -- C++ host classes with the reference's names and signatures for the ray-casting-correspondence path, implemented over
// the C ABI (include/rmcl_b200.h).  These are what rmcl_ros' loadSensor / RmclNode would instantiate for a "b200" backend string
// (INTEGRATION.md).  Header-only; link with -lrmcl_b200.
//
//   rmcl::Correspondences_<MemT>            rmcl/include/rmcl/registration/Correspondences.hpp:16-88
//   rmcl::RCCB200{Spherical,Pinhole,O1Dn,OnDn}  twins of rmcl::RCCEmbree* / RCCOptix*  (RCCEmbree.hpp:18-83, RCCOptix.hpp:18-93)
//   rmcl::{Sphere,Pinhole,O1Dn,OnDn}CorrectorB200  v1 API used by rmcl_ros/src/benchmarks/lidar_corrector_{embree,optix}_benchmark.cpp:86-155
//   rmcl::PCDSensorUpdaterB200              rmcl_ros/include/rmcl_ros/rmcl/ParticleUpdater.hpp:39-43 + PCDSensorUpdaterEmbree.cpp:244-352
#pragma once
#include <array>
#include <memory>
#include <stdexcept>
#include <string>
#include <vector>

#include "../rmcl_b200.h"
#include "rmagine_compat.hpp"
#ifdef RMCL_B200_WITH_RMAGINE
// Built inside the reference's tree (or against an installed rmcl): the classes below DERIVE from the reference's own interface, so that
//   std::shared_ptr<rmcl::Correspondences_<rm::VRAM_CUDA>> correspondences_ = std::make_shared<rmcl::RCCB200Spherical>(map);
// compiles exactly like the OptiX line at rmcl_ros/src/nodes/micp_localization.cpp:616-626 (INTEGRATION.md).
#include <rmagine/types/MemoryCuda.hpp>
#include <rmagine/simulation/SimulationResults.hpp>
#include <rmcl/registration/Correspondences.hpp>          // rmcl/include/rmcl/registration/Correspondences.hpp:16-88
#ifdef RMCL_B200_WITH_RMCL_ROS
#include <rmcl_ros/rmcl/SensorUpdater.hpp>                 // rmcl_ros/include/rmcl_ros/rmcl/SensorUpdater.hpp:18-42, ParticleUpdater.hpp:24-43
#include <rmcl_ros/rmcl/RangeMeasurement.hpp>              // rmcl_ros/include/rmcl_ros/rmcl/RangeMeasurement.hpp:10-50
#endif
#define B2_OVERRIDE override
#else
#define B2_OVERRIDE
#endif

namespace rmcl {

namespace rm = rmagine;

// O1Dn / OnDn tables are rm::Memory<Vector, RAM> in rmagine, std::vector in the stand-alone layer
template <typename C> inline auto b2_table_ptr(const C& c) -> decltype(c.raw()) { return c.raw(); }
template <typename T> inline const T* b2_table_ptr(const std::vector<T>& c) { return c.data(); }

inline void b2_check(int rc, const char* what)
{
    // error convention of the reference: std::runtime_error for map / configuration failures (micp_localization.cpp:124, PCDSensorUpdaterEmbree.cpp:165)
    if (rc != B2_OK) throw std::runtime_error(std::string(what) + ": " + b2_last_error());
}

// stands in for rm::EmbreeMap / rm::OptixMap; shared between sensors and plugins like the reference's map container (micp_localization.cpp:545)
class B200Map {
public:
    B200Map(const float* verts_xyz, uint32_t n_vertices, const uint32_t* faces_ijk, uint32_t n_faces, int device = 0, int build_mode = B2_BUILD_DEVICE_LBVH)
    { b2_check(b2_mesh_create(verts_xyz, n_vertices, faces_ijk, n_faces, device, build_mode, &m_), "B200Map"); }
    // rm::import_embree_map(file) twin (micp_localization.cpp:188): .ply / .obj
    explicit B200Map(const std::string& mesh_file, int device = 0, int build_mode = B2_BUILD_DEVICE_LBVH)
    { b2_check(b2_mesh_create_from_file(mesh_file.c_str(), device, build_mode, &m_), "B200Map"); }
    ~B200Map() { b2_mesh_destroy(m_); }
    B200Map(const B200Map&) = delete; B200Map& operator=(const B200Map&) = delete;
    // the map's vertices moved (same faces): refit the resident BVH; dependants set their `outdated` flag like Correspondences.hpp:26-31
    void refit(const float* verts_xyz, uint32_t n_vertices, bool on_device = false) { b2_check(b2_mesh_refit(m_, verts_xyz, n_vertices, on_device ? 1 : 0), "B200Map::refit"); }
    b2_mesh* handle() const { return m_; }
    b2_mesh_info info() const { b2_mesh_info i; b2_check(b2_mesh_get_info(m_, &i), "B200Map::info"); return i; }
private:
    b2_mesh* m_ = nullptr;
};
using B200MapPtr = std::shared_ptr<B200Map>;

// truncated distance field of a map (b2_dfield_*; AMCL's likelihood field, no reference counterpart): built once on the map's device, a
// snapshot of the map (rebuild after B200Map::refit).  bb_min / bb_max null: the map's box grown by truncation.
class B200DistanceField {
public:
    B200DistanceField(B200MapPtr map, float resolution, float truncation, const float* bb_min = nullptr, const float* bb_max = nullptr) : map_(std::move(map))
    {
        if (!map_) throw std::runtime_error("NO MAP");
        const b2_dfield_params p{resolution, truncation, bb_min, bb_max};
        b2_check(b2_dfield_create(map_->handle(), &p, &f_), "B200DistanceField");
    }
    ~B200DistanceField() { b2_dfield_destroy(f_); }
    B200DistanceField(const B200DistanceField&) = delete; B200DistanceField& operator=(const B200DistanceField&) = delete;
    b2_dfield* handle() const { return f_; }
    b2_dfield_info info() const { b2_dfield_info i; b2_check(b2_dfield_get_info(f_, &i), "B200DistanceField::info"); return i; }
    // lookups of n points (xyz), synchronous; on_device: both arrays are device addresses
    void query(const float* points_xyz, uint32_t n, float* dist_out, bool on_device = false) { b2_check(b2_dfield_query(f_, points_xyz, n, dist_out, on_device ? 1 : 0), "B200DistanceField::query"); }
private:
    B200MapPtr map_;
    b2_dfield* f_ = nullptr;
};

// device-resident point cloud views (rm::PointCloudView_<VRAM_CUDA>)
struct PointCloudViewB200 { rm::MemoryView<rm::Vector3f, rm::VRAM_CUDA> points; rm::MemoryView<uint8_t, rm::VRAM_CUDA> mask; rm::MemoryView<rm::Vector3f, rm::VRAM_CUDA> normals; };

#if !(defined(RMCL_B200_WITH_RMAGINE) && defined(RMCL_B200_WITH_RMCL_ROS))
struct ParticleAttributes { rm::Gaussian1D likelihood; float state_sigma[6]; };                // ParticleAttributes.hpp:18-32
struct RangeMeasurement { rm::Vector3f orig, dir; float range; rm::Matrix3x3 cov; };            // RangeMeasurement.hpp:10-21
struct ParticleUpdateResults {};
struct ParticleUpdateConfig {};
struct ParticleUpdateDynamicResults { uint32_t n_particles; };                                    // ParticleUpdater.hpp:49-52
#endif
static_assert(sizeof(ParticleAttributes) == 36 && sizeof(RangeMeasurement) == 64, "rmcl layouts");

// --- Correspondences_ interface, device flavour --------------------------------------------------------------------------------
class CorrespondencesB200
#ifdef RMCL_B200_WITH_RMAGINE
    : public Correspondences_<rm::VRAM_CUDA>            // public: params, adaptive_max_dist_min, dataset, outdated; protected: model_buffers_, Tsb_
#endif
{
public:
#ifndef RMCL_B200_WITH_RMAGINE
    rm::UmeyamaReductionConstraints params{1.0f};      // Correspondences.hpp:22
    float adaptive_max_dist_min = 0.15f;               // :23
    bool outdated = true;                              // :31
#endif

    explicit CorrespondencesB200(B200MapPtr map) : map_(std::move(map))
    {
        if (!map_) throw std::runtime_error("NO MAP");                                           // PCDSensorUpdaterOptix.cpp:179-185
        b2_check(b2_rcc_create(map_->handle(), &h_), "RCCB200");
#ifdef RMCL_B200_WITH_RMAGINE
        params.max_dist = 1.0f; adaptive_max_dist_min = 0.15f;
#endif
    }
    virtual ~CorrespondencesB200() { b2_rcc_destroy(h_); }
    CorrespondencesB200(const CorrespondencesB200&) = delete; CorrespondencesB200& operator=(const CorrespondencesB200&) = delete;

    virtual void setTsb(const rm::Transform& Tsb) B2_OVERRIDE { Tsb_ = Tsb; b2_check(b2_rcc_set_tsb(h_, tf(&Tsb)), "setTsb"); }     // :33-36
    // Stand-alone builds: the public `dataset` field of the reference becomes two setters (the buffers live in HBM, owned by the handle).
    // rmagine builds: the inherited `dataset` member (rm::PointCloud_<VRAM_CUDA>, written directly by the sensor wrapper like
    // MICPSphericalSensorCUDA.cpp:230-232) is what find / computeCrossStatistics / correctOnce read -- bound, not copied; the setters below
    // stay available as the device-side unpackMessage and then take precedence until `dataset` is resized again.
    void setDataset(const rm::Vector3f* points, const uint8_t* mask, size_t n, bool on_device = false)
    { b2_check(b2_rcc_set_dataset(h_, reinterpret_cast<const float*>(points), mask, (uint32_t)n, on_device ? 1 : 0), "setDataset"); outdated = true; own_dataset_ = true; }
    void setRanges(const float* ranges, size_t n, bool on_device = false)                          // MICPSphericalSensorCPU.cpp:181-233 on the device
    { b2_check(b2_rcc_set_ranges(h_, ranges, (uint32_t)n, on_device ? 1 : 0), "setRanges"); outdated = true; own_dataset_ = true; }

    virtual void find(const rm::Transform& Tbm_est) B2_OVERRIDE                                    // :42-44
    { sync_params(); bind_members(); b2_check(b2_rcc_find(h_, tf(&Tbm_est)), "find"); outdated = false; }

    virtual rm::CrossStatistics computeCrossStatistics(const rm::Transform& T_snew_sold, double convergence_progress = 0.0) const B2_OVERRIDE   // :75-77
    {
        sync_params(); const_cast<CorrespondencesB200*>(this)->bind_members();
        rm::CrossStatistics out;
        b2_check(b2_rcc_cross_statistics(h_, tf(&T_snew_sold), convergence_progress, reinterpret_cast<b2_cross_stats*>(&out)), "computeCrossStatistics");
        return out;
    }
#ifndef RMCL_B200_WITH_RMAGINE            // rmagine builds inherit modelView() / datasetView() over model_buffers_ / dataset (Correspondences.hpp:47-62)
    PointCloudViewB200 modelView()                                                                 // :47-54
    {
        float *p = nullptr, *nr = nullptr; uint8_t* hi = nullptr; uint32_t n = 0;
        b2_check(b2_rcc_model_view(h_, &p, &nr, &hi, nullptr, nullptr, &n), "modelView");
        return PointCloudViewB200{{reinterpret_cast<rm::Vector3f*>(p), n}, {hi, n}, {reinterpret_cast<rm::Vector3f*>(nr), n}};
    }
    PointCloudViewB200 datasetView()                                                               // :56-62
    {
        float* p = nullptr; uint8_t* m = nullptr; uint32_t n = 0;
        b2_check(b2_rcc_dataset_view(h_, &p, &m, &n), "datasetView");
        return PointCloudViewB200{{reinterpret_cast<rm::Vector3f*>(p), n}, {m, n}, {nullptr, 0}};
    }
#endif
    // one MICPLocalizationNode::correctOnce for this sensor on the device (micp_localization.cpp:899-984)
    rm::Transform correctOnce(const rm::Transform& Tom, const rm::Transform& Tbo, unsigned iterations = 5, double convergence_progress = 0.0,
                              rm::Transform* T_onew_oold = nullptr, rm::CrossStatistics* Cmerged_o = nullptr)
    {
        sync_params(); bind_members();
        rm::Transform out;
        b2_check(b2_rcc_correct_once(h_, tf(&Tom), tf(&Tbo), iterations, convergence_progress, reinterpret_cast<b2_transform*>(&out),
                                     reinterpret_cast<b2_transform*>(T_onew_oold), reinterpret_cast<b2_cross_stats*>(Cmerged_o)), "correctOnce");
        outdated = false;
        return out;
    }
    // same, with the scan's ranges on the HOST (end-to-end entry): a pinned buffer is read in place by the kernel, a pageable one is uploaded
    rm::Transform correctOnceRanges(const float* ranges_host, size_t n, const rm::Transform& Tom, const rm::Transform& Tbo, unsigned iterations = 5,
                                    double convergence_progress = 0.0, rm::Transform* T_onew_oold = nullptr, rm::CrossStatistics* Cmerged_o = nullptr)
    {
        sync_params(); own_dataset_ = true;
        rm::Transform out;
        b2_check(b2_rcc_correct_once_ranges(h_, ranges_host, (uint32_t)n, tf(&Tom), tf(&Tbo), iterations, convergence_progress, reinterpret_cast<b2_transform*>(&out),
                                            reinterpret_cast<b2_transform*>(T_onew_oold), reinterpret_cast<b2_cross_stats*>(Cmerged_o)), "correctOnceRanges");
        outdated = false;
        return out;
    }
    // ScanMapSegmentationEmbreeNode::scanCB classification (scan_map_segmentation_embree.cpp:110-187): after setRanges(real scan) + find(pose)
    struct Segmentation { std::vector<rm::Vector3f> outlier_scan, outlier_map; };
    Segmentation segment(float min_dist_outlier_scan, float min_dist_outlier_map)
    {
        uint32_t n = 0, ns = 0, nm = 0;
        b2_check(b2_rcc_model_view(h_, nullptr, nullptr, nullptr, nullptr, nullptr, &n), "segment");
        Segmentation r; r.outlier_scan.resize(n); r.outlier_map.resize(n);
        b2_check(b2_rcc_segment(h_, min_dist_outlier_scan, min_dist_outlier_map, reinterpret_cast<float*>(r.outlier_scan.data()), n, &ns,
                                reinterpret_cast<float*>(r.outlier_map.data()), n, &nm, nullptr), "segment");
        r.outlier_scan.resize(ns); r.outlier_map.resize(nm);
        return r;
    }
    void setStream(void* cuda_stream) { b2_check(b2_rcc_set_stream(h_, cuda_stream), "setStream"); }
    b2_rcc* handle() const { return h_; }
    friend void micp_correct(const std::vector<CorrespondencesB200*>& sensors, const std::vector<rm::Transform>& Tbo, const std::vector<double>& merge_weights,
                             rm::Transform& Tom, double& convergence_progress, bool adaptive_max_dist, unsigned n_corrections, unsigned iterations,
                             std::vector<b2_micp_step>* steps);
    void noteModelSize(uint32_t width, uint32_t height) { note_model(width, height); }      // for model tables set through the C ABI directly (rmcl_msgs_adapters.hpp)

protected:
    static const b2_transform* tf(const rm::Transform* T) { return reinterpret_cast<const b2_transform*>(T); }
    void sync_params() const { b2_rcc_set_params(h_, params.max_dist, adaptive_max_dist_min); }
    // model size of the sensor model last given to setModel (RCCOptix keeps a model_cache_ for the same purpose, RCCOptix.hpp:39)
    void note_model(uint32_t width, uint32_t height) { model_w_ = width; model_h_ = height; }
#ifdef RMCL_B200_WITH_RMAGINE
    // Point the handle at the members the reference's interface exposes: model_buffers_ grown like RCCOptix.cpp:30-40 and bound as the find()
    // output, `dataset` bound as the reduction input (unless the device-side unpack of setRanges / setDataset is in charge).
    void bind_members()
    {
        const size_t n = size_t(model_w_) * model_h_;
        if (n > 0) {
            if (n > model_buffers_.points.size()) rm::resize_memory_bundle<rm::VRAM_CUDA>(model_buffers_, model_h_, model_w_, 1);
            b2_check(b2_rcc_bind_model_buffers(h_, reinterpret_cast<float*>(model_buffers_.points.raw()), reinterpret_cast<float*>(model_buffers_.normals.raw()),
                                               model_buffers_.hits.raw(), (uint32_t)model_buffers_.points.size()), "bind model_buffers_");
        }
        if (dataset.points.size() > 0 && (!own_dataset_ || dataset.points.raw() != bound_dataset_ || dataset.points.size() != bound_n_)) {
            if (dataset.mask.size() < dataset.points.size()) throw std::runtime_error("dataset.mask smaller than dataset.points");
            b2_check(b2_rcc_bind_dataset(h_, reinterpret_cast<const float*>(dataset.points.raw()), dataset.mask.raw(), (uint32_t)dataset.points.size()), "bind dataset");
            bound_dataset_ = dataset.points.raw(); bound_n_ = dataset.points.size(); own_dataset_ = false;
        }
    }
    const void* bound_dataset_ = nullptr; size_t bound_n_ = 0;
#else
    void bind_members() {}
    rm::Transform Tsb_ = rm::Transform::Identity();
#endif
    bool own_dataset_ = false;
    uint32_t model_w_ = 0, model_h_ = 0;
    B200MapPtr map_;
    b2_rcc* h_ = nullptr;
};

class RCCB200Spherical : public CorrespondencesB200, public rm::ModelSetter<rm::SphericalModel> {
public:
    explicit RCCB200Spherical(B200MapPtr map) : CorrespondencesB200(std::move(map)) {}
    void setModel(const rm::SphericalModel& m) override                                           // RCCEmbree.cpp:21-24
    {
        b2_spherical_model s{m.phi.min, m.phi.inc, m.phi.size, m.theta.min, m.theta.inc, m.theta.size, m.range.min, m.range.max};
        b2_check(b2_rcc_set_model_spherical(h_, &s), "setModel"); note_model(m.theta.size, m.phi.size);
    }
    // Pc2ToScanNode::convert + fillEmpty + unpackMessage (pc2_to_scan.cpp:105-213, scan_operations.cpp:25-39, MICPSphericalSensorCUDA.cpp:176-235)
    // on the device: a PointCloud2's bytes binned into the model of the last setModel as this sensor's dataset (b2_rcc_set_cloud_spherical)
    void setPointCloud(const void* data, size_t bytes, const b2_cloud_layout& layout, const rm::Transform& T_sensor_cloud, bool on_device = false)
    {
        b2_check(b2_rcc_set_cloud_spherical(h_, data, bytes, &layout, tf(&T_sensor_cloud), on_device ? 1 : 0), "setPointCloud");
        outdated = true; own_dataset_ = true;
    }
};
class RCCB200Pinhole : public CorrespondencesB200, public rm::ModelSetter<rm::PinholeModel> {
public:
    explicit RCCB200Pinhole(B200MapPtr map) : CorrespondencesB200(std::move(map)) {}
    void setModel(const rm::PinholeModel& m) override                                             // RCCEmbree.cpp:53-56
    {
        b2_pinhole_model p{m.width, m.height, m.f[0], m.f[1], m.c[0], m.c[1], m.range.min, m.range.max};
        b2_check(b2_rcc_set_model_pinhole(h_, &p), "setModel"); note_model(m.width, m.height);
    }
};
class RCCB200O1Dn : public CorrespondencesB200, public rm::ModelSetter<rm::O1DnModel> {
public:
    explicit RCCB200O1Dn(B200MapPtr map) : CorrespondencesB200(std::move(map)) {}
    void setModel(const rm::O1DnModel& m) override                                                // RCCEmbree.cpp:84-87
    { b2_check(b2_rcc_set_model_o1dn(h_, m.width, m.height, &m.orig.x, reinterpret_cast<const float*>(b2_table_ptr(m.dirs)), m.range.min, m.range.max), "setModel"); note_model(m.width, m.height); }
    // Pc2ToO1DnNode::convert + unpackMessage + setModel (conversions.cpp:869-1073, scan_operations.cpp:41-143, MICPO1DnSensorCUDA.cpp:142-148,171-230)
    // on the device: an organised PointCloud2's bytes become this sensor's model and dataset (b2_rcc_set_cloud_o1dn)
    void setPointCloud(const void* data, size_t bytes, const b2_cloud_layout& layout, const b2_o1dn_cloud_filter& filter, bool on_device = false)
    {
        b2_check(b2_rcc_set_cloud_o1dn(h_, data, bytes, &layout, &filter, on_device ? 1 : 0), "setPointCloud");
        note_model((layout.width - filter.width_skip_begin - filter.width_skip_end) / filter.width_increment,
                   (layout.height - filter.height_skip_begin - filter.height_skip_end) / filter.height_increment);
        outdated = true; own_dataset_ = true;
    }
};
class RCCB200OnDn : public CorrespondencesB200, public rm::ModelSetter<rm::OnDnModel> {
public:
    explicit RCCB200OnDn(B200MapPtr map) : CorrespondencesB200(std::move(map)) {}
    void setModel(const rm::OnDnModel& m) override                                                // RCCEmbree.cpp:116-119
    {
        b2_check(b2_rcc_set_model_ondn(h_, m.width, m.height, reinterpret_cast<const float*>(b2_table_ptr(m.origs)), reinterpret_cast<const float*>(b2_table_ptr(m.dirs)),
                                       m.range.min, m.range.max), "setModel");
        note_model(m.width, m.height);
    }
};

// rmcl::CPCEmbree twin (rmcl/include/rmcl/registration/CPCEmbree.hpp:20-54): closest-point correspondences on the same map BVH.
// find() = one closest-point query per dataset point (CPCEmbree.cpp:17-43); no sensor model.
class CPCB200 : public CorrespondencesB200 {
public:
    explicit CPCB200(B200MapPtr map) : CorrespondencesB200(std::move(map)) { b2_check(b2_rcc_set_correspondence_type(h_, B2_CORR_CPC), "CPCB200"); }
#ifdef RMCL_B200_WITH_RMAGINE
    void find(const rm::Transform& Tbm_est) override                     // CPCEmbree.cpp:17-43: one model entry per dataset point
    { note_model((uint32_t)dataset.points.size(), dataset.points.size() ? 1u : 0u); CorrespondencesB200::find(Tbm_est); }
#endif
};

// --- v1 batched corrector API (lidar_corrector_embree_benchmark.cpp:86-133) -------------------------------------------------------
struct CorrectionResultsB200 { std::vector<rm::Transform> Tdelta; std::vector<uint32_t> Ncorr; };
struct BenchmarkResultB200 { double sim = 0.0, red = 0.0, svd = 0.0; };                          // lidar_corrector_optix_benchmark.cpp:143-155
template <typename RCC> class CorrectorB200 : public RCC {
public:
    using RCC::RCC;
    // v1 simulate(Tbm, ranges): trace the sensor at Tbm and hand out the simulated ranges (HOST buffer of model-size floats; :117)
    void simulate(const rm::Transform& Tbm, float* ranges_host)
    {
        this->find(Tbm);
        uint32_t n = 0;
        b2_check(b2_rcc_model_view(this->h_, nullptr, nullptr, nullptr, nullptr, nullptr, &n), "simulate");
        b2_check(b2_rcc_download_model(this->h_, nullptr, nullptr, nullptr, nullptr, ranges_host), "simulate");
    }
    // v1 benchmark(Tbm, Nruns) -> {sim, red, svd} seconds: the stages of correct() run unfused and timed separately (:143-155)
    BenchmarkResultB200 benchmark(const std::vector<rm::Transform>& Tbm, size_t Nruns = 100)
    {
        this->sync_params();
        BenchmarkResultB200 r;
        b2_check(b2_rcc_benchmark_batch(this->h_, reinterpret_cast<const b2_transform*>(Tbm.data()), (uint32_t)Tbm.size(), (uint32_t)Nruns, &r.sim, &r.red, &r.svd), "benchmark");
        return r;
    }
    void setInputData(const float* ranges, size_t n, bool on_device = false) { this->setRanges(ranges, n, on_device); }       // :118
    CorrectionResultsB200 correct(const std::vector<rm::Transform>& Tbm)                                                       // :127-133
    {
        this->sync_params();
        CorrectionResultsB200 r; r.Tdelta.resize(Tbm.size()); r.Ncorr.resize(Tbm.size());
        b2_check(b2_rcc_correct_batch(this->h_, reinterpret_cast<const b2_transform*>(Tbm.data()), (uint32_t)Tbm.size(), 0,
                                      reinterpret_cast<b2_transform*>(r.Tdelta.data()), r.Ncorr.data(), nullptr, 0), "correct");
        return r;
    }
};
using SphereCorrectorB200 = CorrectorB200<RCCB200Spherical>;
using PinholeCorrectorB200 = CorrectorB200<RCCB200Pinhole>;
using O1DnCorrectorB200 = CorrectorB200<RCCB200O1Dn>;
using OnDnCorrectorB200 = CorrectorB200<RCCB200OnDn>;

inline rm::Transform umeyama_transform(const rm::CrossStatistics& s, int device = 0)              // micp_localization.cpp:952-953
{
    rm::Transform T;
    b2_check(b2_umeyama_batch(reinterpret_cast<const b2_cross_stats*>(&s), 1, reinterpret_cast<b2_transform*>(&T), 0, device, nullptr), "umeyama_transform");
    return T;
}

// MICPLocalizationNode::correct() (micp_localization.cpp:847-854) / the body of correctionLoop (:1086-1171): n_corrections x correctOnce on the
// device for all sensors of the node, Tom_ and convergence_progress_ (:988-1007) carried between the steps on the device and updated here at the
// end.  merge_weights empty = all 1.0; steps (may be null) receives one record per correction (the fields of MICPSensorStats, :1009-1015).
inline void micp_correct(const std::vector<CorrespondencesB200*>& sensors, const std::vector<rm::Transform>& Tbo, const std::vector<double>& merge_weights,
                         rm::Transform& Tom, double& convergence_progress, bool adaptive_max_dist = true, unsigned n_corrections = 3, unsigned iterations = 5,
                         std::vector<b2_micp_step>* steps = nullptr)
{
    if (sensors.size() != Tbo.size() || (!merge_weights.empty() && merge_weights.size() != sensors.size())) throw std::invalid_argument("micp_correct: one Tbo / weight per sensor");
    std::vector<b2_rcc*> h;
    for (CorrespondencesB200* s : sensors) { s->sync_params(); s->bind_members(); h.push_back(s->h_); }
    if (steps) steps->resize(n_corrections);
    b2_check(b2_micp_correct(h.data(), reinterpret_cast<const b2_transform*>(Tbo.data()), merge_weights.empty() ? nullptr : merge_weights.data(), (uint32_t)h.size(),
                             reinterpret_cast<b2_transform*>(&Tom), &convergence_progress, adaptive_max_dist ? 1 : 0, n_corrections, iterations,
                             steps ? steps->data() : nullptr), "micp_correct");
    for (CorrespondencesB200* s : sensors) s->outdated = false;
}

// The covariance of the correction that just ran on `sensors` (b2_micp_pose_covariance: point-to-plane information of the final correspondences),
// about Tom_new * Tbo_ref in its body frame (Tbo_ref null: Tbo[0]), x y z roll pitch yaw: what publishPose (micp_localization.cpp:1053-1084)
// puts into PoseWithCovariance.  After micp_correct pass steps.back().T_onew_oold and the progress that step gated with (the input progress for
// one step, else steps[n - 2].convergence_progress).
inline b2_micp_covariance micp_pose_covariance(const std::vector<CorrespondencesB200*>& sensors, const std::vector<rm::Transform>& Tbo,
                                               const std::vector<double>& merge_weights, const rm::Transform& T_onew_oold, double convergence_progress,
                                               const rm::Transform* Tbo_ref = nullptr, b2_micp_cov_config cfg = {1e-3, 1e2})
{
    if (sensors.size() != Tbo.size() || (!merge_weights.empty() && merge_weights.size() != sensors.size())) throw std::invalid_argument("micp_pose_covariance: one Tbo / weight per sensor");
    std::vector<b2_rcc*> h;
    for (CorrespondencesB200* s : sensors) h.push_back(s->handle());
    b2_micp_covariance out;
    b2_check(b2_micp_pose_covariance(h.data(), reinterpret_cast<const b2_transform*>(Tbo.data()), merge_weights.empty() ? nullptr : merge_weights.data(),
                                     (uint32_t)h.size(), reinterpret_cast<const b2_transform*>(&T_onew_oold), convergence_progress,
                                     reinterpret_cast<const b2_transform*>(Tbo_ref), &cfg, &out), "micp_pose_covariance");
    return out;
}

// --- particle filter sensor update ------------------------------------------------------------------------------------------------
class PCDSensorUpdaterB200
#if defined(RMCL_B200_WITH_RMAGINE) && defined(RMCL_B200_WITH_RMCL_ROS)
    : public SensorUpdater<rm::VRAM_CUDA>               // = SensorUpdaterBase (init / reset) + ParticleUpdater<VRAM_CUDA> (update), SensorUpdater.hpp:37-42
#define B2_PF_OVERRIDE override
#else
#define B2_PF_OVERRIDE
#endif
{
public:
    // SensorUpdaterBase::init / reset (SensorUpdater.hpp:18-25).  The Embree updater loads its map in init() (PCDSensorUpdaterEmbree.cpp:136-189);
    // here the map arrives through the constructor, so init() only checks it and reset() drops the input cloud and the beams.
    void init() B2_PF_OVERRIDE { if (!map_) throw std::runtime_error("NO MAP"); }
    void reset() B2_PF_OVERRIDE { beams_.clear(); input_ = CloudInput{}; }
    b2_pf_params config{2.0f, 100.0f, 100.0f, 0.0f, 0.05f, 80.0f, 0, 0};                         // PCDSensorUpdaterEmbree.cpp:122-134
    // beam sampling from the input cloud (b2_pf_sample_cloud): `samples` per update (PCDSensorUpdaterEmbree.cpp:124), drawn with (seed, step);
    // every update that samples advances step.  Set seed once (e.g. from the clock); every rank of a sharded set must use the same seed and step.
    uint32_t samples = 100;
    uint64_t seed = 0;
    uint32_t step = 0;
    explicit PCDSensorUpdaterB200(B200MapPtr map) : map_(std::move(map))
    {
        if (!map_) throw std::runtime_error("NO MAP");
        b2_check(b2_pf_create(map_->handle(), &h_), "PCDSensorUpdaterB200");
    }
    ~PCDSensorUpdaterB200() { b2_pf_destroy(h_); }
    void setTsb(const rm::Transform& Tsb) { Tsb_ = Tsb; }
    // Input<PointCloud2::ConstSharedPtr>::setInput (rmcl_localization.cpp:512-530): the PointCloud2 bytes both update()s sample their beams
    // from (PCDSensorUpdaterOptix.cpp:227-311).  The bytes are read when update() runs: keep_alive holds their owner until the next
    // setInput / setBeams / reset.  on_device: `data` is a device address, read in place by a kernel.  Replaces beams set by setBeams.
    void setInput(const void* data, uint64_t bytes, const b2_cloud_layout& layout, bool on_device, std::shared_ptr<const void> keep_alive = {})
    {
        input_ = CloudInput{true, data, bytes, layout, on_device, std::move(keep_alive)};
        beams_.clear();
    }
    // beams passed as they are (quirk D5: the caller samples the cloud into RangeMeasurements); replaces the input cloud
    void setBeams(const std::vector<RangeMeasurement>& beams) { beams_ = beams; input_ = CloudInput{}; }
    // how rays are mapped to lanes (a schedule, results identical): 0 beams of one particle, 1 particles, 2 particles sorted by pose, 3 (default) by timing
    void setMapping(int mode) { b2_check(b2_pf_set_mapping(h_, mode), "setMapping"); }
    // likelihood field: while a field is set, the VRAM update() evaluates each beam from it (b2_pf_sensor_update_field) instead of tracing the
    // map, and the RAM update() throws.  The updater keeps the field alive; nullptr returns to the map.
    void setDistanceField(std::shared_ptr<B200DistanceField> field) { field_ = std::move(field); }
    // ParticleUpdater<RAM>::update
    ParticleUpdateResults update(rm::MemoryView<rm::Transform, rm::RAM> poses, rm::MemoryView<ParticleAttributes, rm::RAM> attrs, const ParticleUpdateConfig& = {})
    {
        if (field_) throw std::runtime_error("update: a distance field is set; the field update takes device particles only");
        const uint32_t n = particle_count("update", poses, attrs);
        sample_input();
        b2_check(b2_pf_sensor_update_host(h_, reinterpret_cast<const b2_transform*>(poses.raw()), reinterpret_cast<b2_particle_attr*>(attrs.raw()), n,
                                          reinterpret_cast<const b2_transform*>(&Tsb_), reinterpret_cast<const b2_range_meas*>(beams_.data()), (uint32_t)beams_.size(), &config), "update");
        return {};
    }
    // ParticleUpdater<VRAM_CUDA>::update (ParticleUpdater.hpp:39-43)
    ParticleUpdateResults update(rm::MemoryView<rm::Transform, rm::VRAM_CUDA> poses, rm::MemoryView<ParticleAttributes, rm::VRAM_CUDA> attrs, const ParticleUpdateConfig& = {}) B2_PF_OVERRIDE
    {
        const uint32_t n = particle_count("update", poses, attrs);
        sample_input();
        if (field_) {
            b2_check(b2_pf_sensor_update_field(h_, field_->handle(), reinterpret_cast<const b2_transform*>(poses.raw()), reinterpret_cast<b2_particle_attr*>(attrs.raw()),
                                               n, reinterpret_cast<const b2_transform*>(&Tsb_), reinterpret_cast<const b2_range_meas*>(beams_.data()),
                                               (uint32_t)beams_.size(), &config), "update");
            return {};
        }
        b2_check(b2_pf_sensor_update(h_, reinterpret_cast<const b2_transform*>(poses.raw()), reinterpret_cast<b2_particle_attr*>(attrs.raw()), n,
                                     reinterpret_cast<const b2_transform*>(&Tsb_), reinterpret_cast<const b2_range_meas*>(beams_.data()), (uint32_t)beams_.size(), &config), "update");
        return {};
    }
    // rest of the cycle on the device (particles stay in HBM): TFMotionUpdaterGPU (particle_motion.cu:36-46) and compute_stats (resampling.cu:84-92)
    void motionUpdate(rm::MemoryView<rm::Transform, rm::VRAM_CUDA> poses, rm::MemoryView<ParticleAttributes, rm::VRAM_CUDA> attrs, const rm::Transform& T_bnew_bold, double forget_rate,
                      bool check_collision = false)       // true: the wall check of TFMotionUpdaterCPU (TFMotionUpdaterCPU.cpp:205-216)
    {
        b2_check(b2_pf_motion_update(h_, reinterpret_cast<b2_transform*>(poses.raw()), reinterpret_cast<b2_particle_attr*>(attrs.raw()), particle_count("motionUpdate", poses, attrs),
                                     reinterpret_cast<const b2_transform*>(&T_bnew_bold), forget_rate, check_collision ? 1 : 0), "motionUpdate");
    }
    // The surface-constrained motion update of docs/RMCL.md:72 (b2_pf_project_to_surface): each particle is put on the walkable surface
    // under it, in place; one with no such surface in the probe window gets the likelihood {0, 0, MAX_N_MEAS}.  Call it after motionUpdate,
    // after initSamplesUniform and after resampling.  surface_config() gives the suggested values.
    static b2_surface_config surface_config() { return b2_surface_config{0.5f, 1.0f, 0.0f, 0.6f, 1}; }
    void projectToSurface(rm::MemoryView<rm::Transform, rm::VRAM_CUDA> poses, rm::MemoryView<ParticleAttributes, rm::VRAM_CUDA> attrs,
                          const b2_surface_config& cfg = surface_config())
    {
        b2_check(b2_pf_project_to_surface(h_, reinterpret_cast<b2_transform*>(poses.raw()), reinterpret_cast<b2_particle_attr*>(attrs.raw()),
                                          particle_count("projectToSurface", poses, attrs), &cfg),
                 "projectToSurface");
    }
    // Where on the map does the scan fit best (b2_pf_global_search; SURVEY appendix M): every pose of cfg's (x, y, yaw) grid scored from
    // `field` as the field update scores a particle there from {0, 0, 0} (with this updater's Tsb and config), the local maxima of the
    // scores ranked and separated.  surface (may be null) puts the candidates where projectToSurface would; scores_dev (may be null, n_candidates
    // device floats) receives the likelihood map.  Returns the kept peaks, best first; result (may be null) receives the counts.  Synchronises.
    // search_config(...) gives the suggested values over an (x, y) box.
    static b2_search_config search_config(float x_min, float y_min, float x_max, float y_max, float z0, float step = 0.25f)
    {
        return b2_search_config{x_min, y_min, z0, step, (uint32_t)((x_max - x_min) / step) + 1u, (uint32_t)((y_max - y_min) / step) + 1u, 72u, 8u, 1.0f,
                                0.52359878f};
    }
    std::vector<b2_search_record> globalSearch(const B200DistanceField& field, const b2_range_meas* beams, uint32_t n_beams, const b2_search_config& cfg,
                                               const b2_surface_config* surface = nullptr, float* scores_dev = nullptr, b2_search_result* result = nullptr)
    {
        std::vector<b2_search_record> recs(cfg.max_records >= 1 && cfg.max_records <= 64 ? cfg.max_records : 1);
        b2_search_result r{};
        b2_check(b2_pf_global_search(h_, field.handle(), reinterpret_cast<const b2_transform*>(&Tsb_), beams, n_beams, &config, &cfg, surface, recs.data(),
                                     scores_dev, &r), "globalSearch");
        recs.resize(r.n_records);
        if (result) *result = r;
        return recs;
    }
    // globalSearch's records on grids too large or too fine to score exhaustively (b2_pf_global_search_bnb; SURVEY appendix N): an exact
    // branch and bound over a min-pooled pyramid of the field.  Returns globalSearch's records whose score is >= min_ratio times the best,
    // in the same order (min_ratio 0: all of them); result (may be null) receives the search's counts.  Synchronises.
    std::vector<b2_search_record> globalSearchBnB(const B200DistanceField& field, const b2_range_meas* beams, uint32_t n_beams, const b2_search_config& cfg,
                                                  const b2_surface_config* surface = nullptr, float min_ratio = 0.0f, b2_search_bnb_result* result = nullptr)
    {
        std::vector<b2_search_record> recs(cfg.max_records >= 1 && cfg.max_records <= 64 ? cfg.max_records : 1);
        b2_search_bnb_result r{};
        b2_check(b2_pf_global_search_bnb(h_, field.handle(), reinterpret_cast<const b2_transform*>(&Tsb_), beams, n_beams, &config, &cfg, surface, min_ratio,
                                         recs.data(), &r), "globalSearchBnB");
        recs.resize(r.n_records);
        if (result) *result = r;
        return recs;
    }
    // Stein variational steps toward the beams' likelihood over the field of setDistanceField (b2_pf_stein_update; SURVEY appendix L): in
    // place on the device poses, on the handle's stream; x, y and yaw move, z, roll, pitch and the attributes stay.  Throws without a field.
    // Returns the result record (a 32-byte read-back and a synchronise).  stein_config() gives the suggested values.
    static b2_stein_config stein_config() { return b2_stein_config{10u, 4096u, 0.02f, 0.01f, 0.05f, 0.02f, 0.05f, 0.0f}; }
    b2_stein_result steinUpdate(rm::MemoryView<rm::Transform, rm::VRAM_CUDA> poses, const b2_range_meas* beams, uint32_t n_beams,
                                const b2_stein_config& cfg = stein_config(), uint64_t seed = 0, uint32_t step = 0)
    {
        if (!field_) throw std::runtime_error("steinUpdate: no distance field (setDistanceField first)");
        b2_stein_result r{};
        b2_check(b2_pf_stein_update(h_, field_->handle(), reinterpret_cast<b2_transform*>(poses.raw()), (uint32_t)poses.size(),
                                    reinterpret_cast<const b2_transform*>(&Tsb_), beams, n_beams, &config, &cfg, seed, step, &r), "steinUpdate");
        return r;
    }
    // The same steps on a particle set sharded over GPUs (b2_pf_stein_slice_*; SURVEY L14), for a node with its own communicator: steinBegin
    // opens this rank's session (its slice [first, first + n_local) of n_all, its range [j_first, j_first + j_count) of J's m references;
    // uploads the beams, a synchronise).  Per iteration k the caller all-gathers the poses into poses_all, calls steinScore(poses_all, k,
    // snap) (j_count entries), all-gathers the snapshots in J's order into snap_all (m entries), then steinMove(poses_all, snap_all, k,
    // out) (n_local poses; out may be poses_all + first).  Both only launch on the handle's stream.  steinResult reads the record (a
    // synchronise).  The slices concatenated equal steinUpdate of the whole set byte for byte.  Throws on a call out of sequence.
    void steinBegin(uint32_t n_all, uint32_t first, uint32_t n_local, uint32_t j_first, uint32_t j_count, const b2_range_meas* beams, uint32_t n_beams,
                    const b2_stein_config& cfg = stein_config(), uint64_t seed = 0, uint32_t step = 0)
    {
        if (!field_) throw std::runtime_error("steinBegin: no distance field (setDistanceField first)");
        b2_check(b2_pf_stein_slice_begin(h_, field_->handle(), n_all, first, n_local, j_first, j_count, reinterpret_cast<const b2_transform*>(&Tsb_), beams,
                                         n_beams, &config, &cfg, seed, step), "steinBegin");
    }
    void steinScore(rm::MemoryView<rm::Transform, rm::VRAM_CUDA> poses_all, uint32_t iteration, b2_stein_ref* snap_dev)
    {
        b2_check(b2_pf_stein_slice_score(h_, reinterpret_cast<const b2_transform*>(poses_all.raw()), iteration, snap_dev), "steinScore");
    }
    void steinMove(rm::MemoryView<rm::Transform, rm::VRAM_CUDA> poses_all, const b2_stein_ref* snap_all_dev, uint32_t iteration,
                   rm::MemoryView<rm::Transform, rm::VRAM_CUDA> poses_out)
    {
        b2_check(b2_pf_stein_slice_move(h_, reinterpret_cast<const b2_transform*>(poses_all.raw()), snap_all_dev, iteration,
                                        reinterpret_cast<b2_transform*>(poses_out.raw())), "steinMove");
    }
    b2_stein_slice_result steinResult()
    {
        b2_stein_slice_result r{};
        b2_check(b2_pf_stein_slice_result(h_, &r), "steinResult");
        return r;
    }
    // Recovery from a kidnapping (Augmented MCL, b2_pf_recovery_*): recoveryObserve after each update keeps a slow and a fast average of the
    // set's mean likelihood at recovery_config's rates (AMCL's recovery_alpha_slow / _fast); recoveryInject after resampling replaces a
    // fraction p_inject = max(0, 1 - w_fast / w_slow) of the particles with random poses of the box (on the map's ground when `surface` is
    // given).  Call recoveryReset after (re)initialising the set.  With want_state / want_result the call reads the record back into
    // last_recovery_state / last_recovery and synchronises; otherwise it only enqueues.
    b2_recovery_config recovery_config{0.001, 0.1};
    b2_recovery_state last_recovery_state{};
    b2_recovery_result last_recovery{};
    void recoveryReset() { b2_check(b2_pf_recovery_reset(h_), "recoveryReset"); }
    void recoveryObserve(rm::MemoryView<ParticleAttributes, rm::VRAM_CUDA> attrs, bool want_state = false)
    {
        b2_check(b2_pf_recovery_observe(h_, reinterpret_cast<const b2_particle_attr*>(attrs.raw()), (uint32_t)attrs.size(), &recovery_config,
                                        want_state ? &last_recovery_state : nullptr), "recoveryObserve");
    }
    void recoveryInject(rm::MemoryView<rm::Transform, rm::VRAM_CUDA> poses, rm::MemoryView<ParticleAttributes, rm::VRAM_CUDA> attrs,
                        const std::array<double, 6>& bb_min, const std::array<double, 6>& bb_max, const b2_surface_config* surface = nullptr,
                        uint32_t max_tries = 16, uint64_t seed = 1234, uint32_t step = 0, uint32_t first = 0, bool want_result = false)
    {
        b2_check(b2_pf_recovery_inject(h_, reinterpret_cast<b2_transform*>(poses.raw()), reinterpret_cast<b2_particle_attr*>(attrs.raw()), first,
                                       particle_count("recoveryInject", poses, attrs),
                                       bb_min.data(), bb_max.data(), surface, max_tries, seed, step, want_result ? &last_recovery : nullptr), "recoveryInject");
    }
    struct SimpleLikelihoodStats { float sum = 0.0f; float max = -1.0f; };                       // resampling.cuh:26-30
    SimpleLikelihoodStats computeStats(rm::MemoryView<ParticleAttributes, rm::VRAM_CUDA> attrs)
    {
        SimpleLikelihoodStats s;
        b2_check(b2_pf_likelihood_stats(h_, reinterpret_cast<const b2_particle_attr*>(attrs.raw()), (uint32_t)attrs.size(), &s.sum, &s.max), "computeStats");
        return s;
    }
    // GladiatorResamplerGPU::resample (resampling.cu:201-221; config GladiatorResamplerConfig.hpp:7-20).  `poses/attrs` = all particles
    // opponents are drawn from; the outputs receive champions first .. first+poses_new.size()-1 (single GPU: first = 0, same sizes).
    b2_gladiator_config resampler_config{0.03f, 0.03f, 0.0f, 0.0f, 0.0f, 0.01f, 0.3f, 0.2f};
    void resample(rm::MemoryView<rm::Transform, rm::VRAM_CUDA> poses, rm::MemoryView<ParticleAttributes, rm::VRAM_CUDA> attrs,
                  rm::MemoryView<rm::Transform, rm::VRAM_CUDA> poses_new, rm::MemoryView<ParticleAttributes, rm::VRAM_CUDA> attrs_new,
                  uint64_t seed = 1234, uint32_t step = 0, uint32_t first = 0)
    {
        const uint32_t n_all = particle_count("resample", poses, attrs), n_local = particle_count("resample", poses_new, attrs_new);
        b2_check(b2_pf_resample_gladiator(h_, reinterpret_cast<const b2_transform*>(poses.raw()), reinterpret_cast<const b2_particle_attr*>(attrs.raw()), n_all,
                                          first, n_local, reinterpret_cast<b2_transform*>(poses_new.raw()), reinterpret_cast<b2_particle_attr*>(attrs_new.raw()),
                                          &resampler_config, seed, step, nullptr, nullptr), "resample");
    }
    // ResidualResamplerCPU::update (ResidualResamplerCPU.cpp:55-202; config and defaults :35-47) on the device: all of `poses/attrs` resampled
    // into an output set of n_new slots (0: first + poses_new.size(), the node's whole max_particles buffer); the outputs receive slots
    // first .. first+poses_new.size()-1, and only those below the returned n_particles are written.  `last_residual` keeps the whole record.
    b2_residual_config residual_config{0.03f, 0.03f, 0.0f, 0.0f, 0.0f, 0.01f, 0.3f, 0.2f};
    b2_residual_result last_residual{};
    ParticleUpdateDynamicResults resampleResidual(rm::MemoryView<rm::Transform, rm::VRAM_CUDA> poses, rm::MemoryView<ParticleAttributes, rm::VRAM_CUDA> attrs,
                                                  rm::MemoryView<rm::Transform, rm::VRAM_CUDA> poses_new, rm::MemoryView<ParticleAttributes, rm::VRAM_CUDA> attrs_new,
                                                  uint64_t seed = 1234, uint32_t step = 0, uint32_t first = 0, uint32_t n_new = 0)
    {
        const uint32_t n = particle_count("resampleResidual", poses, attrs), n_local = particle_count("resampleResidual", poses_new, attrs_new);
        if (n_new == 0) n_new = first + n_local;
        b2_check(b2_pf_resample_residual(h_, reinterpret_cast<const b2_transform*>(poses.raw()), reinterpret_cast<const b2_particle_attr*>(attrs.raw()), n,
                                         n_new, first, n_local, reinterpret_cast<b2_transform*>(poses_new.raw()),
                                         reinterpret_cast<b2_particle_attr*>(attrs_new.raw()), &residual_config, seed, step, &last_residual), "resampleResidual");
        ParticleUpdateDynamicResults res;
        res.n_particles = (uint32_t)last_residual.n_particles;
        return res;
    }
    // KLD-sampling (Fox 2003; the open TODO of docs/RMCL.md:80-83) on the device (b2_pf_resample_kld): all of `poses/attrs` resampled into at
    // most n_max slots (0: first + poses_new.size(), the node's whole max_particles buffer), as many as the bins of the drawn set call for;
    // the outputs receive slots first .. first+poses_new.size()-1, and only those below the returned n_particles are written.  The copies
    // use resampler_config; kld_config holds the suggested bins and bound.  `last_kld` keeps the whole record.
    b2_kld_config kld_config{0.5f, 0.0f, 0.17453292f, 100u, 0.01, 0.99};       // res_xy, res_z, res_yaw (10 deg), n_min, epsilon, z
    b2_kld_result last_kld{};
    ParticleUpdateDynamicResults resampleKLD(rm::MemoryView<rm::Transform, rm::VRAM_CUDA> poses, rm::MemoryView<ParticleAttributes, rm::VRAM_CUDA> attrs,
                                             rm::MemoryView<rm::Transform, rm::VRAM_CUDA> poses_new, rm::MemoryView<ParticleAttributes, rm::VRAM_CUDA> attrs_new,
                                             uint64_t seed = 1234, uint32_t step = 0, uint32_t first = 0, uint32_t n_max = 0)
    {
        const uint32_t n = particle_count("resampleKLD", poses, attrs), n_local = particle_count("resampleKLD", poses_new, attrs_new);
        if (n_max == 0) n_max = first + n_local;
        b2_check(b2_pf_resample_kld(h_, reinterpret_cast<const b2_transform*>(poses.raw()), reinterpret_cast<const b2_particle_attr*>(attrs.raw()), n,
                                    n_max, first, n_local, reinterpret_cast<b2_transform*>(poses_new.raw()),
                                    reinterpret_cast<b2_particle_attr*>(attrs_new.raw()), &resampler_config, &kld_config, seed, step, &last_kld), "resampleKLD");
        ParticleUpdateDynamicResults res;
        res.n_particles = (uint32_t)last_kld.n_particles;
        return res;
    }
    // RmclNode::initSamplesUniform (rmcl_localization.cpp:277-342) on the device: particles first .. first+poses.size()-1 of a set drawn
    // uniformly from [bb_min, bb_max] (x, y, z, roll, pitch, yaw).  Draws keyed by (seed, global index): shards concatenate to the whole set.
    void initSamplesUniform(rm::MemoryView<rm::Transform, rm::VRAM_CUDA> poses, rm::MemoryView<ParticleAttributes, rm::VRAM_CUDA> attrs,
                            const std::array<double, 6>& bb_min, const std::array<double, 6>& bb_max, uint64_t seed, uint32_t first = 0)
    {
        b2_check(b2_pf_init_uniform(h_, reinterpret_cast<b2_transform*>(poses.raw()), reinterpret_cast<b2_particle_attr*>(attrs.raw()), first,
                                    particle_count("initSamplesUniform", poses, attrs),
                                    bb_min.data(), bb_max.data(), seed), "initSamplesUniform");
    }
    // RmclNode::initSamples(PoseWithCovarianceStamped) (rmcl_localization.cpp:165-275) on the device: `pose` and the 36 row-major covariance
    // entries of the message; the noise acts in the pose frame.
    void initSamples(rm::MemoryView<rm::Transform, rm::VRAM_CUDA> poses, rm::MemoryView<ParticleAttributes, rm::VRAM_CUDA> attrs,
                     const rm::Transform& pose, const std::array<double, 36>& covariance, uint64_t seed, uint32_t first = 0)
    {
        b2_check(b2_pf_init_gaussian(h_, reinterpret_cast<b2_transform*>(poses.raw()), reinterpret_cast<b2_particle_attr*>(attrs.raw()), first,
                                     particle_count("initSamples", poses, attrs),
                                     reinterpret_cast<const b2_transform*>(&pose), covariance.data(), seed), "initSamples");
    }
    // RmclNode::estimateStats (rmcl_localization.cpp:642-731) on the device over the induction slice the caller passes, as the node passes
    // poses(0, k) with k = min(n_particles, max_induction_particles).  The record's fields are those of rmcl_msgs/ParticleStats
    // (rmcl::b200::fillParticleStats in rmcl_msgs_adapters.hpp copies them into the message).
    b2_particle_stats estimateStats(rm::MemoryView<rm::Transform, rm::VRAM_CUDA> poses, rm::MemoryView<ParticleAttributes, rm::VRAM_CUDA> attrs)
    {
        b2_particle_stats s;
        b2_check(b2_pf_estimate_stats(h_, reinterpret_cast<const b2_transform*>(poses.raw()), reinterpret_cast<const b2_particle_attr*>(attrs.raw()),
                                      particle_count("estimateStats", poses, attrs), &s), "estimateStats");
        return s;
    }
    // The filter's pose hypotheses (b2_pf_cluster_stats; AMCL's cluster statistics): the clusters of the set, heaviest first, at most
    // cluster_config.max_records of them, each with the estimateStats of its members alone in `stats` and its share of the set in `weight`.
    // `labels`, if given, receives every particle's rank (0xFFFFFFFF: in no cluster).  `last_clusters` keeps the counts of the whole set.
    b2_cluster_config cluster_config{0.5f, 0.0f, 0.17453292f, 8u};             // res_xy, res_z, res_yaw (10 deg), max_records
    b2_cluster_result last_clusters{};
    std::vector<b2_cluster_record> estimateClusters(rm::MemoryView<rm::Transform, rm::VRAM_CUDA> poses, rm::MemoryView<ParticleAttributes, rm::VRAM_CUDA> attrs,
                                                    uint32_t* labels = nullptr)
    {
        const uint32_t n = particle_count("estimateClusters", poses, attrs);
        std::vector<b2_cluster_record> recs(16);                                // max_records is at most 16
        b2_check(b2_pf_cluster_stats(h_, reinterpret_cast<const b2_transform*>(poses.raw()), reinterpret_cast<const b2_particle_attr*>(attrs.raw()), n,
                                     &cluster_config, recs.data(), labels, &last_clusters), "estimateClusters");
        recs.resize(last_clusters.n_records);
        return recs;
    }
private:
    // The C ABI takes one count for a call's poses and attributes: views that differ in size are refused before anything runs
    template <typename P, typename A> static uint32_t particle_count(const char* method, const P& poses, const A& attrs)
    {
        if (poses.size() != attrs.size()) throw std::invalid_argument(std::string(method) + ": poses and attrs differ in size");
        return (uint32_t)poses.size();
    }
    struct CloudInput { bool set = false; const void* data = nullptr; uint64_t bytes = 0; b2_cloud_layout layout{}; bool on_device = false; std::shared_ptr<const void> keep_alive; };
    // with an input cloud: this update's beams, `samples` drawn with (seed, step), then step advances
    void sample_input()
    {
        if (!input_.set) return;
        beams_.resize(samples);
        uint32_t n = 0;
        b2_check(b2_pf_sample_cloud(h_, input_.data, input_.bytes, &input_.layout, input_.on_device ? 1 : 0, samples, seed, step,
                                    reinterpret_cast<b2_range_meas*>(beams_.data()), &n), "update");
        beams_.resize(n);
        step++;
    }
    B200MapPtr map_;
    b2_pf* h_ = nullptr;
    std::shared_ptr<B200DistanceField> field_;
    rm::Transform Tsb_ = rm::Transform::Identity();
    std::vector<RangeMeasurement> beams_;
    CloudInput input_;
};

}  // namespace rmcl
