// rmcl_msgs_adapters.hpp -- the wire formats of the path (rmcl_msgs/msg/{ScanInfo,DepthInfo,O1DnInfo,OnDnInfo,RangeData,Scan,Depth,O1Dn,OnDn}.msg)
// fed straight into the B200 correspondence classes.  Duck-typed templates: they accept the rosidl-generated C++ structs (rmcl_msgs::msg::*)
// as well as any struct with the same field names (tests/test_cpp_boundary.py uses plain PODs), so this header does not depend on ROS 2.
//
// What each function replaces in the reference:
//   setModel(rcc, info)      rmcl::convert(info, sensor_model_) + setModel  (rmcl_ros/src/util/conversions.cpp:22-34, 48-60, 74-94, 96-120;
//                                                                          MICPSphericalSensorCPU.cpp:155-160)
//   setData(rcc, data)       the per-ray loop of MICP*Sensor*::unpackMessage (rmcl_ros/src/micpl/MICPSphericalSensorCPU.cpp:193-228): here one
//                            512 KiB upload + the unpack kernel on the device (dataset point = direction * range (+ origin), mask = range in [min, max];
//                            RangeData.mask is ignored exactly like the reference ignores it: "TODOs: use input mask values", :189-191)
//   unpackMessage(rcc, msg)  both, for a whole Scan / Depth / O1Dn / OnDn message (or its *Stamped payload)
//   unpackPointCloud(rcc, cloud, filter)  pc2_to_o1dn (Pc2ToO1DnNode::convert: conversions.cpp:869-1073 + scan_operations.cpp:41-143) and the
//                            O1Dn sensor's unpackMessage + setModel in one device call (RCCB200O1Dn::setPointCloud); fields x, y, z looked up by name
//   unpackPointCloud(rcc, cloud, T)  pc2_to_scan (Pc2ToScanNode::convert + fillEmpty: pc2_to_scan.cpp:105-213, scan_operations.cpp:25-39) and the
//                            spherical sensor's unpackMessage in one device call (RCCB200Spherical::setPointCloud), into the model of its setModel
//   setInput(updater, msg)   Input<PointCloud2::ConstSharedPtr>::setInput of the PF sensor updater (rmcl_localization.cpp:512-530): its
//                            updates sample their beams from the message (PCDSensorUpdaterB200::setInput), which it holds meanwhile
//   fillSensorStats(...)     rmcl_msgs/MICPSensorStats as published at rmcl_ros/src/nodes/micp_localization.cpp:1009-1015
//   fillParticleStats(...)   rmcl_msgs/ParticleStats as RmclNode::estimateStats returns it (rmcl_ros/src/nodes/rmcl_localization.cpp:642-731)
#pragma once
#include <vector>

#include "rcc_b200.hpp"

namespace rmcl {
namespace b200 {

template <typename ScanInfoT> inline void setModel(RCCB200Spherical& rcc, const ScanInfoT& info)
{
    rm::SphericalModel m;                                                   // conversions.cpp:22-34
    m.phi.min = info.phi_min; m.phi.inc = info.phi_inc; m.phi.size = info.phi_n;
    m.theta.min = info.theta_min; m.theta.inc = info.theta_inc; m.theta.size = info.theta_n;
    m.range.min = info.range_min; m.range.max = info.range_max;
    rcc.setModel(m);
}
template <typename DepthInfoT> inline void setModel(RCCB200Pinhole& rcc, const DepthInfoT& info)
{
    rm::PinholeModel m;                                                     // conversions.cpp:48-60
    m.width = info.width; m.height = info.height; m.f[0] = info.fx; m.f[1] = info.fy; m.c[0] = info.cx; m.c[1] = info.cy;
    m.range.min = info.range_min; m.range.max = info.range_max;
    rcc.setModel(m);
}
// O1Dn / OnDn: the Point32 arrays go to the C ABI as packed xyz floats (no intermediate rm::Memory)
template <typename O1DnInfoT> inline void setModel(RCCB200O1Dn& rcc, const O1DnInfoT& info)
{
    std::vector<float> dirs(3 * info.dirs.size());                          // conversions.cpp:74-94
    for (size_t i = 0; i < info.dirs.size(); i++) { dirs[3 * i] = info.dirs[i].x; dirs[3 * i + 1] = info.dirs[i].y; dirs[3 * i + 2] = info.dirs[i].z; }
    const float orig[3] = {info.orig.x, info.orig.y, info.orig.z};
    if (dirs.size() != 3 * size_t(info.width) * info.height) throw std::runtime_error("O1DnInfo: dirs.size() != width * height");
    b2_check(b2_rcc_set_model_o1dn(rcc.handle(), info.width, info.height, orig, dirs.data(), info.range_min, info.range_max), "setModel(O1DnInfo)");
    rcc.noteModelSize(info.width, info.height);
}
template <typename OnDnInfoT> inline void setModel(RCCB200OnDn& rcc, const OnDnInfoT& info)
{
    if (info.origs.size() != info.dirs.size() || info.dirs.size() != size_t(info.width) * info.height) throw std::runtime_error("OnDnInfo: origs / dirs size != width * height");
    std::vector<float> origs(3 * info.origs.size()), dirs(3 * info.dirs.size());                    // conversions.cpp:96-120
    for (size_t i = 0; i < info.dirs.size(); i++) {
        origs[3 * i] = info.origs[i].x; origs[3 * i + 1] = info.origs[i].y; origs[3 * i + 2] = info.origs[i].z;
        dirs[3 * i] = info.dirs[i].x; dirs[3 * i + 1] = info.dirs[i].y; dirs[3 * i + 2] = info.dirs[i].z;
    }
    b2_check(b2_rcc_set_model_ondn(rcc.handle(), info.width, info.height, origs.data(), dirs.data(), info.range_min, info.range_max), "setModel(OnDnInfo)");
    rcc.noteModelSize(info.width, info.height);
}

// RangeData -> dataset (device-side unpackMessage)
template <typename RangeDataT> inline void setData(CorrespondencesB200& rcc, const RangeDataT& data) { rcc.setRanges(data.ranges.data(), data.ranges.size()); }

// Scan / Depth / O1Dn / OnDn: { info, data }
template <typename RCC, typename MsgT> inline void unpackMessage(RCC& rcc, const MsgT& msg) { setModel(rcc, msg.info); setData(rcc, msg.data); }

// sensor_msgs/PointCloud2 -> b2_cloud_layout: fields x, y, z looked up by name (conversions.cpp:899-953, pc2_to_scan.cpp:141-155), a missing
// one marked B2_CLOUD_NO_FIELD (the device call refuses it)
template <typename PointCloud2T> inline b2_cloud_layout cloudLayout(const PointCloud2T& cloud)
{
    b2_cloud_layout L{};
    L.width = cloud.width; L.height = cloud.height; L.point_step = cloud.point_step; L.row_step = cloud.row_step;
    L.offset_x = L.offset_y = L.offset_z = B2_CLOUD_NO_FIELD;
    for (const auto& f : cloud.fields) {
        if (f.name == "x") { L.offset_x = f.offset; L.datatype = (uint8_t)f.datatype; }
        else if (f.name == "y") L.offset_y = f.offset;
        else if (f.name == "z") L.offset_z = f.offset;
    }
    L.is_bigendian = cloud.is_bigendian ? 1 : 0;
    return L;
}

// sensor_msgs/PointCloud2 (+ the node's FilterOptions2D-shaped parameters: range_min, range_max, width / height .skip_begin .skip_end .increment)
template <typename PointCloud2T, typename FilterOptionsT> inline void unpackPointCloud(RCCB200O1Dn& rcc, const PointCloud2T& cloud, const FilterOptionsT& opt)
{
    const b2_cloud_layout L = cloudLayout(cloud);
    auto u32 = [](uint64_t v) { if (v > 0xffffffffu) throw std::runtime_error("unpackPointCloud: filter option out of range"); return (uint32_t)v; };
    const b2_o1dn_cloud_filter F{u32(opt.height.skip_begin), u32(opt.height.skip_end), u32(opt.height.increment),
                                 u32(opt.width.skip_begin), u32(opt.width.skip_end), u32(opt.width.increment), (float)opt.range_min, (float)opt.range_max};
    rcc.setPointCloud(cloud.data.data(), cloud.data.size(), L, F);
}

// sensor_msgs/PointCloud2 into the spherical model the sensor holds (pc2_to_scan's convert + the spherical unpackMessage); T_sensor_cloud is
// the transform the node looks up from the cloud's frame to the sensor frame (pc2_to_scan.cpp:111-133), identity when they are the same
template <typename PointCloud2T> inline void unpackPointCloud(RCCB200Spherical& rcc, const PointCloud2T& cloud,
                                                              const rm::Transform& T_sensor_cloud = rm::Transform::Identity())
{
    rcc.setPointCloud(cloud.data.data(), cloud.data.size(), cloudLayout(cloud), T_sensor_cloud);
}

// RmclNode::sensorUpdate hands each cloud to the updater (rmcl_localization.cpp:512-530); the updater holds the message as Input<> holds
// input_, and its next update() samples the beams from it on the host
template <typename PointCloud2T> inline void setInput(PCDSensorUpdaterB200& updater, const std::shared_ptr<const PointCloud2T>& msg)
{
    if (!msg) throw std::invalid_argument("setInput: null message");
    updater.setInput(msg->data.data(), msg->data.size(), cloudLayout(*msg), false, msg);
}

// rmcl_msgs/MICPSensorStats (micp_localization.cpp:1009-1015): valid_matches = Cmerged_o.n_meas, cov_trace = trace(Cmerged_o.covariance)
template <typename StatsMsgT> inline void fillSensorStats(StatsMsgT& stats, const rm::CrossStatistics& Cmerged_o, uint32_t total_measurements, uint32_t valid_measurements)
{
    stats.total_measurements = total_measurements; stats.valid_measurements = valid_measurements;
    stats.valid_matches = Cmerged_o.n_meas; stats.cov_trace = Cmerged_o.covariance.trace();
}
// rmcl_msgs/ParticleStats as RmclNode::estimateStats fills it (rmcl_ros/src/nodes/rmcl_localization.cpp:677-726), from
// PCDSensorUpdaterB200::estimateStats; the message's pose goes to publishStats (:733-795) unchanged
template <typename StatsMsgT> inline void fillParticleStats(StatsMsgT& msg, const b2_particle_stats& s)
{
    msg.nparticles = s.nparticles;
    msg.pose.pose.position.x = s.position[0]; msg.pose.pose.position.y = s.position[1]; msg.pose.pose.position.z = s.position[2];
    msg.pose.pose.orientation.x = s.orientation[0]; msg.pose.pose.orientation.y = s.orientation[1];
    msg.pose.pose.orientation.z = s.orientation[2]; msg.pose.pose.orientation.w = s.orientation[3];
    for (int i = 0; i < 36; i++) msg.pose.covariance[i] = s.covariance[i];
    msg.shift = s.shift;
    msg.trans_bb_min.x = s.trans_bb_min[0]; msg.trans_bb_min.y = s.trans_bb_min[1]; msg.trans_bb_min.z = s.trans_bb_min[2];
    msg.trans_bb_max.x = s.trans_bb_max[0]; msg.trans_bb_max.y = s.trans_bb_max[1]; msg.trans_bb_max.z = s.trans_bb_max[2];
    msg.likelihood.min = s.likelihood.min; msg.likelihood.max = s.likelihood.max;
    msg.likelihood.mean = s.likelihood.mean; msg.likelihood.sigma = s.likelihood.sigma;
}

}  // namespace b200
}  // namespace rmcl
