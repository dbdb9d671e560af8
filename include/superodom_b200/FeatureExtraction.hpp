// =============================================================================
// superodom_b200/FeatureExtraction.hpp -- header-only shim for the two per-point
// loops of the reference's feature-extraction node that sit directly in front
// of the registration path (SURVEY.md section 8f row 2):
//
//   featureExtraction::removePointDistortion<BufferType>(lidar_start_time, lidar_end_time, buffer, lidar_msg)
//       super_odometry/src/FeatureExtraction/featureExtraction.cpp:222-314
//   featureExtraction::uniformFeatureExtraction(pc_in, pc_out_surf, skip_num, block_range)
//       super_odometry/src/FeatureExtraction/featureExtraction.cpp:504-525
// and the edge cloud featureExtraction::extractFeatures publishes empty (:429-436): extractEdgeFeatures.
//
// Same argument meaning as upstream; the node's members they read or write
// (T_i_l, q_w_original_l, t_w_original_l) are explicit arguments here.  The pose
// buffer is anything that iterates like MapRingBuffer::measMap_ (a
// std::map<double, Meas>) together with a functor that turns a measurement into
// a pose -- upstream's `extractPose` lambda (:230-253).  Forwards to
// so_scan_deskew / so_scan_extract_uniform (superodom_b200.h).
// =============================================================================
#pragma once
#include <type_traits>

#include "LidarSlam.hpp"

namespace super_odometry {
namespace b200 {

// Offsets of x (must be 0), time and the record stride of the caller's raw point type (point_os::PointcloudXYZITR upstream:
// stride 32, time at byte 20).
template <class PointT>
inline void raw_point_layout(size_t* stride, size_t* time_off) {
    PointT p{};
    *stride = sizeof(PointT);
    *time_off = size_t(reinterpret_cast<const char*>(&p.time) - reinterpret_cast<const char*>(&p));
}

// removePointDistortion.  `meas` : ordered container of (stamp, measurement) pairs (std::map<double, Meas>);
// `extract_pose(measurement)` -> something Transformd converts from (rot + pos); imu_only = the Imu::Ptr instantiation
// (rotation-only samples, motion conjugated by T_i_l).  Rewrites x, y, z of every finite point of *lidar_msg in place and
// returns T_w_original_sensor = {q_w_original_l, t_w_original_l} (:283-289).  lidar_end_time is unused, as upstream.
template <class MeasMap, class ExtractPose, class RawCloudPtr>
inline Transformd removePointDistortion(Context& ctx, double lidar_start_time, double /*lidar_end_time*/, const MeasMap& meas, ExtractPose extract_pose,
                                        bool imu_only, const Transformd& T_i_l, RawCloudPtr& lidar_msg) {
    using PointT = typename std::decay<decltype(lidar_msg->points[0])>::type;
    if (!ctx.h) throw Error("removePointDistortion: context not created (set the resolutions and call Context::ensure first)");
    std::vector<double> stamps, poses;
    stamps.reserve(meas.size());
    poses.reserve(meas.size() * 7);
    for (const auto& kv : meas) {
        const Transformd T(extract_pose(kv.second));
        double p[7];
        T.to_pose7(p);
        stamps.push_back(kv.first);
        poses.insert(poses.end(), p, p + 7);
    }
    size_t stride = 0, toff = 0;
    raw_point_layout<PointT>(&stride, &toff);
    double til[7], start[7];
    T_i_l.to_pose7(til);
    size_t past_end = 0;
    const int rc = so_scan_deskew(ctx.h, lidar_msg->points.data(), lidar_msg->size(), stride, toff, lidar_start_time, stamps.data(), poses.data(),
                                  stamps.size(), imu_only ? 1 : 0, til, start, &past_end);
    if (rc < 0) throw Error(std::string("so_scan_deskew: ") + so_last_error());
    return Transformd::from_pose7(start);
}

// uniformFeatureExtraction: appends to *pc_out_surf (a cloud of points with float x, y, z, intensity -- pcl::PointXYZI
// upstream) every skip_num-th point of *pc_in that passes the predecessor-difference test, intensity = the raw point's time.
template <class RawCloudPtr, class CloudPtr>
inline void uniformFeatureExtraction(Context& ctx, const RawCloudPtr& pc_in, CloudPtr& pc_out_surf, int skip_num, float block_range, bool int_abs = false) {
    using RawT = typename std::decay<decltype(pc_in->points[0])>::type;
    using OutT = typename std::decay<decltype(pc_out_surf->points[0])>::type;
    if (!ctx.h) throw Error("uniformFeatureExtraction: context not created");
    size_t stride = 0, toff = 0;
    raw_point_layout<RawT>(&stride, &toff);
    const size_t n = pc_in->size();
    std::vector<float> out(4 * (n ? n : 1));
    size_t m = 0;
    const int rc = so_scan_extract_uniform(ctx.h, pc_in->points.data(), n, stride, toff, skip_num, block_range, int_abs ? 1 : 0, out.data(), n ? n : 1, &m);
    if (rc < 0) throw Error(std::string("so_scan_extract_uniform: ") + so_last_error());
    const size_t base = pc_out_surf->points.size();
    pc_out_surf->points.resize(base + m);
    for (size_t i = 0; i < m; ++i) {
        OutT p{};
        p.x = out[4 * i]; p.y = out[4 * i + 1]; p.z = out[4 * i + 2]; p.intensity = out[4 * i + 3];
        pc_out_surf->points[base + i] = p;
    }
}

// ... and the offset of the uint16 `ring` field (byte 24 in point_os::PointcloudXYZITR)
template <class PointT>
inline void raw_point_layout(size_t* stride, size_t* time_off, size_t* ring_off) {
    raw_point_layout<PointT>(stride, time_off);
    PointT p{};
    *ring_off = size_t(reinterpret_cast<const char*>(&p.ring) - reinterpret_cast<const char*>(&p));
}

// The edgePoints cloud extractFeatures leaves empty (featureExtraction.cpp:429-436): LOAM edge selection over the rings of *pc_in
// (so_scan_extract_edges), appended to *pc_out_edge with intensity = the raw point's time.  opts.voxel_leaf = lineRes applies
// laserMapping's corner filter (downSizeFilterCorner, laserMapping.cpp:635-640) on the device.
template <class RawCloudPtr, class CloudPtr>
inline void extractEdgeFeatures(Context& ctx, const RawCloudPtr& pc_in, CloudPtr& pc_out_edge, const so_edge_opts& opts = so_edge_opts{}) {
    using RawT = typename std::decay<decltype(pc_in->points[0])>::type;
    using OutT = typename std::decay<decltype(pc_out_edge->points[0])>::type;
    if (!ctx.h) throw Error("extractEdgeFeatures: context not created");
    size_t stride = 0, toff = 0, roff = 0;
    raw_point_layout<RawT>(&stride, &toff, &roff);
    const size_t n = pc_in->size();
    std::vector<float> out(4 * (n ? n : 1));
    size_t m = 0;
    const int rc = so_scan_extract_edges(ctx.h, pc_in->points.data(), n, stride, toff, roff, &opts, out.data(), n ? n : 1, &m);
    if (rc < 0) throw Error(std::string("so_scan_extract_edges: ") + so_last_error());
    const size_t base = pc_out_edge->points.size();
    pc_out_edge->points.resize(base + m);
    for (size_t i = 0; i < m; ++i) {
        OutT p{};
        p.x = out[4 * i]; p.y = out[4 * i + 1]; p.z = out[4 * i + 2]; p.intensity = out[4 * i + 3];
        pc_out_edge->points[base + i] = p;
    }
}

}  // namespace b200
}  // namespace super_odometry
