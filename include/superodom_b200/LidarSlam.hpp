// =============================================================================
// superodom_b200/LidarSlam.hpp -- header-only C++ shim that keeps the reference's
// LidarSLAM / LocalMap call surface (super_odometry/include/super_odometry/
// LidarProcess/LidarSlam.h, LocalMap.h) and forwards to the C ABI
// (superodom_b200.h).  laserMapping.cpp uses exactly these members
// (SURVEY.md section 8b):
//   call   slam.Localization(bool, PredictionSource, Transformd, edge, planner, t)   laserMapping.cpp:713-714
//   write  slam.localMap.{lineRes_,planeRes_}, Visual_confidence_factor, Pos/Ori_degeneracy_threshold,
//          LocalizationICPMaxIter, OptSet.*, map_dir, localization_mode, init_*, last_T_w_lidar,
//          frame_count, laser_imu_sync                                               :102-120,312,648-649,703-711,740-741
//          slam.localMap.setOrigin(t), slam.localMap.addSurfPointCloud(cloud)        :161,166
//   read   slam.T_w_lidar, startupCount, isDegenerate, stats, pos_in_localmap,
//          localMap.get5x5LocalMap(pos), localMap.getAllLocalMap()                   :387,439,450,563,581-596,734-738
//
// The shim is dependency-free: it ships tiny Eigen-compatible value types
// (x()/y()/z()/w() accessors, converting constructors from anything with the same
// accessors, so Eigen::Quaterniond / Eigen::Vector3d / the reference's Transformd
// drop in) and is templated on the point-cloud pointer type (anything with
// ->points.data(), ->size() and a point struct holding float x,y,z,intensity --
// pcl::PointCloud<pcl::PointXYZI>::Ptr in the node).  See INTEGRATION.md.
// =============================================================================
#pragma once
#include <array>
#include <cmath>
#include <cstddef>
#include <cstdint>
#include <cstring>
#include <stdexcept>
#include <string>
#include <tuple>
#include <vector>

#include "../superodom_b200.h"
#include "KeyframeIO.hpp"

namespace super_odometry {
namespace b200 {

struct Vector3d {
    double v[3] = {0, 0, 0};
    Vector3d() = default;
    Vector3d(double x, double y, double z) : v{x, y, z} {}
    template <class E, class = decltype(std::declval<const E&>().x())>
    Vector3d(const E& e) : v{double(e.x()), double(e.y()), double(e.z())} {}
    double x() const { return v[0]; } double y() const { return v[1]; } double z() const { return v[2]; }
    double& x() { return v[0]; } double& y() { return v[1]; } double& z() { return v[2]; }
    double norm() const { return std::sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]); }
};
struct Vector3i {
    int v[3] = {0, 0, 0};
    int x() const { return v[0]; } int y() const { return v[1]; } int z() const { return v[2]; }
    int& x() { return v[0]; } int& y() { return v[1]; } int& z() { return v[2]; }
};
struct Quaterniond {
    double q[4] = {0, 0, 0, 1};   // x y z w (Eigen coefficient order)
    Quaterniond() = default;
    Quaterniond(double w, double x, double y, double z) : q{x, y, z, w} {}   // Eigen ctor order (w, x, y, z)
    template <class E, class = decltype(std::declval<const E&>().w())>
    Quaterniond(const E& e) : q{double(e.x()), double(e.y()), double(e.z()), double(e.w())} {}
    double x() const { return q[0]; } double y() const { return q[1]; } double z() const { return q[2]; } double w() const { return q[3]; }
    Quaterniond conjugate() const { return Quaterniond(q[3], -q[0], -q[1], -q[2]); }
    Quaterniond operator*(const Quaterniond& b) const {
        return Quaterniond(q[3] * b.q[3] - q[0] * b.q[0] - q[1] * b.q[1] - q[2] * b.q[2],
                           q[3] * b.q[0] + q[0] * b.q[3] + q[1] * b.q[2] - q[2] * b.q[1],
                           q[3] * b.q[1] + q[1] * b.q[3] + q[2] * b.q[0] - q[0] * b.q[2],
                           q[3] * b.q[2] + q[2] * b.q[3] + q[0] * b.q[1] - q[1] * b.q[0]);
    }
    Vector3d operator*(const Vector3d& p) const {
        double ux = q[1] * p.v[2] - q[2] * p.v[1], uy = q[2] * p.v[0] - q[0] * p.v[2], uz = q[0] * p.v[1] - q[1] * p.v[0];
        ux += ux; uy += uy; uz += uz;
        return Vector3d(p.v[0] + q[3] * ux + (q[1] * uz - q[2] * uy), p.v[1] + q[3] * uy + (q[2] * ux - q[0] * uz),
                        p.v[2] + q[3] * uz + (q[0] * uy - q[1] * ux));
    }
};
// utils/Twist.h `Transformd`: rot + pos, operator*, inverse()
struct Transformd {
    Quaterniond rot;
    Vector3d pos;
    Transformd() = default;
    Transformd(const Quaterniond& r, const Vector3d& p) : rot(r), pos(p) {}
    template <class T, class = decltype(std::declval<const T&>().rot.w())>
    Transformd(const T& t) : rot(t.rot), pos(t.pos) {}
    Transformd inverse() const {
        Transformd o; o.rot = rot.conjugate(); Vector3d t = o.rot * pos; o.pos = Vector3d(-t.x(), -t.y(), -t.z()); return o;
    }
    Transformd operator*(const Transformd& b) const {
        Transformd o; o.rot = rot * b.rot; Vector3d t = rot * b.pos; o.pos = Vector3d(t.x() + pos.x(), t.y() + pos.y(), t.z() + pos.z()); return o;
    }
    void to_pose7(double out[7]) const { out[0] = pos.x(); out[1] = pos.y(); out[2] = pos.z(); out[3] = rot.x(); out[4] = rot.y(); out[5] = rot.z(); out[6] = rot.w(); }
    static Transformd from_pose7(const double p[7]) { return Transformd(Quaterniond(p[6], p[3], p[4], p[5]), Vector3d(p[0], p[1], p[2])); }
};

// super_odometry_msgs/msg/{IterationStats,OptimizationStats}.msg as plain structs (same field names)
struct IterationStats { double translation_norm = 0, rotation_norm = 0, num_surf_from_scan = 0, num_corner_from_scan = 0; };
struct OptimizationStats {
    int32_t laser_cloud_surf_from_map_num = 0, laser_cloud_corner_from_map_num = 0, laser_cloud_surf_stack_num = 0, laser_cloud_corner_stack_num = 0;
    double total_translation = 0, total_rotation = 0, translation_from_last = 0, rotation_from_last = 0, time_elapsed = 0, latency = 0;
    int32_t n_iterations = 0;
    double average_distance = 0, uncertainty_x = 0, uncertainty_y = 0, uncertainty_z = 0, uncertainty_roll = 0, uncertainty_pitch = 0, uncertainty_yaw = 0;
    int32_t plane_match_success = 0, plane_no_enough_neighbor = 0, plane_neighbor_too_far = 0, plane_badpca_structure = 0,
            plane_invalid_numerical = 0, plane_mse_too_large = 0, plane_unknown = 0, prediction_source = 0;
    std::vector<IterationStats> iterations;
};

class Error : public std::runtime_error { public: using std::runtime_error::runtime_error; };

// Shared handle to the device context; LocalMap and LidarSLAM both forward through it.
struct Context {
    so_ctx* h = nullptr;
    so_config cfg{};
    void ensure(float line_res, float plane_res) {
        if (!h) {
            cfg.line_res = line_res; cfg.plane_res = plane_res;
            h = so_create(&cfg);
            if (!h) throw Error(std::string("so_create: ") + so_last_error());
        }
    }
    ~Context() { if (h) so_destroy(h); }
};

// point layout of the caller's cloud type
template <class PointT>
inline void point_layout(size_t* stride, size_t* ioff) {
    PointT p{};
    *stride = sizeof(PointT);
    *ioff = size_t(reinterpret_cast<const char*>(&p.intensity) - reinterpret_cast<const char*>(&p));
}

class LidarSLAM;

// ------------------------------------------------------------------------------------------------ LocalMap (LocalMap.h:123-766)
class LocalMap {
    friend class LidarSLAM;                    // alignKeyframes registers against another LocalMap's context
public:
    static constexpr int laserCloudWidth = 21, laserCloudHeight = 21, laserCloudDepth = 11;
    static constexpr int laserCloudNum = laserCloudWidth * laserCloudHeight * laserCloudDepth;
    float lineRes_ = 0.2f;     // LocalMap.h:761
    float planeRes_ = 0.4f;    // LocalMap.h:762
    Vector3i origin_;

    explicit LocalMap(Context* c) : ctx_(c) { origin_.v[0] = 10; origin_.v[1] = 10; origin_.v[2] = 5; }

    template <class V> Vector3i setOrigin(const V& t_w_cur) {                       // LocalMap.h:146-164
        sync_resolution();
        const double t[3] = {double(t_w_cur.x()), double(t_w_cur.y()), double(t_w_cur.z())};
        check(so_map_set_origin(ctx_->h, t, origin_.v), "so_map_set_origin");
        return origin_;
    }
    template <class V> Vector3i shiftMap(const V& t_w_cur) {                        // LocalMap.h:169-287
        sync_resolution();
        const double t[3] = {double(t_w_cur.x()), double(t_w_cur.y()), double(t_w_cur.z())};
        Vector3i ijk;
        check(so_map_shift(ctx_->h, t, ijk.v), "so_map_shift");
        check(so_map_get_origin(ctx_->h, origin_.v), "so_map_get_origin");
        return ijk;
    }
    std::tuple<int, int> get5x5LocalMapFeatureSize(const Vector3i& position) {      // LocalMap.h:291-318
        sync_resolution();
        int32_t ne = 0, ns = 0;
        check(so_map_counts_5x5(ctx_->h, position.v, &ne, &ns), "so_map_counts_5x5");
        return std::make_tuple(int(ne), int(ns));
    }
    template <class Cloud> void addSurfPointCloud(Cloud& laserCloudSurfStack) {     // LocalMap.h:591-645 (world-frame points)
        sync_resolution();
        if (laserCloudSurfStack.size() == 0) return;
        size_t stride, ioff;
        point_layout<typename std::decay<decltype(laserCloudSurfStack.points[0])>::type>(&stride, &ioff);
        check(so_map_add_surf(ctx_->h, laserCloudSurfStack.points.data(), laserCloudSurfStack.size(), stride, ioff), "so_map_add_surf");
    }
    template <class Cloud> void addEdgePointCloud(Cloud& laserCloudEdgeStack) {     // LocalMap.h:529-589 (world-frame points)
        sync_resolution();
        if (laserCloudEdgeStack.size() == 0) return;
        size_t stride, ioff;
        point_layout<typename std::decay<decltype(laserCloudEdgeStack.points[0])>::type>(&stride, &ioff);
        check(so_map_add_edge(ctx_->h, laserCloudEdgeStack.points.data(), laserCloudEdgeStack.size(), stride, ioff), "so_map_add_edge");
    }
    // getAllLocalMap / get5x5LocalMap (LocalMap.h:647-687) fill a caller cloud type (resize + x,y,z,intensity)
    template <class Cloud> Cloud getAllLocalMap() { return download<Cloud>(0, nullptr); }
    template <class Cloud> Cloud get5x5LocalMap(const Vector3i& position) { return download<Cloud>(1, position.v); }
    size_t size() const { return ctx_->h ? so_map_size(ctx_->h) : 0; }
    // Shim only: the block archive (so_map_archive).  Keeps the blocks the window drops, with room for cap points per store; 0 turns
    // it off.  In localization mode, call it before setOrigin and the prior-map load so that the whole prior map is kept.
    void setArchive(size_t cap) {
        sync_resolution();
        check(so_map_archive(ctx_->h, cap), "so_map_archive");
    }
    // Shim only: load an already voxel-filtered world-frame surf map as the whole map (so_map_set_points), e.g. a map saved with
    // getWholeMap + writePointCloud.  With the archive on, the blocks outside the window go to the archive instead of being dropped
    // (addSurfPointCloud, the reference's load, filters the cloud and keeps only the window).
    template <class Cloud> void loadPriorMap(const Cloud& cloud) {
        sync_resolution();
        size_t stride, ioff;
        point_layout<typename std::decay<decltype(cloud.points[0])>::type>(&stride, &ioff);
        check(so_map_set_points(ctx_->h, cloud.points.data(), cloud.points.size(), stride, ioff), "so_map_set_points");
    }
    // Points held in the archive (surf and edge stores together)
    size_t archiveSize() const {
        size_t s = 0, e = 0;
        if (ctx_->h) { so_map_archive_info(ctx_->h, 0, &s, nullptr, nullptr); so_map_archive_info(ctx_->h, 1, &e, nullptr, nullptr); }
        return s + e;
    }
    // Shim only, no reference counterpart: remove the map points the sensor-frame cloud (at pose) saw clearly past, e.g. what a moving
    // object left (so_map_clear_free_space; stores: 1 surf, 2 edge, 3 both).  Give it the full-resolution cloud: it leaves fewer
    // pixels without a return near the sensor than the voxel-filtered surf stack.
    template <class Cloud> so_free_space_result clearFreeSpace(const Cloud& cloud, const Transformd& pose, const so_free_space& opts, int stores = 3) {
        sync_resolution();
        size_t stride, ioff;
        point_layout<typename std::decay<decltype(cloud.points[0])>::type>(&stride, &ioff);
        double p[7];
        pose.to_pose7(p);
        so_free_space_result r{};
        check(so_map_clear_free_space(ctx_->h, stores, cloud.size() ? cloud.points.data() : nullptr, cloud.size(), stride, ioff, p, &opts, &r),
              "so_map_clear_free_space");
        return r;
    }
    static so_free_space defaultFreeSpace() { so_free_space o{}; so_free_space_defaults(&o); return o; }
    // The whole surf map, window plus archive, ordered by world block (so_map_download_all): a session's map as the next one's prior map
    template <class Cloud> Cloud getWholeMap() {
        sync_resolution();
        size_t n = 0;
        check(so_map_download_all(ctx_->h, 0, nullptr, 0, &n), "so_map_download_all");
        std::vector<float> buf(4 * (n ? n : 1));
        check(so_map_download_all(ctx_->h, 0, buf.data(), n, &n), "so_map_download_all");
        return to_cloud<Cloud>(buf, n);
    }

    // Shim only: keyframes (so_keyframe_*) for a loop-closing back end.  Room for `points` points in each of the surf and edge pools
    // and for `frames` keyframes (0, 0 frees them); LidarSLAM::addKeyframe fills them.
    void reserveKeyframes(size_t points, size_t frames) {
        sync_resolution();
        check(so_keyframe_reserve(ctx_->h, points, frames), "so_keyframe_reserve");
    }
    // The keyframes' poses: as added, or as the last rebuild (LidarSLAM::rebuildFromKeyframes) placed them
    std::vector<Transformd> keyframePoses() const {
        std::vector<Transformd> out;
        if (!ctx_->h) return out;
        size_t n = 0;
        check(so_keyframe_poses(ctx_->h, nullptr, 0, &n), "so_keyframe_poses");
        std::vector<double> p(7 * n);
        check(so_keyframe_poses(ctx_->h, p.data(), n, &n), "so_keyframe_poses");
        for (size_t i = 0; i < n; ++i) out.push_back(Transformd::from_pose7(p.data() + 7 * i));
        return out;
    }
    // This map's stores (surf and edge) replaced by the map of src's keyframes ids, keyframe ids[i] at poses[i]
    // (so_map_from_keyframes): a loop-verification submap, or with src == *this the rebuild after a pose-graph correction.  The map is
    // then exactly its keyframes: a prior map loaded with loadPriorMap and free-space removals are not kept.
    void buildFromKeyframes(const LocalMap& src, const std::vector<int32_t>& ids, const std::vector<Transformd>& poses) {
        if (ids.size() != poses.size()) throw Error("buildFromKeyframes: one pose per keyframe id");
        sync_resolution();
        std::vector<double> p(7 * poses.size());
        for (size_t i = 0; i < poses.size(); ++i) poses[i].to_pose7(p.data() + 7 * i);
        check(so_map_from_keyframes(ctx_->h, src.ctx_->h, ids.data(), ids.size(), p.data(), 3), "so_map_from_keyframes");
    }
    // Shim only: this map cleared against the surf clouds of src's keyframes ids, keyframe ids[i] at poses[i]
    // (so_map_clear_free_space_keyframes; stores: 1 surf, 2 edge, 3 both): the map clearFreeSpace of each keyframe in turn would leave,
    // in one device call.  After buildFromKeyframes(*this, ...) it takes out again what the live clearing had removed; with another
    // src it clears a prior map with a session's keyframes.
    so_free_space_keyframes_result clearFreeSpaceFromKeyframes(const LocalMap& src, const std::vector<int32_t>& ids,
                                                               const std::vector<Transformd>& poses, const so_free_space& opts, int stores = 3) {
        if (ids.size() != poses.size()) throw Error("clearFreeSpaceFromKeyframes: one pose per keyframe id");
        sync_resolution();
        std::vector<double> p(7 * poses.size());
        for (size_t i = 0; i < poses.size(); ++i) poses[i].to_pose7(p.data() + 7 * i);
        so_free_space_keyframes_result r{};
        check(so_map_clear_free_space_keyframes(ctx_->h, src.ctx_->h, ids.data(), ids.size(), p.data(), stores, &opts, &r),
              "so_map_clear_free_space_keyframes");
        return r;
    }
    // Shim only: sessions (KeyframeIO.hpp; INTEGRATION.md "Sessions").  saveKeyframes writes every keyframe (pose, surf and edge
    // clouds in the sensor frame) and the caller's graph edges to one file; loadKeyframes appends a saved session's keyframes to this
    // map's store (so_keyframe_import) and returns the first new id, their count and the saved edges (node ids as saved: add `first`
    // to place them in this store).  Neither call touches the map; the store must have room (reserveKeyframes).
    struct LoadedKeyframes { int32_t first = 0; int32_t count = 0; std::vector<so_pose_edge> edges; };
    void saveKeyframes(const std::string& path, const std::vector<so_pose_edge>& edges) {
        sync_resolution();
        KeyframeSession s;
        size_t n = 0;
        check(so_keyframe_poses(ctx_->h, nullptr, 0, &n), "so_keyframe_poses");
        std::vector<double> p(7 * n);
        check(so_keyframe_poses(ctx_->h, p.data(), n, &n), "so_keyframe_poses");
        s.poses.resize(n); s.surf.resize(n); s.edge.resize(n);
        for (size_t i = 0; i < n; ++i) {
            std::memcpy(s.poses[i].data(), p.data() + 7 * i, 7 * sizeof(double));
            for (int store = 0; store < 2; ++store) {
                std::vector<float>& dst = store ? s.edge[i] : s.surf[i];
                size_t m = 0;
                check(so_keyframe_download(ctx_->h, int32_t(i), store, nullptr, nullptr, 0, &m), "so_keyframe_download");
                dst.resize(4 * m);
                if (m) check(so_keyframe_download(ctx_->h, int32_t(i), store, nullptr, dst.data(), m, &m), "so_keyframe_download");
            }
        }
        s.edges = edges;
        std::string err;
        if (!writeKeyframeSession(path, s, &err)) throw Error(err);
    }
    LoadedKeyframes loadKeyframes(const std::string& path) {
        sync_resolution();
        KeyframeSession s;
        std::string err;
        if (!readKeyframeSession(path, &s, &err)) throw Error(err);
        LoadedKeyframes out;
        size_t have = 0;
        check(so_keyframe_info(ctx_->h, &have, nullptr, nullptr), "so_keyframe_info");
        out.first = int32_t(have);
        for (size_t i = 0; i < s.poses.size(); ++i) {
            int32_t id = -1;
            check(so_keyframe_import(ctx_->h, s.surf[i].data(), s.surf[i].size() / 4, s.edge[i].data(), s.edge[i].size() / 4, 16, 12,
                                     s.poses[i].data(), &id), "so_keyframe_import");
            ++out.count;
        }
        out.edges = std::move(s.edges);
        return out;
    }
    void sync_resolution() {
        ctx_->ensure(lineRes_, planeRes_);
        if (lineRes_ != pushed_line_ || planeRes_ != pushed_plane_) {
            check(so_map_set_resolution(ctx_->h, lineRes_, planeRes_), "so_map_set_resolution");
            pushed_line_ = lineRes_; pushed_plane_ = planeRes_;
        }
    }

private:
    template <class Cloud> Cloud download(int mode, const int32_t* ijk) {
        sync_resolution();
        size_t n = 0;
        const size_t cap = so_map_size(ctx_->h);
        std::vector<float> buf(4 * (cap ? cap : 1));
        check(so_map_download(ctx_->h, mode, ijk, buf.data(), cap, &n), "so_map_download");
        if (n > cap) {                     // a pending origin change restored archived blocks: the window grew in this call
            buf.assign(4 * n, 0.f);
            check(so_map_download(ctx_->h, mode, ijk, buf.data(), n, &n), "so_map_download");
        }
        return to_cloud<Cloud>(buf, n);
    }
    template <class Cloud> static Cloud to_cloud(const std::vector<float>& buf, size_t n) {
        Cloud out;
        out.points.resize(n);
        for (size_t i = 0; i < n; ++i) { auto& p = out.points[i]; p.x = buf[4 * i]; p.y = buf[4 * i + 1]; p.z = buf[4 * i + 2]; p.intensity = buf[4 * i + 3]; }
        return out;
    }
    static void check(int rc, const char* what) { if (rc < 0) throw Error(std::string(what) + ": " + so_last_error()); }
    Context* ctx_;
    float pushed_line_ = -1.f, pushed_plane_ = -1.f;
};

// ------------------------------------------------------------------------------------------------ LidarSLAM (LidarSlam.h:40-423)
class LidarSLAM {
public:
    enum class PredictionSource { IMU_ORIENTATION, LIO_ODOM, VIO_ODOM, NEURAL_IMU_ODOM, CONSTANT_VELOCITY };
    enum UndistortionMode { NONE = 0, APPROXIMATED = 1, OPTIMIZED = 2 };                         // LidarSlam.h:65-82
    enum MatchingResult : uint8_t { SUCCESS = 0, NOT_ENOUGH_NEIGHBORS = 1, NEIGHBORS_TOO_FAR = 2, BAD_PCA_STRUCTURE = 3,
                                    INVAVLID_NUMERICAL = 4, MSE_TOO_LARGE = 5, UNKNON = 6, nRejectionCauses = 7 };
    enum Feature_observability : uint8_t { rx_cross = 0, neg_rx_cross = 1, ry_cross = 2, neg_ry_cross = 3, rz_cross = 4, neg_rz_cross = 5,
                                           tx_dot = 6, ty_dot = 7, tz_dot = 8, nFeatureObs = 9 };
    struct LaserOptSet {
        double imu_roll_pitch[4] = {0, 0, 0, 1};
        bool debug_view_enabled = false, use_imu_roll_pitch = false;
        float velocity_failure_threshold = 30.f, yaw_ratio = 0.f;
        int max_surface_features = 2000;
    };
    struct RegistrationError {                                   // LidarSlam.h:122-148
        double PositionError = 0., PositionUncertainty = 0., MaxPositionError = 0.1, PosInverseConditionNum = 1.0;
        Vector3d PositionErrorDirection;
        double OrientationError = 0., OrientationUncertainty = 0., MaxOrientationError = 10, OriInverseConditionNum = 1.0;
        Vector3d OrientationErrorDirection;
        std::array<double, 36> Covariance{};                     // row-major, DoF order X,Y,Z,rX,rY,rZ
    };
    struct LidarOdomUncertainty { double uncertainty_x = 0, uncertainty_y = 0, uncertainty_z = 0, uncertainty_roll = 0, uncertainty_pitch = 0, uncertainty_yaw = 0; };

    Context context;                 // owns the device context (declared first: localMap points into it)
    LocalMap localMap;
    OptimizationStats stats;
    RegistrationError LocalizationUncertainty;
    LidarOdomUncertainty lidarOdomUncer;
    LaserOptSet OptSet;
    Transformd T_w_lidar, last_T_w_lidar, T_w_initial_guess;
    Vector3i pos_in_localmap;
    int frame_count = 0, laser_imu_sync = 0, startupCount = 0;
    float Pos_degeneracy_threshold = 0, Ori_degeneracy_threshold = 0, Visual_confidence_factor = 0;
    std::string map_dir;
    float init_x = 0, init_y = 0, init_z = 0, init_roll = 0, init_pitch = 0, init_yaw = 0, localization_mode = 0, update_map = 0;
    double lasttimeLaserOdometry = 0;
    // isDegenerate: set after every registration by the reference's commented-out rule (LidarSlam.cpp:976-985) on the final covariance,
    // pos_inv_cond < Pos_degeneracy_threshold || ori_inv_cond < Ori_degeneracy_threshold (never with the default thresholds of 0)
    bool bInitialization = false, isDegenerate = false;
    // shim only: with Undistortion == NONE, register through so_register_degeneracy (constrain = 1, the degeneracy thresholds above):
    // each ICP iteration's solve leaves the directions the scan does not constrain alone
    bool DegeneracyAware = false;
    so_degeneracy_result last_degeneracy{};                      // DegeneracyAware: what the analysis reported for the last scan
    std::array<int, nFeatureObs> PlaneFeatureHistogramObs{};
    std::array<int, nRejectionCauses> MatchRejectionHistogramLine{}, MatchRejectionHistogramPlane{};
    size_t LocalizationICPMaxIter = 4;                           // LidarSlam.h:273
    UndistortionMode Undistortion = NONE;                        // LidarSlam.h:266; APPROXIMATED: so_register_undistort, OPTIMIZED:
                                                                 // so_register_optimized; time in intensity
    // OPTIMIZED: information per accepted correspondence of the motion prior D0 = undistort_prev_pose^-1 * position (translation
    // xyz, rotation xyz).  0, a free motion, has the smallest worst-case pose error of the accuracy sweep in DESIGN.md §4; a larger
    // value helps only while the velocity stays what the previous registration saw
    double OptimizedMotionInformation[6] = {0, 0, 0, 0, 0, 0};
    Transformd LastMotion;                                       // OPTIMIZED: the motion D the last registration estimated (identity otherwise)
    bool UndistortRotation = true;                               // shim only: false when the cloud's rotation was already removed
                                                                 // (featureExtraction's IMU branch, so_scan_deskew imu_only)
    Transformd undistort_prev_pose;                              // pose of the previous scan (last_T_w_lidar is the prior by then)
    bool undistort_has_prev = false;
    so_icp_result last_result{};                                 // everything the device reported for the last scan
    // shim only: before its inserts, Localization removes from both stores the map points the registered scan saw clearly past
    // (so_map_clear_free_space_registered with FreeSpaceOpts; set its image geometry for the sensor).  Off by default.
    bool ClearFreeSpace = false;
    so_free_space FreeSpaceOpts = LocalMap::defaultFreeSpace();
    so_free_space_result last_free_space{};                      // ClearFreeSpace: what the last clearing removed

    explicit LidarSLAM(int device = 0, uint32_t max_map_points = 0, uint32_t max_scan_points = 0) : localMap(&context) {
        context.cfg.device = device; context.cfg.max_map_points = max_map_points; context.cfg.max_scan_points = max_scan_points;
    }
    template <class NodePtr> void initROSInterface(NodePtr) {}   // the six Float32 uncertainty publishers stay in the node (LidarSlam.cpp:20-28)

    // LidarSLAM::Localization (LidarSlam.cpp:30-51)
    template <class CloudPtr>
    void Localization(bool initialization, PredictionSource predictodom, const Transformd& position, const CloudPtr& edge_point,
                      const CloudPtr& planner_point, double timeLaserOdometry) {
        T_w_lidar = position; T_w_initial_guess = position; last_T_w_lidar = position;          // initializeState (:53-57)
        localMap.sync_resolution();
        size_t stride, ioff;
        using PointT = typename std::decay<decltype(planner_point->points[0])>::type;
        point_layout<PointT>(&stride, &ioff);
        const void* surf = planner_point->size() ? planner_point->points.data() : nullptr;
        double pose[7];
        if (!initialization) {                                                                   // initializeMapping (:83-94)
            localMap.setOrigin(T_w_lidar.pos);
            T_w_lidar.to_pose7(pose);
            if (edge_point && edge_point->size()) check(so_map_add_scan_edge(context.h, edge_point->points.data(), edge_point->size(), stride, ioff, pose), "so_map_add_scan_edge");
            if (planner_point->size()) check(so_map_add_scan(context.h, surf, planner_point->size(), stride, ioff, pose), "so_map_add_scan");
            lasttimeLaserOdometry = timeLaserOdometry;
            undistort_prev_pose = T_w_lidar; undistort_has_prev = true;
            return;
        }
        EstimateLidarUncertainty();                                                              // (:915-986), from the PREVIOUS scan's histogram
        so_icp_opts o{};
        o.max_icp_iters = int32_t(LocalizationICPMaxIter);
        o.max_surface_features = OptSet.max_surface_features;
        o.lm_max_iterations = 4;
        o.yaw_ratio = OptSet.yaw_ratio;
        // shouldAddAbsolutePoseConstraints (LidarSlam.cpp:281-283)
        if (predictodom == PredictionSource::VIO_ODOM && isDegenerate && Visual_confidence_factor != 0) {
            o.use_pose_prior = 1;
            o.visual_confidence_factor = Visual_confidence_factor;
            o.prior_uncertainty[0] = float(lidarOdomUncer.uncertainty_x);
            o.prior_uncertainty[1] = float(lidarOdomUncer.uncertainty_y);
            o.prior_uncertainty[2] = float(lidarOdomUncer.uncertainty_z);
        }
        position.to_pose7(pose);
        const double dt = timeLaserOdometry - lasttimeLaserOdometry;
        int rc;
        LastMotion = Transformd();
        const bool has_edges = edge_point && edge_point->size();
        bool edges_registered = false;                             // the edge cloud is still on the device (so_map_add_registered_edges)
        if (Undistortion == OPTIMIZED && dt > 0 && !o.use_pose_prior) {
            so_motion m{};                                         // so_register_optimized* refuses the pose prior
            m.dt = dt;
            const Transformd D0 = undistort_has_prev ? undistort_prev_pose.inverse() * position : Transformd();
            D0.to_pose7(m.motion_prior);
            for (int k = 0; k < 6; ++k) m.motion_info[k] = OptimizedMotionInformation[k];
            so_motion_result mr{};
            if (has_edges) {
                rc = so_register_optimized_edges(context.h, surf, planner_point->size(), edge_point->points.data(), edge_point->size(), stride,
                                                 ioff, ioff, pose, &m, &o, &mr);
                check(rc, "so_register_optimized_edges");
                edges_registered = true;
            } else {
                rc = so_register_optimized(context.h, surf, planner_point->size(), stride, ioff, ioff, pose, &m, &o, &mr);
                check(rc, "so_register_optimized");
            }
            last_result = mr.icp;
            LastMotion = Transformd::from_pose7(mr.motion);
        } else if (Undistortion == APPROXIMATED && undistort_has_prev && dt > 0) {
            so_undistort u{};                                      // both clouds carry their time in intensity
            u.mode = 1; u.rotation = UndistortRotation ? 1 : 0; u.dt = dt;
            undistort_prev_pose.to_pose7(u.prev_pose);
            if (has_edges) {
                rc = so_register_undistort_edges(context.h, surf, planner_point->size(), edge_point->points.data(), edge_point->size(), stride,
                                                 ioff, ioff, pose, &u, &o, &last_result);
                check(rc, "so_register_undistort_edges");
                edges_registered = true;
            } else {
                rc = so_register_undistort(context.h, surf, planner_point->size(), stride, ioff, ioff, pose, &u, &o, &last_result);
                check(rc, "so_register_undistort");
            }
        } else if (DegeneracyAware && Undistortion == NONE) {
            so_degeneracy d{};
            d.pos_threshold = Pos_degeneracy_threshold; d.ori_threshold = Ori_degeneracy_threshold; d.constrain = 1;
            rc = so_register_degeneracy(context.h, surf, planner_point->size(), edge_point ? (const void*)edge_point->points.data() : nullptr,
                                        edge_point ? edge_point->size() : 0, stride, ioff, pose, &d, &o, &last_degeneracy);
            check(rc, "so_register_degeneracy");
            last_result = last_degeneracy.icp;
        } else {
            rc = so_register(context.h, surf, planner_point->size(), edge_point ? (const void*)edge_point->points.data() : nullptr,
                             edge_point ? edge_point->size() : 0, stride, ioff, pose, &o, &last_result);
            check(rc, "so_register");
        }
        const so_icp_result& r = last_result;
        pos_in_localmap.v[0] = r.pos_in_localmap[0]; pos_in_localmap.v[1] = r.pos_in_localmap[1]; pos_in_localmap.v[2] = r.pos_in_localmap[2];
        check(so_map_get_origin(context.h, localMap.origin_.v), "so_map_get_origin");
        stats.laser_cloud_corner_from_map_num = r.map_edge_5x5; stats.laser_cloud_surf_from_map_num = r.map_surf_5x5;   // updateFeatureStats (:371-377)
        stats.laser_cloud_corner_stack_num = int32_t(edge_point ? edge_point->size() : 0); stats.laser_cloud_surf_stack_num = int32_t(planner_point->size());
        stats.iterations.clear();
        if (rc == SO_STATUS_NOT_ENOUGH_FEATURES) return;                                         // (:113-116) WARN + return, pose = prior
        for (int i = 0; i < r.n_iterations; ++i) {                                               // recordIterationStats (:242-251)
            IterationStats it; it.num_surf_from_scan = r.iter_n_surf[i]; it.num_corner_from_scan = r.iter_n_edge[i];
            it.translation_norm = r.iter_dtrans[i]; it.rotation_norm = r.iter_drot[i];
            stats.iterations.push_back(it);
        }
        stats.prediction_source = r.prediction_source;                                            // (:278,297)
        for (int i = 0; i < 9; ++i) PlaneFeatureHistogramObs[i] = r.hist_obs[i];
        for (int i = 0; i < 7; ++i) { MatchRejectionHistogramPlane[i] = r.hist_reject_plane[i]; MatchRejectionHistogramLine[i] = r.hist_reject_line[i]; }
        LocalizationUncertainty.PositionError = r.pos_err; LocalizationUncertainty.PosInverseConditionNum = r.pos_inv_cond;
        LocalizationUncertainty.OrientationError = r.ori_err_deg; LocalizationUncertainty.OriInverseConditionNum = r.ori_inv_cond;
        LocalizationUncertainty.PositionErrorDirection = Vector3d(r.pos_dir[0], r.pos_dir[1], r.pos_dir[2]);
        LocalizationUncertainty.OrientationErrorDirection = Vector3d(r.ori_dir[0], r.ori_dir[1], r.ori_dir[2]);
        std::memcpy(LocalizationUncertainty.Covariance.data(), r.cov, sizeof(r.cov));
        isDegenerate = r.pos_inv_cond < Pos_degeneracy_threshold || r.ori_inv_cond < Ori_degeneracy_threshold;
        T_w_lidar = Transformd::from_pose7(r.pose);                                              // after MannualYawCorrection (:891-913)
        stats.time_elapsed = r.time_ms;                                                          // updateOptimizationStats (:198-210)
        stats.total_translation = r.total_translation; stats.total_rotation = r.total_rotation;
        stats.translation_from_last = r.translation_from_last; stats.rotation_from_last = r.rotation_from_last;
        stats.n_iterations = r.n_iterations;
        last_T_w_lidar = T_w_lidar;
        // checkMotionThresholds always accepts (:193) -> transformAndAddToMap (:163-167)
        if (ClearFreeSpace && planner_point->size())
            check(so_map_clear_free_space_registered(context.h, 3, r.pose, &FreeSpaceOpts, &last_free_space), "so_map_clear_free_space_registered");
        if (edges_registered) check(so_map_add_registered_edges(context.h, r.pose), "so_map_add_registered_edges");    // compensated, at r.pose
        else if (has_edges) check(so_map_add_scan_edge(context.h, edge_point->points.data(), edge_point->size(), stride, ioff, r.pose), "so_map_add_scan_edge");
        if (planner_point->size()) check(so_map_add_registered_scan(context.h, r.pose), "so_map_add_registered_scan");   // the scan is still on the device
        lasttimeLaserOdometry = timeLaserOdometry;
        undistort_prev_pose = T_w_lidar; undistort_has_prev = true;
    }

    // Global localization against the prior map (so_localize_global; extends localization mode, laserMapping.cpp:163-173,306-313):
    // call once after the prior map is loaded and before the first Localization(), with a rough start pose whose roll and pitch are
    // trusted (IMU gravity).  Sets T_w_lidar and last_T_w_lidar as initializeFirstFrame does in localization mode -- to the refined
    // pose, or to the centre when nothing was found.  Returns the status; last_global holds the whole result.
    so_global_result last_global{};
    template <class CloudPtr>
    int globalLocalize(const CloudPtr& planner_point, const Transformd& centre, const so_global_opts& opts) {
        localMap.sync_resolution();
        size_t stride, ioff;
        using PointT = typename std::decay<decltype(planner_point->points[0])>::type;
        point_layout<PointT>(&stride, &ioff);
        so_icp_opts o{};
        o.max_icp_iters = int32_t(LocalizationICPMaxIter);
        o.max_surface_features = OptSet.max_surface_features;
        o.lm_max_iterations = 4;
        o.yaw_ratio = OptSet.yaw_ratio;
        double c[7];
        centre.to_pose7(c);
        const void* surf = planner_point->size() ? planner_point->points.data() : nullptr;
        const int rc = so_localize_global(context.h, surf, planner_point->size(), stride, ioff, c, &opts, &o, nullptr, 0, &last_global);
        check(rc, "so_localize_global");
        T_w_lidar = Transformd::from_pose7(last_global.pose);
        last_T_w_lidar = T_w_lidar;
        return rc;
    }

    // globalLocalize over the whole prior map, for a robot that restarts with no idea where it is (so_localize_global_bnb, same
    // result as so_localize_global on the same region): half_x / half_y are set from so_map_bounds so that the region covers the
    // surf map, so the centre supplies only z, roll/pitch and the yaw origin.  The other options (yaw_half, res, ...) are used as
    // given.  Sets T_w_lidar and last_T_w_lidar as globalLocalize does; last_bnb holds the search statistics.
    so_bnb_stats last_bnb{};
    template <class CloudPtr>
    int globalLocalizeInMap(const CloudPtr& planner_point, const Transformd& centre, so_global_opts opts) {
        return localizeInBox(planner_point, centre, opts, false);
    }

    // globalLocalizeInMap over the whole prior map held in the window AND the block archive (setArchive -> setOrigin -> loadPriorMap
    // first): the region is taken from so_map_bounds_all and whole_map is set, so the candidates are registered window by window and
    // the window is left where the winner is (so_global_opts.whole_map, superodom_b200.h).  Sets T_w_lidar, last_T_w_lidar, last_global
    // and last_bnb as globalLocalizeInMap does.
    template <class CloudPtr>
    int globalLocalizeInWholeMap(const CloudPtr& planner_point, const Transformd& centre, so_global_opts opts) {
        return localizeInBox(planner_point, centre, opts, true);
    }

    // Shim only: loop closure (so_keyframe_*, so_register_keyframes, so_map_from_keyframes; INTEGRATION.md "Loop closure").
    // addKeyframe keeps the scan the last Localization() registered, at T_w_lidar, and returns its id (localMap.reserveKeyframes first).
    int32_t addKeyframe() {
        double pose[7];
        T_w_lidar.to_pose7(pose);
        int32_t id = -1;
        check(so_keyframe_add_registered(context.h, pose, &id), "so_keyframe_add_registered");
        return id;
    }
    std::vector<Transformd> keyframePoses() const { return localMap.keyframePoses(); }
    // The keyframes ids registered against `submap` from priors (mode NONE: a keyframe is already compensated), with this SLAM's ICP
    // options: each result's pose and cov give a loop factor.  The live map and the registered scan are not touched.
    std::vector<so_icp_result> alignKeyframes(LocalMap& submap, const std::vector<int32_t>& ids, const std::vector<Transformd>& priors) {
        if (ids.size() != priors.size()) throw Error("alignKeyframes: one prior per keyframe id");
        submap.sync_resolution();
        so_icp_opts o{};
        o.max_icp_iters = int32_t(LocalizationICPMaxIter);
        o.max_surface_features = OptSet.max_surface_features;
        o.lm_max_iterations = 4;
        o.yaw_ratio = OptSet.yaw_ratio;
        std::vector<double> p(7 * priors.size());
        for (size_t i = 0; i < priors.size(); ++i) priors[i].to_pose7(p.data() + 7 * i);
        std::vector<so_icp_result> out(ids.size());
        check(so_register_keyframes(submap.ctx_->h, context.h, ids.data(), ids.size(), p.data(), &o, out.data()), "so_register_keyframes");
        return out;
    }
    // Loop detection (so_loop_candidates with loopOpts): the k keyframes whose Scan Context descriptors are closest to keyframe id's,
    // best first (id -1 in unused slots).  Thresholding the distance is the caller's policy (DESIGN.md, "Loop detection").
    so_loop_opts loopOpts = defaultLoopOpts();
    static so_loop_opts defaultLoopOpts() { so_loop_opts o{}; so_loop_opts_defaults(&o); return o; }
    std::vector<so_loop_candidate> loopCandidates(int32_t id, int32_t k) {
        std::vector<so_loop_candidate> out(size_t(k > 0 ? k : 0));
        check(so_loop_candidates(context.h, &id, 1, &loopOpts, k, out.data(), nullptr), "so_loop_candidates");
        return out;
    }
    // The alignment prior of a candidate for alignKeyframes, from keyframePoses(): the candidate keyframe's position, its heading
    // plus c.yaw, and the query's roll and pitch (so_loop_prior)
    Transformd loopPrior(const so_loop_candidate& c) const {
        const std::vector<Transformd> p = keyframePoses();
        if (c.id < 0 || size_t(c.id) >= p.size() || c.query < 0 || size_t(c.query) >= p.size()) throw Error("loopPrior: no such keyframe");
        double cand[7], query[7], out[7];
        p[size_t(c.id)].to_pose7(cand);
        p[size_t(c.query)].to_pose7(query);
        so_loop_prior(cand, query, c.yaw, out);
        return Transformd::from_pose7(out);
    }
    // Loop verification (so_loop_verify with loopVerifyOpts): each candidate's submap built in `scratch` (its map is overwritten), the
    // query aligned to it from loopPrior, and the alignment scored by overlap and visibility conflicts.  An accepted result's rel7 is
    // the loop edge (id, query) for optimizeKeyframes.  Unused slots (id -1) come back skipped.
    so_loop_verify_opts loopVerifyOpts = defaultLoopVerifyOpts();
    static so_loop_verify_opts defaultLoopVerifyOpts() { so_loop_verify_opts o{}; so_loop_verify_opts_defaults(&o); return o; }
    std::vector<so_loop_verify_result> verifyLoop(LocalMap& scratch, const std::vector<so_loop_candidate>& candidates,
                                                  const so_loop_verify_opts& opts) {
        scratch.sync_resolution();
        std::vector<so_loop_verify_result> out(candidates.size());
        check(so_loop_verify(context.h, scratch.ctx_->h, candidates.data(), candidates.size(), &opts, out.data()), "so_loop_verify");
        return out;
    }
    std::vector<so_loop_verify_result> verifyLoop(LocalMap& scratch, const std::vector<so_loop_candidate>& candidates) {
        return verifyLoop(scratch, candidates, loopVerifyOpts);
    }
    // The same with the degeneracy-aware alignment (so_loop_verify_degeneracy): in a corridor or along a long wall the alignment is
    // held along the directions it cannot measure, and `degeneracy[i]` says which; build candidate i's edge with loopEdge.
    // DESIGN.md, "Loop verification", gives the recommended thresholds (translation 0.2, rotation 0.1).
    struct VerifiedLoops { std::vector<so_loop_verify_result> results; std::vector<so_degeneracy_result> degeneracy; };
    VerifiedLoops verifyLoop(LocalMap& scratch, const std::vector<so_loop_candidate>& candidates, const so_degeneracy& d,
                             const so_loop_verify_opts& opts) {
        scratch.sync_resolution();
        VerifiedLoops out;
        out.results.resize(candidates.size());
        out.degeneracy.resize(candidates.size());
        check(so_loop_verify_degeneracy(context.h, scratch.ctx_->h, candidates.data(), candidates.size(), &opts, &d, out.results.data(),
                                        out.degeneracy.data()), "so_loop_verify_degeneracy");
        return out;
    }
    VerifiedLoops verifyLoop(LocalMap& scratch, const std::vector<so_loop_candidate>& candidates, const so_degeneracy& d) {
        return verifyLoop(scratch, candidates, d, loopVerifyOpts);
    }
    // The loop edge (v.id, v.query, Z = v.rel7) of an accepted degeneracy-aware verification for optimizeKeyframes: S (6x6 row-major,
    // x, y, z, rx, ry, rz; from stated sigmas) without the directions the alignment left unconstrained (so_loop_edge_information), so
    // the graph takes them from the other edges; `cauchy` as so_pose_edge.cauchy
    static so_pose_edge loopEdge(const so_loop_verify_result& v, const so_degeneracy_result& deg, const double S[36], double cauchy) {
        so_pose_edge e{};
        e.i = v.id;
        e.j = v.query;
        for (int k = 0; k < 7; ++k) e.z[k] = v.rel7[k];
        check(so_loop_edge_information(v.reg.pose, &deg, S, e.sqrt_info), "so_loop_edge_information");
        e.cauchy = cauchy;
        return e;
    }
    // loopCandidates over the keyframes [begin, end) only (so_loop_candidates_range with loopOpts; its exclude_recent is not used):
    // a live-session keyframe searched against an earlier session's ids, wherever they lie in the store
    std::vector<so_loop_candidate> loopCandidatesIn(int32_t id, int32_t k, int32_t begin, int32_t end) {
        std::vector<so_loop_candidate> out(size_t(k > 0 ? k : 0));
        check(so_loop_candidates_range(context.h, &id, 1, &loopOpts, begin, end, k, out.data(), nullptr), "so_loop_candidates_range");
        return out;
    }
    // The keyframe pose graph solved on the device (so_pose_graph_solve_constant): edges between keyframe ids, the keyframes where
    // constant[id] != 0 held, started from `init` (one pose per keyframe) or, when it is empty, from keyframePoses().  A live session
    // joined to an earlier one starts from its poses moved into the earlier frame by the loop result (INTEGRATION.md, "Sessions"):
    // the solve is local and does not cross a large change of frame by itself.  The store's poses are not changed: pass `poses` to
    // mergeKeyframes or rebuildFromKeyframes.
    struct GraphSolution { std::vector<Transformd> poses; so_pose_graph_result result{}; std::vector<double> weights; };
    GraphSolution optimizeKeyframes(const std::vector<so_pose_edge>& edges, const std::vector<uint8_t>& constant,
                                    const so_pose_graph_opts& opts, const std::vector<Transformd>& init = {}) {
        const std::vector<Transformd> est = init.empty() ? keyframePoses() : init;
        if (constant.size() != est.size()) throw Error("optimizeKeyframes: one constant flag per keyframe");
        std::vector<double> x(7 * est.size());
        for (size_t i = 0; i < est.size(); ++i) est[i].to_pose7(x.data() + 7 * i);
        GraphSolution out;
        out.weights.resize(edges.size());
        check(so_pose_graph_solve_constant(context.h, x.data(), est.size(), edges.data(), edges.size(), constant.data(), &opts, x.data(),
                                           out.weights.data(), &out.result), "so_pose_graph_solve_constant");
        for (size_t i = 0; i < est.size(); ++i) out.poses.push_back(Transformd::from_pose7(x.data() + 7 * i));
        return out;
    }
    // The live session continues in the frame of `corrected` (one pose per keyframe, in id order; an earlier session's keyframes held
    // constant in it): the change of frame C = corrected[live_id] * est[live_id]^-1 at the live session's newest keyframe live_id moves
    // T_w_lidar, last_T_w_lidar and undistort_prev_pose; the window is re-centred at the new T_w_lidar; then both stores are rebuilt
    // from every keyframe.  The window goes first: the corrected frame can lie far from the old one, and a rebuild under the old window
    // would drop (or archive) the map around the sensor.
    void mergeKeyframes(const std::vector<Transformd>& corrected, int32_t live_id) {
        const std::vector<Transformd> est = keyframePoses();
        if (corrected.size() != est.size()) throw Error("mergeKeyframes: one corrected pose per keyframe");
        if (live_id < 0 || size_t(live_id) >= est.size()) throw Error("mergeKeyframes: no such keyframe");
        const Transformd C = corrected[size_t(live_id)] * est[size_t(live_id)].inverse();
        T_w_lidar = C * T_w_lidar;
        last_T_w_lidar = C * last_T_w_lidar;
        undistort_prev_pose = C * undistort_prev_pose;
        localMap.setOrigin(T_w_lidar.pos);
        std::vector<int32_t> ids(corrected.size());
        for (size_t i = 0; i < ids.size(); ++i) ids[i] = int32_t(i);
        localMap.buildFromKeyframes(localMap, ids, corrected);
    }
    // mergeKeyframes, then both stores cleared against every keyframe at its corrected pose (so_map_clear_free_space_keyframes with
    // `clear`), so the merged map keeps out what either session's free-space clearing had removed.  last_keyframe_clear holds the result.
    so_free_space_keyframes_result last_keyframe_clear{};
    void mergeKeyframes(const std::vector<Transformd>& corrected, int32_t live_id, const so_free_space& clear) {
        mergeKeyframes(corrected, live_id);
        clearAllKeyframes(corrected, clear);
    }
    // The map rebuilt from every keyframe at the corrected poses (one per keyframe, in id order), both stores; T_w_lidar and
    // last_T_w_lidar become the corrected pose of the last keyframe, so the next Localization() continues from the corrected map.
    void rebuildFromKeyframes(const std::vector<Transformd>& corrected) {
        std::vector<int32_t> ids(corrected.size());
        for (size_t i = 0; i < ids.size(); ++i) ids[i] = int32_t(i);
        localMap.buildFromKeyframes(localMap, ids, corrected);
        if (!corrected.empty()) { T_w_lidar = corrected.back(); last_T_w_lidar = T_w_lidar; }
        undistort_prev_pose = T_w_lidar;
    }
    // rebuildFromKeyframes, then both stores cleared against every keyframe at its corrected pose (so_map_clear_free_space_keyframes
    // with `clear`): with ClearFreeSpace on, the rebuilt map would otherwise bring back every point the live clearing removed.
    // last_keyframe_clear holds the result.
    void rebuildFromKeyframes(const std::vector<Transformd>& corrected, const so_free_space& clear) {
        rebuildFromKeyframes(corrected);
        clearAllKeyframes(corrected, clear);
    }

private:
    void clearAllKeyframes(const std::vector<Transformd>& corrected, const so_free_space& clear) {
        std::vector<int32_t> ids(corrected.size());
        for (size_t i = 0; i < ids.size(); ++i) ids[i] = int32_t(i);
        last_keyframe_clear = localMap.clearFreeSpaceFromKeyframes(localMap, ids, corrected, clear, 3);
    }

public:
    // LidarSLAM::EstimateLidarUncertainty (LidarSlam.cpp:915-975)
    void EstimateLidarUncertainty() {
        const auto& h = PlaneFeatureHistogramObs;
        const double tt = double(h[6]) + double(h[7]) + double(h[8]);
        const double tr = double(h[0]) + h[1] + h[2] + h[3] + h[4] + h[5];
        auto cap = [](double v) { return v < 1.0 ? v : 1.0; };
        lidarOdomUncer.uncertainty_x = cap(h[6] / tt * 3); lidarOdomUncer.uncertainty_y = cap(h[7] / tt * 3); lidarOdomUncer.uncertainty_z = cap(h[8] / tt * 3);
        lidarOdomUncer.uncertainty_roll = cap((double(h[0]) + h[1]) / tr * 3); lidarOdomUncer.uncertainty_pitch = cap((double(h[2]) + h[3]) / tr * 3);
        lidarOdomUncer.uncertainty_yaw = cap((double(h[4]) + h[5]) / tr * 3);
        if (tt == 0 || tr == 0) lidarOdomUncer = LidarOdomUncertainty{};
        stats.uncertainty_x = lidarOdomUncer.uncertainty_x; stats.uncertainty_y = lidarOdomUncer.uncertainty_y; stats.uncertainty_z = lidarOdomUncer.uncertainty_z;
        stats.uncertainty_roll = lidarOdomUncer.uncertainty_roll; stats.uncertainty_pitch = lidarOdomUncer.uncertainty_pitch; stats.uncertainty_yaw = lidarOdomUncer.uncertainty_yaw;
    }

private:
    // globalLocalizeInMap (whole = false) / globalLocalizeInWholeMap (whole = true)
    template <class CloudPtr>
    int localizeInBox(const CloudPtr& planner_point, const Transformd& centre, so_global_opts opts, bool whole) {
        localMap.sync_resolution();
        size_t stride, ioff;
        using PointT = typename std::decay<decltype(planner_point->points[0])>::type;
        point_layout<PointT>(&stride, &ioff);
        so_icp_opts o{};
        o.max_icp_iters = int32_t(LocalizationICPMaxIter);
        o.max_surface_features = OptSet.max_surface_features;
        o.lm_max_iterations = 4;
        o.yaw_ratio = OptSet.yaw_ratio;
        double c[7];
        centre.to_pose7(c);
        float lo[3], hi[3];
        size_t n_map = 0;
        if (whole) {
            check(so_map_bounds_all(context.h, lo, hi, &n_map), "so_map_bounds_all");
            opts.whole_map = 1;
        } else {
            check(so_map_bounds(context.h, lo, hi, &n_map), "so_map_bounds");
        }
        auto half = [](double l, double h, double x) { const double a = h - x, b = x - l; return a > b ? (a > 0.0 ? a : 0.0) : (b > 0.0 ? b : 0.0); };
        opts.half_x = half(lo[0], hi[0], c[0]);
        opts.half_y = half(lo[1], hi[1], c[1]);
        const void* surf = planner_point->size() ? planner_point->points.data() : nullptr;
        const int rc = so_localize_global_bnb(context.h, surf, planner_point->size(), stride, ioff, c, &opts, &o, nullptr, 0, &last_global,
                                             &last_bnb);
        check(rc, "so_localize_global_bnb");
        T_w_lidar = Transformd::from_pose7(last_global.pose);
        last_T_w_lidar = T_w_lidar;
        return rc;
    }

    static void check(int rc, const char* what) { if (rc < 0) throw Error(std::string(what) + ": " + so_last_error()); }
};

}  // namespace b200
}  // namespace super_odometry
