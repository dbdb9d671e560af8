/* =============================================================================
 * superodom_b200.h -- C ABI of the H100-native (sm_90a) ICP registration hot path.
 *
 * This is the drop-in boundary for ONE path of superxslam/SuperOdom: the per-scan
 * registration in LidarSLAM::performLocalizationAndMapping.  The reference has no
 * FFI layer; its seam is the C++ class surface of LidarSLAM / LocalMap as used by
 * laserMapping (SURVEY.md section 8b).  Each entry point below names the reference
 * interface it replaces (file:line under /root/reference/super_odometry/).  The C++
 * shim include/superodom_b200/LidarSlam.hpp keeps the reference member names and
 * forwards to these functions; INTEGRATION.md shows the maintainer-side binding.
 *
 * Conventions
 *   - plain pointers and sizes only; caller owns every host buffer; the context owns
 *     all device memory, streams and CUDA graphs; no allocation crosses the ABI.
 *   - pose7 = {tx,ty,tz,qx,qy,qz,qw}: the reference's pose_parameters layout
 *     (src/LidarProcess/LidarSlam.cpp:7-9).
 *   - point clouds are arrays of points with a byte stride; x,y,z are floats at byte
 *     offsets 0,4,8 and intensity is a float at byte offset `intensity_offset`
 *     (pcl::PointXYZI: stride 32, intensity at 16; packed float4: stride 16, at 12).
 *   - return value: 0 = ok; >0 = reference-defined soft status (see SO_STATUS_*);
 *     <0 = CUDA / argument error, text via so_last_error().  Nothing throws.
 *   - one host thread per context, one context per GPU (the reference is
 *     non-reentrant: file-scope pose globals, LidarSlam.cpp:7-9).
 *   - there is NO CPU fallback: every entry point fails with SO_ERR_CUDA when no
 *     sm_90 device / kernel image is available.
 * ============================================================================= */
#ifndef SUPERODOM_B200_H
#define SUPERODOM_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SO_MAX_ICP_ITERS 32

/* soft statuses (>0) and errors (<0) */
#define SO_OK 0
#define SO_STATUS_NOT_ENOUGH_FEATURES 1 /* hasEnoughFeatures() false: pose = prior (LidarSlam.cpp:113-116,379-381) */
#define SO_STATUS_NO_CORRESPONDENCES 2  /* every scan point was rejected; reference would CHECK-fail in ceres::Covariance */
#define SO_STATUS_INVALID_EVALUATION 3  /* the first evaluation of an ICP iteration's solve has a non-finite cost: an edge row weighted NaN
                                           (line fit on an exactly collinear neighbourhood); the reference CHECK-fails in ceres::Corrector.
                                           pose = the pose that ICP iteration started from, its iter_cost NaN, cov and errors zero */
#define SO_ERR_ARG (-1)
#define SO_ERR_CUDA (-2)
#define SO_ERR_CAPACITY (-3)

/* LidarSLAM::MatchingResult (include/super_odometry/LidarProcess/LidarSlam.h:85-94) */
enum so_match_result {
    SO_MATCH_SUCCESS = 0, SO_MATCH_NOT_ENOUGH_NEIGHBORS = 1, SO_MATCH_NEIGHBORS_TOO_FAR = 2,
    SO_MATCH_BAD_PCA_STRUCTURE = 3, SO_MATCH_INVALID_NUMERICAL = 4, SO_MATCH_MSE_TOO_LARGE = 5,
    SO_MATCH_UNKNOWN = 6, SO_MATCH_N = 7,
    SO_MATCH_SKIPPED = 255 /* not in the reference: point dropped by shouldProcessPoint (LidarSlam.cpp:353-359) */
};

typedef struct so_ctx so_ctx;

/* Construction-time capacities.  Zero fields take defaults. */
typedef struct {
    int32_t device;            /* CUDA device ordinal */
    uint32_t max_map_points;   /* default 4,194,304 */
    uint32_t max_scan_points;  /* per scan, default 262,144 */
    uint32_t max_batch;        /* scans registered concurrently by so_register_batch*, default 1 */
    float line_res;            /* LocalMap::lineRes_  (LocalMap.h:761; node default laserMapping.cpp:102-103) */
    float plane_res;           /* LocalMap::planeRes_ (LocalMap.h:762) */
} so_config;

/* Per-call options == the LidarSLAM members laserMapping writes (laserMapping.cpp:102-120,703-711). */
typedef struct {
    int32_t max_icp_iters;        /* LidarSLAM::LocalizationICPMaxIter (LidarSlam.h:273); config max_iterations */
    int32_t max_surface_features; /* OptSet.max_surface_features (LidarSlam.h:118); 0 = uncapped */
    int32_t lm_max_iterations;    /* ceres options.max_num_iterations = 4 (LidarSlam.cpp:232); 0 -> 4 */
    float yaw_ratio;              /* OptSet.yaw_ratio (LidarSlam.cpp:905) */
    int32_t skip_map_checks;      /* 1: do not run shiftMap / hasEnoughFeatures (replay against a frozen map) */
    /* SE3AbsolutatePoseFactor on T_w_initial_guess (LidarSlam.cpp:281-298): set when shouldAddAbsolutePoseConstraints()
     * holds, i.e. predictodom == VIO_ODOM && isDegenerate && Visual_confidence_factor != 0 (dormant in the shipped node:
     * isDegenerate is never set, LidarSlam.cpp:976-985). */
    int32_t use_pose_prior;
    float visual_confidence_factor;   /* LidarSLAM::Visual_confidence_factor */
    float prior_uncertainty[3];       /* lidarOdomUncer.uncertainty_{x,y,z} (EstimateLidarUncertainty, LidarSlam.cpp:915-964) */
} so_icp_opts;

/* Everything the reference leaves in LidarSLAM members after Localization():
 * T_w_lidar, stats (OptimizationStats.msg), LocalizationUncertainty (RegistrationError, LidarSlam.h:122-148),
 * PlaneFeatureHistogramObs / MatchRejectionHistogram* (LidarSlam.h:267-269). */
typedef struct {
    double pose[7];       /* T_w_lidar after MannualYawCorrection (LidarSlam.cpp:891-913) */
    double pose_opt[7];   /* optimiser output (pose_parameters) before the RPY round trip */
    int32_t status;       /* SO_OK / SO_STATUS_* */
    int32_t n_iterations; /* ICP iterations executed (stats.iterations.size()) */
    int32_t iter_n_surf[SO_MAX_ICP_ITERS];        /* IterationStats.num_surf_from_scan */
    int32_t iter_n_edge[SO_MAX_ICP_ITERS];        /* IterationStats.num_corner_from_scan */
    double iter_dtrans[SO_MAX_ICP_ITERS];         /* IterationStats.translation_norm */
    double iter_drot[SO_MAX_ICP_ITERS];           /* IterationStats.rotation_norm */
    int32_t iter_lm_steps[SO_MAX_ICP_ITERS];      /* ceres summary: iterations of this solve (diagnostic) */
    int32_t iter_lm_successful[SO_MAX_ICP_ITERS]; /* ceres summary.num_successful_steps (drives the break, :141) */
    int32_t iter_lm_termination[SO_MAX_ICP_ITERS];/* 0 max-iter 1 gradient 2 parameter 3 function 4 radius 5 invalid 6 empty */
    double iter_cost[SO_MAX_ICP_ITERS];           /* final cost of this solve */
    int32_t hist_obs[9];          /* PlaneFeatureHistogramObs of the last ICP iteration */
    int32_t hist_reject_plane[7]; /* MatchRejectionHistogramPlane of the last ICP iteration */
    int32_t hist_reject_line[7];  /* MatchRejectionHistogramLine of the last ICP iteration (all 0 without an edge cloud) */
    double cov[36];               /* RegistrationError::Covariance, row-major, order x,y,z,rx,ry,rz */
    double pos_err, pos_dir[3], pos_inv_cond;     /* PositionError, PositionErrorDirection, PosInverseConditionNum (a negative
                                                     rounding of the smallest eigenvalue below a cut direction reads as 0, not NaN) */
    double ori_err_deg, ori_dir[3], ori_inv_cond; /* OrientationError (degrees), ...Direction, OriInverseConditionNum */
    double total_translation, total_rotation, translation_from_last, rotation_from_last; /* stats.* (LidarSlam.cpp:198-210) */
    int32_t map_surf_5x5, map_edge_5x5, scan_surf_num, scan_edge_num; /* stats.laser_cloud_* (LidarSlam.cpp:371-377) */
    int32_t pos_in_localmap[3];   /* LidarSLAM::pos_in_localmap (shiftMap return) */
    int32_t prediction_source;    /* stats.prediction_source: 1 when the pose prior rows were added (LidarSlam.cpp:278,297) */
    double time_ms;               /* stats.time_elapsed: the ICP loop, device time measured with CUDA events */
    double time_total_ms;         /* whole so_register call incl. H2D / D2H (host clock) */
    int32_t knn_searched;         /* reserved, always 0 */
    int32_t knn_verified;         /* reserved, always 0 */
} so_icp_result;

/* One accepted/rejected plane correspondence, for stage-level parity tests
 * (LidarSLAM::OptimizationParameter, LidarSlam.h:209-222, reduced to what the solver reads). */
typedef struct {
    double n[3];      /* NormDir */
    double d;         /* negative_OA_dot_norm */
    double w;         /* residualCoefficient */
    uint32_t nn[5];   /* neighbour ids = index of the map point in the order given to so_map_set_points / so_map_add_surf output */
    float nn_d2[5];
    uint8_t status;   /* so_match_result */
    uint8_t obs[3];   /* Feature_observability labels histogrammed (LidarSlam.cpp:336-339) */
    uint8_t pad_[4];
} so_corr;

/* One edge / line correspondence (stage-level parity of the dormant edge branch, LidarSlam.cpp:402-493). */
typedef struct {
    double a[3], b[3];      /* corres: mean +- 0.1 * line direction */
    double w;               /* residualCoefficient */
    uint32_t nn[10];        /* the 10 nearest edge-map points (ids as given to so_map_set_edge_points / insert output order) */
    uint32_t selected_mask; /* bit j: nn[j] kept by nearestKSearchSpecificEdgePoint's best-line selection (bit 0 always) */
    uint8_t status;         /* so_match_result */
    uint8_t n_selected;
    uint8_t pad_[2];
} so_edge_corr;

/* ---- lifetime ------------------------------------------------------------------------------------ */
/* replaces: LidarSLAM::LidarSLAM() + LocalMap::LocalMap() (LidarSlam.cpp:14-19, LocalMap.h:141-144) */
so_ctx* so_create(const so_config* cfg);
void so_destroy(so_ctx* ctx);
const char* so_last_error(void);
/* 1 when a CUDA device of compute capability 9.x is usable by this library */
int so_device_available(void);
/* Use an externally owned CUDA stream (cudaStream_t as void*) for all work of this context; NULL = own stream. */
int so_set_stream(so_ctx* ctx, void* cuda_stream);

/* ---- map (LocalMap) ------------------------------------------------------------------------------- */
/* replaces: slam.localMap.lineRes_/planeRes_ = ... (laserMapping.cpp:102-103,648-649). Rebuilds the neighbour
 * index when plane_res changes (cell edge derives from sqrt(3*planeRes)). */
int so_map_set_resolution(so_ctx* ctx, float line_res, float plane_res);
/* replaces: LocalMap::setOrigin (LocalMap.h:146-164): origin_ = -blockOf(t).  out_origin may be NULL. */
int so_map_set_origin(so_ctx* ctx, const double t_w_cur[3], int32_t out_origin[3]);
int so_map_get_origin(so_ctx* ctx, int32_t out_origin[3]);
/* replaces: LocalMap::shiftMap (LocalMap.h:169-287): roll the 21x21x11 block grid so the sensor block stays in
 * [3,17]x[3,17]x[3,7]; blocks rolled off the grid are dropped.  Returns the sensor block in out_ijk. */
int so_map_shift(so_ctx* ctx, const double t_w_cur[3], int32_t out_ijk[3]);
/* Load an ALREADY voxel-filtered world-frame surf cloud as the whole map (no filtering): replay / localization
 * mode with a prebuilt map.  Point ids (so_corr.nn) are indices into this array.
 * A store counts as built only once its neighbour index is: when a map change cannot build it (SO_ERR_CAPACITY: the map spans
 * too many 50 m blocks for the cell table at this planeRes; SO_ERR_CUDA), every later call that reads the map (registration,
 * k-NN, global localization, so_map_counts_5x5, so_map_download, so_map_shift, the inserts) returns the same error until a
 * later change lets the index build, e.g. so_map_set_points of a smaller cloud. */
int so_map_set_points(so_ctx* ctx, const void* xyzi, size_t n, size_t stride_bytes, size_t intensity_offset);
/* Same for the edge clouds (MapBlock::pedge_pc_): an already lineRes-filtered world-frame edge cloud as the whole edge map. */
int so_map_set_edge_points(so_ctx* ctx, const void* xyzi, size_t n, size_t stride_bytes, size_t intensity_offset);
/* replaces: LocalMap::addSurfPointCloud (LocalMap.h:591-645): bin world-frame points into blocks, voxel-centroid
 * filter every touched block at leaf planeRes (pcl::VoxelGrid semantics), rebuild the neighbour index.  When the index cannot
 * be built, the filtered points stay in the store and it stays unbuilt, with the rule of so_map_set_points. */
int so_map_add_surf(so_ctx* ctx, const void* xyzi, size_t n, size_t stride_bytes, size_t intensity_offset);
/* replaces: LocalMap::addEdgePointCloud (LocalMap.h:529-589): the same insert at leaf lineRes into the edge clouds. */
int so_map_add_edge(so_ctx* ctx, const void* xyzi, size_t n, size_t stride_bytes, size_t intensity_offset);
/* replaces: LidarSLAM::transformAndAddToMap(cloud, world_cloud, false) (LidarSlam.cpp:60-80): transform the
 * sensor-frame scan by pose (utils::TransformPoint: double math, float store) on the device, then so_map_add_surf. */
int so_map_add_scan(so_ctx* ctx, const void* xyzi, size_t n, size_t stride_bytes, size_t intensity_offset, const double pose[7]);
/* Same insert for the surf cloud of the last single-scan registration (so_register, so_register_prefiltered, so_register_undistort,
 * so_register_optimized and their prefiltered forms, so_localize_global*), which is still in device memory: the live loop
 * Localization() -> transformAndAddToMap() (LidarSlam.cpp:155-171) without uploading the scan a second time.  Fails with SO_ERR_ARG,
 * before any device work, when a call that reuses the scan buffers ran in between: so_scan_prefilter, so_scan_deskew,
 * so_scan_extract_uniform, so_correspond, so_correspond_seeded, so_register_injected, the host batches so_register_batch*, so_evaluate_optimized,
 * so_solve_optimized (not so_register_batch_device, the k-NN, the other map calls, so_undistort_points, so_correspond_edge or so_solve).  SO_OK and nothing inserted
 * before the first registration. */
int so_map_add_registered_scan(so_ctx* ctx, const double pose[7]);
/* ... and transformAndAddToMap(cloud, world_cloud, true) for the edge cloud. */
int so_map_add_scan_edge(so_ctx* ctx, const void* xyzi, size_t n, size_t stride_bytes, size_t intensity_offset, const double pose[7]);
/* The same insert for the edge cloud of the last single-scan registration, which is still in device memory.  After so_register it
 * inserts exactly what so_map_add_scan_edge of the same cloud inserts; after so_register_undistort_edges it inserts the edge cloud
 * undistorted with the D that pose gives, world = T(pose) * pInit, and after so_register_optimized_edges T(pose) * u_e(D_opt), as
 * so_map_add_registered_scan does for the surf cloud.  Fails
 * with SO_ERR_ARG, before any device work, whenever so_map_add_registered_scan would, and after so_correspond_edge.  SO_OK and
 * nothing inserted when that registration had no edge cloud (every other so_register* entry point). */
int so_map_add_registered_edges(so_ctx* ctx, const double pose[7]);
/* replaces: LocalMap::get5x5LocalMapFeatureSize (LocalMap.h:291-318) */
int so_map_counts_5x5(so_ctx* ctx, const int32_t ijk[3], int32_t* n_edge, int32_t* n_surf);
/* replaces: LocalMap::getAllLocalMap (mode 0, LocalMap.h:647-658) / get5x5LocalMap(pos) (mode 1, :660-687).
 * Writes packed float4 {x,y,z,intensity} in block order then point-id order; *n_out = points available. */
int so_map_download(so_ctx* ctx, int mode, const int32_t ijk[3], float* out_xyzi, size_t cap_points, size_t* n_out);
size_t so_map_size(so_ctx* ctx);
/* ---- block archive: the map beyond the 21x21x11 window ------------------------------------------------------------------------
 * Off by default; while it is off every call above behaves as LocalMap does and nothing is allocated for it.  With it on, each store
 * behaves like a LocalMap over an UNBOUNDED block grid that every search sees through the window.  A block is named by its world
 * block coordinate w = g - origin (g: the grid index LocalMap.h:594-605 gives a point; w does not depend on the origin).
 *   - Eviction: when an origin change (so_map_shift, so_map_set_origin, the shift inside a single-scan registration) moves a
 *     non-empty block out of the window, the rebuild that applies it moves the block's cloud to the archive unchanged: the same
 *     points in the same order.  Non-finite points are still dropped, and so are points more than 2^19 blocks (26 214 km) from the
 *     world origin.
 *   - Restore: when an origin change moves an archived block back into the window, its cloud comes back unchanged and leaves the
 *     archive.  A block's point order is its k-NN tie-break and its voxel-filter order, so registrations against restored blocks
 *     give what they gave before the blocks left, bit for bit (only so_corr.nn ids, positions in the store, may differ).
 *   - Loading: so_map_set_points / so_map_set_edge_points replace the window and the archive together; points outside the window go
 *     to the archive, so setOrigin(start) followed by the prior-map load keeps the whole map.  They accept up to max_map_points +
 *     cap_points points; SO_ERR_CAPACITY, before any change, when the part inside the window exceeds max_map_points or the rest
 *     exceeds cap_points.
 *   - Inserts are unchanged: so_map_add_* and the registered-scan inserts filter the window blocks they touch and drop points
 *     outside the window.  This is the one place where a store differs from an unbounded map.
 *   - Every read (registration, k-NN, so_map_counts_5x5, so_map_download, so_map_bounds) sees the window only.  Global localization
 *     sees the window only unless so_global_opts.whole_map is 1; so_map_bounds_all covers the window and the archive.
 *   - Nothing is lost silently: an eviction the archive has no room for fails the call that applies it with SO_ERR_CAPACITY and
 *     leaves the store unbuilt, with the rule of so_map_set_points; growing the archive recovers it with nothing lost, turning it off
 *     recovers it by dropping the blocks.
 * so_map_archive: turn the archive on with room for cap_points points per store; again with another value to resize it (contents
 * kept; SO_ERR_CAPACITY when the value is below what a store holds; both stores change or neither); 0 turns it off and frees it
 * with its contents.
 * Host cost: with the archive on, so_map_set_points / so_map_set_edge_points classify and stably sort the cloud on the host (a host
 * copy of the whole cloud, O(n log n)), and so_map_download_all copies the window and the whole pool to the host; both are meant for
 * one-time loads and saves.  Shifts and origin changes run on the device and cost the blocks that move. */
int so_map_archive(so_ctx* ctx, size_t cap_points);
/* Points and blocks held in the archive of store 0 (surf) or 1 (edge), and its capacity; any pointer may be NULL. */
int so_map_archive_info(so_ctx* ctx, int store, size_t* n_points, size_t* n_blocks, size_t* cap_points);
/* The whole map of store 0 (surf) or 1 (edge): the window plus the archive as packed float4 {x,y,z,intensity}, ordered by world
 * block (z, then y, then x) and by the order within the block.  *n_out = points available (only cap_points are written).  Saved and
 * loaded with so_map_set_points, it is the next session's prior map. */
int so_map_download_all(so_ctx* ctx, int store, float* out_xyzi, size_t cap_points, size_t* n_out);

/* ---- keyframes: registered scans kept on the device, and the map rebuilt from them after a loop closure --------------------------
 * No reference counterpart (the reference is an odometry front end).  What a loop-closing back end needs from the device: the scans
 * with their poses, a submap built from chosen scans to register a kept scan against (the loop constraint: pose and cov), and the map
 * rebuilt from every keyframe once a pose graph has moved them (so_pose_graph_solve below, or the caller's own).  Off until
 * so_keyframe_reserve; nothing else calls these, and no other call changes behaviour.
 * so_keyframe_reserve: one pool of cap_points points for surf clouds and one for edge clouds, and room for cap_frames keyframes; again
 * with other values to resize (contents kept); 0, 0 frees the store.  SO_ERR_ARG when only one of the two is 0 or when either is below
 * what the store holds. */
int so_keyframe_reserve(so_ctx* ctx, size_t cap_points, size_t cap_frames);
/* Keep the scan of the last single-scan registration (and its edge cloud when it had one) as keyframe *id (0, 1, ... in call order),
 * with pose.  Each cloud is kept exactly as so_map_add_registered_scan / so_map_add_registered_edges would place it before the world
 * transform: in the sensor frame and, after APPROXIMATED / OPTIMIZED registration, compensated with pose as the insert would be.  The
 * map is not touched.  SO_ERR_ARG, before any device work, without a store, for a non-finite pose, before the first registration or
 * after one of an empty scan, and whenever so_map_add_registered_scan would fail (or so_map_add_registered_edges, when the
 * registration had an edge cloud).  SO_ERR_CAPACITY
 * with the store unchanged when a pool or the frame table is full. */
int so_keyframe_add_registered(so_ctx* ctx, const double pose[7], int32_t* id);
/* Append one keyframe from host clouds, as *id: surf_xyzi[n_surf] and edge_xyzi[n_edge] (either count may be 0), records of
 * stride_bytes with x, y, z floats at 0 and the intensity float at intensity_offset (0 when it lies past the record), already in the
 * sensor frame and already compensated, at pose.  The clouds are kept verbatim: so_keyframe_download(id, store, NULL) returns them bit
 * for bit, so a session's keyframes saved through so_keyframe_poses and so_keyframe_download come back unchanged in another context.
 * The registered scan, the map and every other keyframe's cached descriptor are not touched; the new keyframe is described lazily,
 * as any other.  SO_ERR_ARG, before any device work, without a store, for a non-finite pose, a NULL cloud with a non-zero count or
 * stride_bytes < 12; SO_ERR_CAPACITY with the store unchanged when a pool or the frame table is full. */
int so_keyframe_import(so_ctx* ctx, const void* surf_xyzi, size_t n_surf, const void* edge_xyzi, size_t n_edge, size_t stride_bytes,
                       size_t intensity_offset, const double pose[7], int32_t* id);
/* Keyframes held and the points of the surf and edge pools; any pointer may be NULL. */
int so_keyframe_info(so_ctx* ctx, size_t* n_frames, size_t* n_points, size_t* n_edge_points);
/* The keyframes' poses, [*n][7]; only cap are written.  A pose is the one the keyframe was added with, or the one the last
 * so_map_from_keyframes of its own context (dst == src) rebuilt it at. */
int so_keyframe_poses(so_ctx* ctx, double* out7, size_t cap, size_t* n);
/* Keyframe id of store 0 (surf) or 1 (edge) as packed float4 {x,y,z,intensity}: in the sensor frame (pose7 NULL), or at pose7 by the
 * device arithmetic of so_map_add_scan and so_map_from_keyframes (qrot in double, float store).  *n_out = its points; only cap_points
 * are written.  SO_ERR_ARG for an id the store does not hold. */
int so_keyframe_download(so_ctx* ctx, int32_t id, int store, const double pose7[7], float* out_xyzi, size_t cap_points, size_t* n_out);
/* Replace the selected stores of dst (stores: 1 surf, 2 edge, 3 both) with the map of src's keyframes ids[0..n_ids), keyframe ids[i]
 * at poses7[i].  dst == src is the rebuild after a pose-graph correction (the keyframes' poses become poses7); another context on the
 * same device builds a loop-verification submap.  The result, under dst's origin and leaf (planeRes surf, lineRes edge):
 *   - the union is the keyframes in ids order, each in its point order, each point transformed as so_keyframe_download(pose) does;
 *   - every 50 m block of the union is filtered on its own, as an insert filters a touched block (pcl::VoxelGrid, centroids summed in
 *     union order); the window's blocks make the window's cloud, block by block;
 *   - with the block archive on, every block outside the window is filtered the same way and becomes dst's archive; with it off,
 *     those blocks are dropped, as an insert drops them.
 * One filter over the union, not a replay of inserts (which average centroids of centroids): rebuilding at unchanged poses gives a
 * different, cleaner map than the live one.  The rebuilt stores hold their keyframes and nothing else: a prior map loaded with
 * so_map_set_points, and points free-space clearing removed, are not kept (so_map_clear_free_space_keyframes clears the rebuilt map
 * against the keyframes).  The index is rebuilt as by any map change.
 * SO_ERR_ARG, before any device work, for contexts on different devices, an id src does not hold, a non-finite pose or stores outside
 * 1..3.  SO_ERR_CAPACITY, with both stores as they were, when the window's points exceed max_map_points, the off-window blocks exceed
 * the archive, the window's blocks exceed the cell table, or 2^31 points or more are selected. */
int so_map_from_keyframes(so_ctx* dst, so_ctx* src, const int32_t* ids, size_t n_ids, const double* poses7, int stores);

/* ---- loop detection: which old keyframe a new one revisits (Scan Context, Kim & Kim, IROS 2018) ---------------------------------
 * No reference counterpart.  Appearance-based, so it does not read the drifted positions of the keyframes: each keyframe is described
 * by a polar max-height image of its surf cloud, and a query is compared with every eligible keyframe at every column shift.  The
 * search is exhaustive (no ring-key prefilter); thresholding the distance is the caller's policy (DESIGN.md, "Loop detection").
 * Descriptor of keyframe i, in FP64 without contractible multiply-adds (DESIGN.md gives the exact expression order):
 *   - levelling: R = R(q_i) of its CURRENT pose (so_keyframe_poses), psi = atan2(R10, R00), L = Rz(-psi) R: roll and pitch come from
 *     the pose, heading is left out; each finite point p of the sensor-frame surf cloud goes to v = L p;
 *   - rho = hypot(vx, vy), points with rho >= max_range skipped; ring floor(rho / max_range * rings) (at most rings - 1);
 *     az = atan2(vy, vx) in [-pi, pi), sector floor((az + pi) / (2 pi / sectors)), at most sectors - 1;
 *   - cell value: the maximum of max(0, float(vz + height_offset)) over its points, 0 when empty (a cell whose maximum height lies
 *     below -height_offset reads 0); column norms in FP64, summed in ring order.
 * Distance of query a to candidate b at shift s: over query columns j with candidate column (j + s) mod sectors, pairs where both norms
 * are non-zero, d = 1 - (sum of cosines in ascending j) / n_pairs, each dot summed in ring order in FP64; d = 1 with no pair.  The pair
 * distance is the minimum over s, ties to the lowest s; yaw = s * 2 pi / sectors wrapped to (-pi, pi] is the query's heading minus the
 * candidate's, in their levelled frames.
 * Descriptors are cached per keyframe and computed lazily by the calls below: a descriptor is valid for the options and the pose it
 * was computed with (the self-rebuild of so_map_from_keyframes marks the keyframes it moves stale; other options invalidate all).  No
 * other call launches anything for them.  Both calls fail with SO_ERR_ARG, before any device work, without a keyframe store, for an id
 * the store does not hold, and for options outside: rings 1..64, sectors 2..360 (the query image and its norms, at most 95 040 B, sit
 * in shared memory), max_range finite and > 0, height_offset finite, exclude_recent >= 0. */
typedef struct {
    int32_t rings;            /* default 20 */
    int32_t sectors;          /* default 60 */
    double max_range;         /* metres, default 80 */
    double height_offset;     /* the sensor's height above the ground, metres, default 2.0 */
    int32_t exclude_recent;   /* keyframe id is eligible for query q when id < q - exclude_recent; default 30 */
    int32_t pad_;
} so_loop_opts;
typedef struct {
    int32_t query;            /* the query keyframe */
    int32_t id;               /* the candidate keyframe; -1 in unused slots (fewer than k eligible) */
    double distance;          /* in [0, 1] up to rounding; 1 without evidence */
    int32_t shift;            /* best column shift s */
    int32_t n_pairs;          /* column pairs that counted at that shift */
    double yaw;               /* s * 2 pi / sectors wrapped to (-pi, pi]: query heading - candidate heading (radians) */
} so_loop_candidate;
typedef struct {
    uint64_t n_described;     /* keyframes this call described (not found valid in the cache) */
    double time_describe_ms;  /* device time of the describe stage (CUDA events), 0 when nothing was described */
    double time_search_ms;    /* device time of the search and top-k stages (CUDA events) */
} so_loop_stats;
void so_loop_opts_defaults(so_loop_opts* opts);
/* For each of queries[0..n): its k best eligible keyframes, out[i * k .. i * k + k), by distance ascending, then id ascending.  Every
 * query is compared with every eligible keyframe at every shift.  stats may be NULL.  SO_ERR_ARG also for k outside 1..64. */
int so_loop_candidates(so_ctx* ctx, const int32_t* queries, size_t n, const so_loop_opts* opts, int32_t k, so_loop_candidate* out,
                       so_loop_stats* stats);
/* so_loop_candidates over the ids [id_begin, id_end) instead of the ids below q - exclude_recent: every keyframe of the range but the
 * query itself is eligible, wherever the range lies relative to the query (a later session's query searching an earlier session's
 * ids, imported before or after it started).  opts.exclude_recent is not used.  With the range [0, q - exclude_recent) the result is
 * bit-identical to so_loop_candidates for query q.  A range that holds no eligible keyframe leaves every slot unused (id -1).
 * SO_ERR_ARG, before any device work, as so_loop_candidates, and for id_begin < 0, id_end < id_begin or id_end past the keyframes
 * the store holds. */
int so_loop_candidates_range(so_ctx* ctx, const int32_t* queries, size_t n, const so_loop_opts* opts, int32_t id_begin, int32_t id_end,
                             int32_t k, so_loop_candidate* out, so_loop_stats* stats);
/* The descriptors of keyframes ids[0..n) as the search sees them, out[n][rings][sectors] (described first where the cache holds none). */
int so_keyframe_descriptors(so_ctx* ctx, const int32_t* ids, size_t n, const so_loop_opts* opts, float* out);

/* ---- pose graph: move the keyframes so that they agree with odometry and loop factors (sparse SE(3) least squares) -----------------
 * No reference counterpart.  The Ceres problem a pose graph is written as, solved by the trust-region rules of the registration's
 * solve (DESIGN.md section 3; "Pose graph" in section 4 states the definition in full):
 *   - nodes k = 0 .. n-1, pose7 values, one parameter block each with PoseLocalParameterization's Plus; node `fixed` held constant
 *     (it is not a parameter: norms, the gradient and the columns cover the free nodes only);
 *   - edge (i, j, z, S, c): r = S [t_E ; Log(R_E)] with E = Z^-1 X_i^-1 X_j, Log's angle in [0, pi]; S is a 6x6 square-root
 *     information matrix, row-major, order x, y, z, rx, ry, rz;
 *   - cost 1/2 sum rho(|r|^2): rho(s) = s for c = 0, Cauchy rho(s) = c^2 log(1 + s / c^2) for c > 0, through Ceres' corrector;
 *   - Jacobi scaling at iteration 0, LM diagonal [1e-6, 1e32], initial radius 1e4, tolerances 1e-10 (gradient), 1e-8 (parameter),
 *     1e-6 (function), termination codes as so_icp_result.iter_lm_termination.
 * Only the linear solve differs from Ceres' DENSE_QR: preconditioned conjugate gradients in FP64 with a block-tridiagonal
 * preconditioner over the node order (exact for a graph of consecutive edges alone).  Results are bit-identical run to run. */
typedef struct {
    int32_t i, j;             /* nodes of the edge, i != j */
    double z[7];              /* measured X_i^-1 X_j, pose7 */
    double sqrt_info[36];     /* S, row-major */
    double cauchy;            /* c: 0 for no loss, > 0 for CauchyLoss(c) with c*c finite and normal (1.5e-154 <= c <= 1.3e154) */
} so_pose_edge;
typedef struct {
    int32_t fixed;            /* the node held constant, default 0 */
    int32_t max_iterations;   /* trust-region iterations, default 50 (Ceres' default); 0 evaluates the start only */
} so_pose_graph_opts;
typedef struct {
    int32_t iterations, successful, unsuccessful, termination;   /* counted as Ceres counts them; termination codes as the registration's */
    uint64_t pcg_iterations;  /* conjugate-gradient iterations over all trust-region steps */
    double initial_cost, final_cost;
    double gmax;              /* max-norm of the gradient through Plus at the solution */
    double radius;            /* the trust-region radius the solve ends with */
    double time_ms;           /* device time of the solve (CUDA events) */
} so_pose_graph_result;
void so_pose_graph_opts_defaults(so_pose_graph_opts* opts);
/* Host-only: SO_ERR_ARG, with so_last_error naming the cause, for n_nodes < 2, an edge id out of range, i == j, a non-finite or
 * zero-norm z quaternion, a non-finite z or S, c < 0 or non-finite, fixed out of range, max_iterations < 0, and a graph in which some
 * node is not connected to `fixed`.  Duplicate edges are allowed. */
int so_pose_graph_check(size_t n_nodes, const so_pose_edge* edges, size_t n_edges, const so_pose_graph_opts* opts);
/* Solve from init7[n_nodes][7] (every pose finite with a non-zero quaternion; SO_ERR_ARG otherwise, and for every case of
 * so_pose_graph_check, before any device work).  out7[n_nodes][7] gets the solution (the fixed node as given) and may alias init7;
 * edge_weights (NULL or [n_edges]) gets each edge's rho' at it (1 without a loss).  opts NULL: the defaults.  result may be NULL. */
int so_pose_graph_solve(so_ctx* ctx, const double* init7, size_t n_nodes, const so_pose_edge* edges, size_t n_edges,
                        const so_pose_graph_opts* opts, double* out7, double* edge_weights, so_pose_graph_result* result);
/* The same problem with every node k where constant[k] != 0 held constant (Ceres' SetParameterBlockConstant on each): norms, the
 * gradient and the columns cover the free nodes only; opts->fixed is not used.  The multi-session merge holds an earlier session's
 * keyframes constant while a later one is joined to them.  A mask with exactly one node set gives results bit-identical to
 * so_pose_graph_solve with that node as `fixed`: poses, weights and every field of the result.  so_pose_graph_check_constant is
 * so_pose_graph_check with the fixed-node rules replaced by: constant not NULL, at least one constant node, at least one free node
 * unless max_iterations == 0, and every node connected to some constant node.  The solve fails with SO_ERR_ARG for every case of the
 * check, and for a non-finite init, before any device work.  Constant nodes come back as given (their quaternion normalised). */
int so_pose_graph_check_constant(size_t n_nodes, const so_pose_edge* edges, size_t n_edges, const uint8_t* constant,
                                 const so_pose_graph_opts* opts);
int so_pose_graph_solve_constant(so_ctx* ctx, const double* init7, size_t n_nodes, const so_pose_edge* edges, size_t n_edges,
                                 const uint8_t* constant, const so_pose_graph_opts* opts, double* out7, double* edge_weights,
                                 so_pose_graph_result* result);

/* ---- free-space clearing: take out the map points a scan sees through (moving objects) ---------------------------------------
 * No reference counterpart (LocalMap::addSurfPointCloud only adds points).  Off unless called; nothing else calls it.
 * Rule (DESIGN.md §2): the scan, in the frame of pose with the sensor at the pose's origin, is projected to a range image in FP64 --
 * column floor((az + pi) / az_res), az = atan2(y, x) in [-pi, pi), W = ceil(360 / az_res_deg) columns that wrap; row
 * floor((el - el_min) / el_res), el = atan2(z, hypot(x, y)), points with el outside [el_min, el_max) left out -- and each pixel keeps
 * the minimum float range of its finite points with r > 0.  A window map point m, at q = R^T (m - t) (FP64, quaternion normalised),
 * range r_m, is a candidate when min_range <= r_m <= max_range, its (2 dilate + 1)^2 pixel neighbourhood lies inside the elevation
 * span and every pixel of it has a return; it is removed when the neighbourhood minimum exceeds r_m + max(margin, margin_rel r_m).
 * Pixels without a return never remove anything, and a point behind something the scan saw is never removed.
 * Removal keeps the order of the points left (a block's k-NN tie-break and voxel-filter order) and rebuilds the index; when nothing
 * is removed the store is left bit for bit as it was.  With the block archive on only the window is carved. */
typedef struct {
    float az_res_deg, el_res_deg;   /* pixel size; el_res at least the sensor's beam spacing (VLP-16 2.0, OS1-128 0.4) */
    float el_min_deg, el_max_deg;   /* elevation span of the image */
    int32_t dilate;                 /* neighbourhood half-width in pixels, 0..4 (default 2: 5x5) */
    float margin, margin_rel;       /* metres, fraction of range */
    float min_range, max_range;     /* map points considered (sensor distance, metres) */
} so_free_space;
typedef struct {
    uint64_t n_image_points;        /* scan points that went into the range image */
    uint64_t n_pixels_hit;          /* pixels with a return */
    uint64_t n_candidates;          /* map points tested against a fully observed neighbourhood, over the stores carved */
    uint64_t n_removed;             /* map points removed, over the stores carved */
    uint64_t n_after[2];            /* points in the surf and the edge window afterwards */
} so_free_space_result;
/* The defaults: the OS1-128 image geometry (az_res 0.4, el_res 0.4, el span [-23, 23]), dilate 2, margin 0.3 m, margin_rel 0.02,
 * ranges [0.5, 60] m.  Set el_res and the span for the sensor at hand (VLP-16: el_res 2, span [-16, 16]). */
void so_free_space_defaults(so_free_space* opts);
/* Clear the map against a host cloud in the frame of pose (already motion-compensated if it needs it); stores: bit 0 surf, bit 1 edge.
 * One range image per call serves every store selected.  SO_ERR_ARG before any device work, both stores as they were: NULL opts or
 * pose, a pose that is not finite, a NULL cloud with n > 0, a resolution that is not finite or not positive, el_max <= el_min (or not
 * finite), W * H > 2^24, dilate outside 0..4, a negative or non-finite margin, min_range >= max_range, stores outside 1..3.
 * SO_ERR_CAPACITY: n > max_scan_points.  A pending origin or resolution change is applied first; an unbuilt store returns its error.
 * result may be NULL. */
int so_map_clear_free_space(so_ctx* ctx, int stores, const void* xyzi, size_t n, size_t stride_bytes, size_t intensity_offset,
                            const double pose[7], const so_free_space* opts, so_free_space_result* result);
/* The same against the surf cloud of the last single-scan registration, exactly as so_map_add_registered_scan(pose) would insert it
 * (compensated under APPROXIMATED / OPTIMIZED), without uploading it again: it is placed in the surf store's tail as the insert
 * places it.  The registration's record stays valid, so the insert can follow.  Fails as so_map_add_registered_scan does for a missing
 * or overwritten record (SO_ERR_ARG), and with SO_ERR_CAPACITY when the scan does not fit behind the surf window; SO_OK and nothing
 * removed before the first registration. */
int so_map_clear_free_space_registered(so_ctx* ctx, int stores, const double pose[7], const so_free_space* opts, so_free_space_result* result);
/* Clear dst's map against the surf clouds of src's keyframes ids[0..n_ids), keyframe ids[i] at poses7[i]: bit for bit what
 *   for i in 0 .. n_ids-1: so_map_clear_free_space(dst, stores, <so_keyframe_download(src, ids[i], 0, NULL)>, poses7 + 7 i, opts)
 * leaves -- the same points in both stores in the same order, the same index, the same n_removed -- with no host round trip.  One
 * keyframe's decision on a map point reads only its own image and that point, so a point goes when any keyframe saw clearly past it,
 * and each store that lost points is compacted once.  dst == src clears the map so_map_from_keyframes rebuilt, which brings back every
 * point the live clearing had removed; dst != src (same device) clears another map, e.g. a prior map loaded with so_map_set_points,
 * with a session's keyframes.  Duplicate ids are allowed.  Only the surf clouds are imaged; the window is carved, the block archive
 * is not; a pending origin or resolution change is applied first; with nothing removed the stores are left bit for bit.  The
 * keyframes are imaged in tiles of consecutive entries whose images fit 256 MiB (kFreeTileBytes, so_free_rule.h); the result does not
 * depend on the tiling.  A keyframe is tested against a 50 m block only when its sensor position can lie within max_range of the block.
 * SO_ERR_ARG before any device work, both stores as they were: every case of so_map_clear_free_space's options, stores outside 1..3,
 * contexts on different devices, src without a keyframe store, NULL ids or poses7 with n_ids > 0, an id src does not hold, a pose that
 * is not finite.  n_ids == 0 does nothing.  result may be NULL. */
typedef struct {
    uint64_t n_keyframes;           /* n_ids */
    uint64_t n_image_points;        /* keyframe points that went into the images: the sum of the per-keyframe calls' counts */
    uint64_t n_pixels_hit;          /* pixels with a return, summed over the keyframes' images */
    uint64_t n_candidates;          /* map points with a fully observed neighbourhood in at least one keyframe, over the stores carved */
    uint64_t n_removed;             /* map points removed, over the stores carved */
    uint64_t n_after[2];            /* points in the surf and the edge window afterwards */
    uint64_t n_tiles;               /* image tiles */
    double time_ms;                 /* device time of the call (CUDA events) */
} so_free_space_keyframes_result;
int so_map_clear_free_space_keyframes(so_ctx* dst, so_ctx* src, const int32_t* ids, size_t n_ids, const double* poses7, int stores,
                                      const so_free_space* opts, so_free_space_keyframes_result* result);

/* ---- loop verification: check a loop candidate before it becomes a pose-graph edge --------------------------------------------
 * No reference counterpart.  A Scan Context match (so_loop_candidates) is appearance only, and look-alike places match closely
 * (DESIGN.md §4, "Loop verification").  so_loop_verify builds each candidate's submap, aligns the query keyframe to it from the
 * candidate's prior and scores the alignment with two tests that look-alike places fail in different ways: overlap (the query's points
 * lie on the submap's surfaces) and visibility conflict (either side sees clearly through a surface the other one has).
 * so_loop_prior (host only): the alignment prior of a candidate from the current poses of the candidate (cand7) and the query
 * (query7) keyframes and its so_loop_candidate.yaw: the candidate's position, and the query's orientation turned about the world z
 * axis by psi_cand + yaw - psi_query (psi = atan2(R10, R00), as the descriptor levels a keyframe), i.e. the candidate's heading plus
 * yaw with the query's roll and pitch. */
void so_loop_prior(const double cand7[7], const double query7[7], double yaw, double out7[7]);
typedef struct {
    int32_t half_window;      /* the submap is the candidate's ids +- half_window, 0..8; default 2 */
    int32_t id_begin, id_end; /* the ids a submap may use: [id_begin, id_end) without the query; id_end < 0 (default -1): the ids
                                 below query - exclude_recent, as so_loop_candidates selects them.  A range is for sessions. */
    int32_t exclude_recent;   /* default 30 */
    so_icp_opts icp;          /* the alignment; default max_icp_iters 20, max_surface_features 0 (the whole keyframe), lm 4 */
    double inlier_dist;       /* metres: a query point is an inlier within this of the submap (d^2 <= float(inlier_dist^2)) */
    so_free_space image;      /* the sensor's range-image options of the conflict tests (default: so_free_space_defaults, OS1-128) */
    double min_overlap;       /* accepted only with overlap >= min_overlap */
    double max_conflict;      /* ... and both conflict fractions <= max_conflict */
} so_loop_verify_opts;
typedef struct {
    int32_t query, id;        /* the candidate as given */
    int32_t skipped;          /* 1: an unused slot (id -1); nothing ran and every other field is 0 */
    int32_t accepted;         /* 1: reg.status == 0, overlap >= min_overlap and both conflict fractions <= max_conflict */
    so_icp_result reg;        /* the query aligned to the submap from so_loop_prior */
    double rel7[7];           /* Z = X_id^-1 * reg.pose: the loop edge (id, query, Z) of so_pose_graph_solve */
    int32_t n_submap_keyframes, pad_;
    uint64_t n_submap_points; /* surf points of the submap (scratch's window) */
    uint64_t n_query_points;  /* finite surf points of the query keyframe */
    uint64_t n_inliers;       /* query points at reg.pose whose in-block nearest submap point lies within inlier_dist */
    double overlap;           /* n_inliers / n_query_points (0 without points) */
    double rmse;              /* sqrt(sum d^2 / n_inliers) over the inliers, metres (0 without inliers) */
    uint64_t n_cand_query, n_conflict_query;   /* query points a submap keyframe's image observes / sees clearly past */
    uint64_t n_cand_map, n_conflict_map;       /* submap points the query's image observes / sees clearly past */
    double conflict_query;    /* n_conflict_query / n_cand_query (0 without candidates) */
    double conflict_map;      /* n_conflict_map / n_cand_map (0 without candidates) */
    double time_ms;           /* device time of this candidate (CUDA events on scratch's stream) */
} so_loop_verify_result;
/* The defaults above; inlier_dist, min_overlap and max_conflict as measured in DESIGN.md §4, "Loop verification". */
void so_loop_verify_opts_defaults(so_loop_verify_opts* opts);
/* Verify candidates c[0..n) (as so_loop_candidates / so_loop_candidates_range return them) of ctx's keyframes into out[0..n), one
 * after another through the caller's scratch context (same device, not ctx), whose map is overwritten.  Per candidate (query q,
 * id c; X_k the current pose of keyframe k):
 *   1. submap ids: [c - w, c + w] intersected with the eligible ids, ascending; so_map_set_origin(scratch, X_c position), then
 *      so_map_from_keyframes(scratch, ctx, ids, their X, 1);
 *   2. so_register_keyframes(scratch, ctx, {q}, {so_loop_prior(X_c, X_q, c.yaw)}, &icp) -> reg: bit for bit this manual sequence;
 *   3. overlap: the query's surf points at reg.pose, transformed as so_keyframe_download(reg.pose) transforms them; an inlier is a
 *      finite point whose so_knn(k = 1, max_d2 = float(inlier_dist^2)) neighbour in scratch's surf store exists; sum d^2 in FP64 in
 *      a fixed order (identical run to run);
 *   4. conflicts, with the rule of so_map_clear_free_space: n_conflict_map / n_cand_map are n_removed / n_candidates of
 *      so_map_clear_free_space(scratch, 1, <query's sensor-frame surf cloud>, reg.pose, image), counted, nothing removed;
 *      n_conflict_query / n_cand_query are those of so_map_clear_free_space_keyframes(<a map of the finite points of step 3>, ctx,
 *      submap ids, their X, 1, image);
 *   5. accepted as so_loop_verify_result.accepted states.
 * Each result equals a call with that candidate alone.  Nothing of ctx changes: its map, keyframes, poses, descriptors and
 * registered scan.  A slot with id -1 comes back skipped with no device work.  SO_ERR_ARG before any device work: NULL arguments
 * (c and out may be NULL with n = 0), scratch == ctx, contexts on different devices, ctx without a keyframe store, a query or id
 * the store does not hold, id < -1, query == id, an id outside the eligible range, half_window outside 0..8, exclude_recent < 0,
 * id_end >= 0 with id_begin < 0, id_end < id_begin or id_end past the keyframes, icp options so_register_keyframes refuses,
 * inlier_dist not finite and positive, every case of so_map_clear_free_space's options, (2 half_window + 1) images over 256 MiB,
 * min_overlap or max_conflict outside [0, 1].  Errors of the steps above are returned as they come, with out[0..i) filled. */
int so_loop_verify(so_ctx* ctx, so_ctx* scratch, const so_loop_candidate* c, size_t n, const so_loop_verify_opts* opts,
                   so_loop_verify_result* out);

/* ---- scan pre-filter (the step right before the path; SURVEY 8f row 2) ------------------------------------------ */
/* replaces: laserMapping::adjustVoxelSize (src/LaserMapping/laserMapping.cpp:600-651) for the surf cloud: with
 * auto_voxel_size, pick config_.lineRes/planeRes from the scan statistics (mean|x| * mean|y| * mean|z| < 25 -> 0.1/0.2,
 * > 65 -> 0.4/0.8, else unchanged), then pcl::VoxelGrid(planeRes) on the sensor-frame cloud, then push the resolutions
 * into the map (slam.localMap.lineRes_/planeRes_ = config_, :648-649).  line_res/plane_res are in/out.  The VoxelGrid is PCL 1.12's
 * applyFilter for a cloud that is not dense: points with a non-finite x, y or z are skipped; the voxel index is taken relative to the
 * bounding box of the finite points (idx = i + j div_x + k div_x div_y, 32-bit); when that box spans more than INT32_MAX voxels
 * (dx dy dz, dx = int64((max_x - min_x) * (1/leaf)) + 1, float arithmetic) the cloud is returned verbatim, non-finite points included, as PCL does; one
 * centroid per voxel, float sums in cloud order.  Covered: |coordinate / leaf| < 2^20 - 1 on every axis (about 210 km at leaf 0.2);
 * beyond it PCL's conversions are undefined and the output is not specified (nothing is written past *n_out <= n).  Writes up to cap
 * packed float4 {x,y,z,intensity} points ordered by voxel index; *n_out = points produced. */
int so_scan_prefilter(so_ctx* ctx, const void* xyzi, size_t n, size_t stride_bytes, size_t intensity_offset, int auto_voxel_size,
                      float* line_res, float* plane_res, float* out_xyzi, size_t cap_points, size_t* n_out, double* average_distance);

/* replaces: featureExtraction::removePointDistortion<BufferType> (src/FeatureExtraction/featureExtraction.cpp:222-314).
 * points: n records of stride_bytes, float x,y,z first and the per-point float `time` (seconds after lidar_start_time,
 * point_os::PointcloudXYZITR: stride 32, time at byte 20) at time_offset; x,y,z are rewritten in place into the sensor frame
 * at lidar_start_time, non-finite points are left alone.  The pose buffer (MapRingBuffer::measMap_) is passed as n_samples
 * strictly ascending stamps + poses {tx,ty,tz,qx,qy,qz,qw}; interpolation = std::map::upper_bound, slerp + lerp, with the
 * `< 0.0001` rewind of :258-260.  imu_only != 0 is the Imu::Ptr instantiation: samples contribute rotation only and the motion
 * is conjugated by the IMU-lidar extrinsic T_i_l (parameter.cpp:192-193).  start_pose_out (optional) receives
 * {t_w_original_l, q_w_original_l} (:283-289).  *n_past_end (optional) counts points stamped after the last sample -- the
 * reference dereferences end() there and relies on synchronize_measurements (:187-196) to prevent it; the last interval is
 * extrapolated here. */
int so_scan_deskew(so_ctx* ctx, void* points, size_t n, size_t stride_bytes, size_t time_offset, double lidar_start_time,
                   const double* sample_times, const double* sample_poses, size_t n_samples, int imu_only, const double T_i_l[7],
                   double start_pose_out[7], size_t* n_past_end);
/* replaces: featureExtraction::uniformFeatureExtraction (featureExtraction.cpp:504-525): every skip_num-th point from index 1
 * that differs from its predecessor -- |dx| > 1e-7 || |dy| > 1e-7 || (|dz| > 1e-7 && x*x+y*y+z*z > block_range^2), with that
 * precedence -- is emitted as packed float4 {x, y, z, intensity = time}, input order.  int_abs != 0 evaluates the
 * unqualified abs() of :515-517 as ::abs(int) (its meaning when only <cmath> declared abs); 0 = the float overload.
 * *n_out = points produced (may exceed cap_points; only cap_points are written). */
int so_scan_extract_uniform(so_ctx* ctx, const void* points, size_t n, size_t stride_bytes, size_t time_offset, int skip_num,
                            float block_range, int int_abs, float* out_xyzi, size_t cap_points, size_t* n_out);
/* fills: the edgePoints cloud featureExtraction::extractFeatures publishes empty (featureExtraction.cpp:429-436), so that the line
 * branch of so_register gets real input.  LOAM edge selection (Zhang & Singh, RSS 2014, §V-A, as A-LOAM's scanRegistration, with
 * LOAM's occlusion and parallel-beam rejection; DESIGN.md §9 is the full definition), float32, each operation rounded on its own:
 *   - valid points: x, y, z, time finite and (x*x + y*y) + z*z > min_range^2; ordered by (ring, time, input index);
 *   - per ring of m points, 5 <= k <= m-6: curvature |sum of q_{k-5..k+5} except q_k, minus 10 q_k|^2;
 *   - excluded before selection: the occluded side of a gap (|q_{k+1}-q_k|^2 > 0.1, relative distance < 0.1) and points whose
 *     both neighbour gaps exceed 0.0002 |q_k|^2;
 *   - six sectors per ring (rings below 17 points give nothing); in each, curvature descending (ties by position), up to
 *     max_per_sector points with curvature > edge_threshold that are not excluded are accepted, each excluding itself and up to 5
 *     neighbours per side until a gap |dq|^2 > 0.05;
 *   - output: packed float4 {x, y, z, intensity = time} ordered by (ring, position); with voxel_leaf > 0 then pcl::VoxelGrid(voxel_leaf)
 *     on the sensor frame (laserMapping's corner filter at lineRes, laserMapping.cpp:635-640), bit-equal to so_scan_prefilter's filter
 *     (PCL's bounding-box index and verbatim fall-back included: a small leaf can return the edge cloud unfiltered).
 * points: n records of stride_bytes, float x, y, z at bytes 0, 4, 8, float time at time_offset, uint16 ring at ring_offset
 * (point_os::PointcloudXYZITR: stride 32, time at 20, ring at 24).  Does not touch the scan buffers: so_register_prefiltered and
 * so_map_add_registered_scan stay valid across this call.  *n_out = points produced (may exceed cap_points; only cap_points are
 * written).  SO_ERR_ARG before any device work: a NULL with n > 0, a stride that does not hold the fields, a time or ring overlapping
 * x, y, z or each other, a negative or non-finite option; SO_ERR_CAPACITY: n > max_scan_points.  opts may be NULL (all defaults). */
typedef struct {
    float min_range;          /* points at or inside this range are dropped (default 0: zero returns only) */
    float edge_threshold;     /* curvature a point must exceed (default 0.1) */
    float voxel_leaf;         /* > 0: pcl::VoxelGrid of the edge cloud at this leaf, as so_scan_prefilter's (default 0: off) */
    int32_t max_per_sector;   /* points accepted per sector (default 20, A-LOAM's less-sharp set) */
} so_edge_opts;
int so_scan_extract_edges(so_ctx* ctx, const void* points, size_t n, size_t stride_bytes, size_t time_offset, size_t ring_offset,
                          const so_edge_opts* opts, float* out_xyzi, size_t cap_points, size_t* n_out);

/* ---- registration (LidarSLAM) --------------------------------------------------------------------- */
/* replaces: LidarSLAM::Localization(true, predictodom, position, edge, planner, t) -> performLocalizationAndMapping
 * (LidarSlam.cpp:30-51,107-171), excluding the map insert at its end (call so_map_add_surf with the
 * transformed scan, as transformAndAddToMap does, LidarSlam.cpp:60-80).
 * edge cloud: processed by the edge / line branch (processEdgeFeatures, LidarSlam.cpp:310-321 -> ComputeLineDistanceParameters
 * :402-493, EdgeAnalyticCostFunction lidarOptimization.cpp:12-47) against the edge map; empty in the shipped pipeline
 * (featureExtraction.cpp:429-436), in which case the branch is idle exactly as upstream (LidarSlam.cpp:311). */
int so_register(so_ctx* ctx,
                const void* surf_xyzi, size_t n_surf, const void* edge_xyzi, size_t n_edge,
                size_t stride_bytes, size_t intensity_offset,
                const double pose_in[7], const so_icp_opts* opts, so_icp_result* out);

/* so_register of the cloud the LAST so_scan_prefilter call produced, which is still on the device (laserMapping.cpp:639-649 filters
 * the scan, :713-714 registers the filtered cloud): no download + second upload between the two steps.  The caller may pass
 * out_xyzi = NULL / cap = 0 to so_scan_prefilter when it does not need the filtered cloud on the host.  Fails with SO_ERR_ARG when
 * anything that reuses the scan buffers ran in between.  so_map_add_registered_scan afterwards inserts that same cloud. */
int so_register_prefiltered(so_ctx* ctx, const double pose_in[7], const so_icp_opts* opts, so_icp_result* out);

/* Batched replay against the frozen map (BASELINE cfg4): n_scans independent Localization() calls.
 * scans: n_scans consecutive clouds, scan s has n_points[s] points starting at point offset sum(n_points[0..s)).
 * poses_in: n_scans x 7.  results: n_scans structs.  n_scans <= so_config.max_batch. */
int so_register_batch(so_ctx* ctx, const void* surf_xyzi, const uint32_t* n_points, size_t n_scans,
                      size_t stride_bytes, size_t intensity_offset,
                      const double* poses_in, const so_icp_opts* opts, so_icp_result* results);
/* Same with an edge cloud per scan (the line branch of so_register, per scan): edge_xyzi holds the n_scans edge clouds back to
 * back, n_edge[s] points each (0 allowed); their total must fit so_config.max_scan_points.  Upstream the edge cloud is empty
 * (featureExtraction.cpp:429-436), so this is the batched form of a dormant branch (SURVEY 8a a19) -- complete, not tuned. */
int so_register_batch_edges(so_ctx* ctx, const void* surf_xyzi, const uint32_t* n_points, const void* edge_xyzi, const uint32_t* n_edge,
                            size_t n_scans, size_t stride_bytes, size_t intensity_offset,
                            const double* poses_in, const so_icp_opts* opts, so_icp_result* results);
/* Same, inputs already resident in device memory: packed float4 points (d_scans_xyzi), host n_points / poses.
 * Used for the device-resident throughput figure; results are still copied back to host structs. */
int so_register_batch_device(so_ctx* ctx, const void* d_scans_xyzi, const uint32_t* n_points, size_t n_scans,
                             const double* poses_in, const so_icp_opts* opts, so_icp_result* results);
/* Keyframes ids[0..n) of src (surf clouds; see so_keyframe_add_registered) registered against dst's map from priors7[n][7], read on the
 * device as so_register_batch_device reads device scans: mode NONE (a keyframe is already compensated), the map does not shift, dst's
 * registered scan is untouched and a pose sink gets n rows.  results[i].pose and .cov give a loop factor.  dst and src may be the same
 * context.  SO_ERR_ARG for contexts on different devices or an id src does not hold; SO_ERR_CAPACITY as so_register_batch_device. */
int so_register_keyframes(so_ctx* dst, so_ctx* src, const int32_t* ids, size_t n, const double* priors7, const so_icp_opts* opts,
                          so_icp_result* results);

/* ---- within-scan motion compensation (LidarSlam.h:65-82 UndistortionMode; empty upstream, LidarSlam.cpp:382-400) ------------
 * A constant body-velocity model, re-estimated at the start of every ICP iteration from the current estimate T_cur:
 *   D = T_prev^-1 * T_cur,  alpha_i = double(time_i) / dt (0 for a non-finite time),  q_i = slerp(identity, q_D, alpha_i),
 *   pInit_i = float3(qrot(q_i, p_i) + alpha_i * t_D)
 * and the iteration runs on pInit (rounded to float) in place of the sensor-frame point.  time_i is the float at byte time_offset of
 * each record, in seconds after the instant the pose describes (the shipped pipeline: the scan start, time stored in intensity by
 * uniformFeatureExtraction, so time_offset == intensity_offset).  Surf cloud only (so_register_undistort_edges adds the edge
 * cloud).  Argument errors (mode 2, a bad dt, a
 * non-finite prev_pose) are returned before any device work.  After so_register_undistort / so_register_prefiltered_undistort,
 * so_map_add_registered_scan(pose) inserts the whole cloud undistorted with the D that pose gives: world = T(pose) * pInit. */
typedef struct {
    int32_t mode;          /* 0 NONE (the scan registers exactly as so_register), 1 APPROXIMATED; 2 (OPTIMIZED) -> SO_ERR_ARG:
                              OPTIMIZED estimates a second pose, see so_register_optimized */
    int32_t rotation;      /* 1 rotation + translation, 0 translation only (cloud already rotation-deskewed by so_scan_deskew imu_only) */
    double prev_pose[7];   /* previous registration's pose7 */
    double dt;             /* seconds from prev_pose to the pose being estimated, finite and > 0 */
} so_undistort;
int so_register_undistort(so_ctx* ctx, const void* surf_xyzi, size_t n, size_t stride_bytes, size_t intensity_offset, size_t time_offset,
                          const double pose_in[7], const so_undistort* u, const so_icp_opts* opts, so_icp_result* out);
/* ... with an edge cloud for the line branch (so_register's edge_xyzi): every ICP iteration warps the edge cloud with the same D as
 * the surf cloud, and the line fit and evaluation run on its pInit (rounded to float) in place of the sensor-frame edge points.  Both
 * clouds share stride, intensity offset and time offset (so_scan_extract_uniform and so_scan_extract_edges both store the time in
 * intensity).  n_edge == 0: exactly so_register_undistort; mode 0: exactly so_register with the edge cloud.  Argument errors (those of
 * so_register_undistort, a NULL edge_xyzi with n_edge > 0; SO_ERR_CAPACITY for n_edge > max_scan_points) come before any device
 * work.  so_map_add_registered_edges(pose) afterwards inserts the edge cloud undistorted at pose. */
int so_register_undistort_edges(so_ctx* ctx, const void* surf_xyzi, size_t n_surf, const void* edge_xyzi, size_t n_edge, size_t stride_bytes,
                                size_t intensity_offset, size_t time_offset, const double pose_in[7], const so_undistort* u,
                                const so_icp_opts* opts, so_icp_result* out);
/* ... of the cloud the last so_scan_prefilter left on the device; the time is the filtered cloud's intensity (w). */
int so_register_prefiltered_undistort(so_ctx* ctx, const double pose_in[7], const so_undistort* u, const so_icp_opts* opts, so_icp_result* out);
/* ... of a batch as so_register_batch, u[n_scans]: one so_undistort per scan (mode 0 and 1 may be mixed). */
int so_register_batch_undistort(so_ctx* ctx, const void* surf_xyzi, const uint32_t* n_points, size_t n_scans, size_t stride_bytes,
                                size_t intensity_offset, size_t time_offset, const double* poses_in, const so_undistort* u,
                                const so_icp_opts* opts, so_icp_result* results);
/* Stage hook: pInit of a cloud at T_cur = pose, as packed float4 {x, y, z, intensity} in input order (mode 0: the cloud as is). */
int so_undistort_points(so_ctx* ctx, const void* xyzi, size_t n, size_t stride_bytes, size_t intensity_offset, size_t time_offset,
                        const double pose[7], const so_undistort* u, float* out_xyzi);

/* ---- within-scan motion estimated by the registration (LidarSlam.h:77-81 UndistortionMode::OPTIMIZED; empty upstream) ---------
 * Two pose7 unknowns per scan: T, the pose at time 0 (what every registration estimates), and D, the motion over dt, so that the
 * pose at time dt is T * D.  With alpha_i = double(time_i) / dt (0 for a non-finite time) the solve's point is
 *   u_i(D) = qrot(slerp(identity, q_D, alpha_i), p_i) + alpha_i * t_D
 * and its rows are so_register's plane rows at T on u_i(D), plus six rows of SE3AbsolutatePoseFactor on D (measurement
 * motion_prior, row k multiplied by sqrt(n_ok * motion_info[k]), n_ok the accepted correspondences of the ICP iteration).  Every ICP
 * iteration searches and fits at T on float(u(D)) at the current D.  Surf cloud only (so_register_optimized_edges adds the edge
 * cloud); use_pose_prior must be 0.  Argument errors (a
 * bad dt, a non-finite motion_prior or one with a zero quaternion, a negative or non-finite motion_info, use_pose_prior) are returned
 * before any device work.  icp.cov and the error fields describe T.  After so_register_optimized /
 * so_register_prefiltered_optimized, so_map_add_registered_scan(pose) inserts T(pose) * u_i(D_opt) for the whole cloud. */
typedef struct {
    double dt;               /* seconds the motion spans, finite and > 0 */
    double motion_prior[7];  /* D0, e.g. T_prev^-1 * pose_in; identity {0,0,0, 0,0,0,1} when unknown */
    double motion_info[6];   /* information of D0 per accepted correspondence (translation xyz, rotation xyz), >= 0 */
} so_motion;
typedef struct {
    so_icp_result icp;       /* icp.pose_opt = T */
    double motion[7];        /* D */
    double pose_end[7];      /* T * D, the pose at time dt */
} so_motion_result;
int so_register_optimized(so_ctx* ctx, const void* surf_xyzi, size_t n, size_t stride_bytes, size_t intensity_offset, size_t time_offset,
                          const double pose_in[7], const so_motion* m, const so_icp_opts* opts, so_motion_result* out);
/* ... with an edge cloud for the line branch: every ICP iteration searches and fits the edge cloud at T on float(u_e(D)), and its line
 * rows join the solve over the 12 columns: r = (lp - a) x (lp - b) / |a - b| with lp = R(q) u(D) + t (EdgeAnalyticCostFunction),
 * under ScaledLoss(TukeyLoss(sqrt(3 lineRes))).  The motion prior's multiplier counts accepted planes plus accepted lines;
 * icp.iter_n_edge and icp.hist_reject_line are filled; a NaN-weighted line row ends the registration with
 * SO_STATUS_INVALID_EVALUATION, as in so_register.  Both clouds share stride, intensity offset and time offset.  n_edge == 0: exactly
 * so_register_optimized.  Argument errors (those of so_register_optimized, a NULL edge_xyzi with n_edge > 0; SO_ERR_CAPACITY for
 * n_edge > max_scan_points) come before any device work.  so_map_add_registered_edges(pose) afterwards inserts
 * T(pose) * u_e(D_opt). */
int so_register_optimized_edges(so_ctx* ctx, const void* surf_xyzi, size_t n_surf, const void* edge_xyzi, size_t n_edge, size_t stride_bytes,
                                size_t intensity_offset, size_t time_offset, const double pose_in[7], const so_motion* m,
                                const so_icp_opts* opts, so_motion_result* out);
/* ... of the cloud the last so_scan_prefilter left on the device; the time is the filtered cloud's intensity (w). */
int so_register_prefiltered_optimized(so_ctx* ctx, const double pose_in[7], const so_motion* m, const so_icp_opts* opts, so_motion_result* out);
/* ... of a batch as so_register_batch, m[n_scans]: one so_motion per scan. */
int so_register_batch_optimized(so_ctx* ctx, const void* surf_xyzi, const uint32_t* n_points, size_t n_scans, size_t stride_bytes,
                                size_t intensity_offset, size_t time_offset, const double* poses_in, const so_motion* m,
                                const so_icp_opts* opts, so_motion_result* results);
/* Stage hook: the correspondences at T = pose for float(u(motion)), then the plane rows' normal equations at (T, motion) over the
 * 12 tangent columns (T's translation, rotation, D's translation, rotation): H (row-major 12x12), g, cost; prior rows excluded. */
int so_evaluate_optimized(so_ctx* ctx, const void* xyzi, size_t n, size_t stride_bytes, size_t intensity_offset, size_t time_offset,
                          const double pose[7], const double motion[7], double dt, int32_t max_surface_features, double H[144],
                          double g[12], double* cost);
/* Stage hook: the same with the edge cloud's line rows added (its lines fitted at T on float(u_e(motion))). */
int so_evaluate_optimized_edges(so_ctx* ctx, const void* xyzi, size_t n, const void* edge_xyzi, size_t n_edge, size_t stride_bytes,
                                size_t intensity_offset, size_t time_offset, const double pose[7], const double motion[7], double dt,
                                int32_t max_surface_features, double H[144], double g[12], double* cost);

/* ---- degeneracy-aware registration (the reference's isDegenerate, LidarSlam.h:264; its rule is commented out upstream) -----------
 * Once per ICP iteration, at the start of its solve, the 6x6 normal matrix H at the iteration's start pose (plane rows, line rows,
 * pose-prior rows when use_pose_prior is set; order t, theta) is analysed block by block:
 *   I_t = H_tt - H_tr H_rr^+ H_rt,   I_theta = H_rr - H_rt H_tt^+ H_tr
 * (^+ the pseudo-inverse with ceres::Covariance's cut, sqrt(w_k / w_max) < 1e-7).  These are the inverses of the covariance blocks
 * EstimateRegistrationError analyses, so sqrt(i_min / i_max) of I_t is PosInverseConditionNum when H is invertible (and likewise for
 * theta).  Eigenpair (i_k, u_k) of a block, ascending, is flagged when i_k <= threshold^2 * max(i_max, 0).  constrain = 1 and
 * something flagged: that iteration's solve is Ceres' trust-region solve on the same cost with the local parameterisation
 * x [+] B y, B = the unflagged eigenvectors (6 x m, translation ones first), so the pose does not move along a flagged direction.
 * Otherwise the registration is so_register's, bit for bit.  Combining it with undistortion (so_register_undistort*,
 * so_register_optimized*) is not supported.  Argument errors (a NaN or negative threshold, a threshold >= 1, constrain not 0 or 1) come
 * before any device work.  so_map_add_registered_scan / so_map_add_registered_edges work afterwards as after so_register. */
typedef struct {
    double pos_threshold, ori_threshold;   /* on sqrt(i_k / i_max), each in [0, 1) */
    int32_t constrain;                     /* 0: report only (the registration is so_register's, bit for bit); 1: reduced solve */
    int32_t pad_;
} so_degeneracy;
typedef struct {
    so_icp_result icp;
    int32_t iter_n_flag_pos[SO_MAX_ICP_ITERS], iter_n_flag_ori[SO_MAX_ICP_ITERS];   /* directions flagged per ICP iteration */
    double pos_info[3], pos_axes[9], ori_info[3], ori_axes[9];   /* last ICP iteration: eigenpairs of I_t, I_theta, ascending;
                                                                    axes[3k..3k+2] = eigenvector k */
    int32_t flags_pos, flags_ori;                                 /* bit k: eigenvector k flagged, last ICP iteration */
} so_degeneracy_result;
int so_register_degeneracy(so_ctx* ctx, const void* surf_xyzi, size_t n_surf, const void* edge_xyzi, size_t n_edge, size_t stride_bytes,
                           size_t intensity_offset, const double pose_in[7], const so_degeneracy* d, const so_icp_opts* opts,
                           so_degeneracy_result* out);
/* ... of a batch as so_register_batch (edge_xyzi / n_edge: optional, as so_register_batch_edges), d[n_scans]: one per scan. */
int so_register_batch_degeneracy(so_ctx* ctx, const void* surf_xyzi, const uint32_t* n_points, const void* edge_xyzi, const uint32_t* n_edge,
                                 size_t n_scans, size_t stride_bytes, size_t intensity_offset, const double* poses_in, const so_degeneracy* d,
                                 const so_icp_opts* opts, so_degeneracy_result* results);
/* Test hook: the analysis above on a given symmetric H (row-major 6x6, upper triangle read), by the device code a solve begins with,
 * in a one-thread launch.  Fills pos_info, pos_axes, ori_info, ori_axes and the flags; zeroes the rest.  Replaces the state a
 * preceding so_correspond* left for so_evaluate. */
int so_degeneracy_analysis(so_ctx* ctx, const double* H, const so_degeneracy* d, so_degeneracy_result* out);

/* Test hook: one ICP iteration's solve (Ceres' trust-region LM, LidarSlam.cpp:213-240) on caller-given correspondences, for a batch of
 * n_problems problems, by the device code and the launch sequence a registration of n_problems scans runs -- the fused evaluation +
 * step kernel for one or two problems (unless SO_NO_FUSED_LM is set), evaluation + step kernels otherwise, the degeneracy-aware step
 * kernel when d is given -- without the neighbour search and the plane fit.  The rows of problem b follow those of problem b - 1 in
 * `rows`; every row counts as an accepted plane correspondence (also with w = 0: it then adds nothing but counts towards the prior's
 * information, as features_corres.size() does).  The registration's plane_res sets the Tukey loss.  n_rows <= so_config.max_scan_points,
 * n_problems <= max_batch.  d: NULL or one so_degeneracy per problem.  Replaces the state a preceding so_correspond* left for
 * so_evaluate and the scan buffer so_ordered_scans reads. */
typedef struct {
    float p[3];                /* scan point, sensor frame */
    float pad_;
    double n[3], d, w;         /* plane n.x + d = 0 and its residualCoefficient */
} so_solve_row;
typedef struct {
    uint32_t n_rows;
    int32_t lm_max_iterations; /* <= 0: 4; at most 16 */
    double pose[7];            /* start of the solve */
    int32_t use_pose_prior;    /* SE3 prior rows (addAbsolutePoseConstraints) with measurement x0 */
    float visual_confidence_factor, prior_uncertainty[3];
    int32_t pad_;
    double x0[7];
} so_solve_problem;
typedef struct {
    double pose[7];
    double initial_cost, final_cost;
    int32_t lm_iterations, successful, unsuccessful, termination;   /* termination: as so_icp_result.iter_lm_termination */
    double radius, decrease_factor, gmax;                           /* the trust-region state the solve ended in */
    int32_t n_flag_pos, n_flag_ori;                                 /* flagged directions (degeneracy-aware solves) */
    int32_t status, pad_;                                           /* so_icp_result.status */
} so_solve_result;
int so_solve(so_ctx* ctx, const so_solve_row* rows, const so_solve_problem* problems, size_t n_problems, const so_degeneracy* d,
             so_solve_result* out);
/* Test hook: the same for the two-block solve of so_register_optimized (T and the motion D over 12 tangent columns), by its kernels
 * (k_motion_eval + k_motion_step) launched as one ICP iteration of a registration of n_problems scans launches them, without the warp,
 * the neighbour search and the plane fit.  times[i] is the time of row i (alpha = time / dt, 0 when not finite); n_rows * info_k sets
 * the motion prior's rows.  The solve runs with max_icp_iters = 1, so it ends with the covariance: cov is T's 6x6 block of the 12x12
 * pseudo-inverse.  An empty problem ends with termination 6 and SO_STATUS_NO_CORRESPONDENCES.  Argument errors (those of so_solve,
 * those of so_register_optimized's so_motion, a NULL times with rows) come before any device work.  Replaces the state a preceding
 * so_correspond* left for so_evaluate, the scan buffer so_ordered_scans reads, and the scan and times so_map_add_registered_scan
 * inserts, which then refuses until the next registration. */
typedef struct {
    uint32_t n_rows;
    int32_t lm_max_iterations; /* <= 0: 4; at most 16 */
    double pose[7];            /* T at the start */
    double motion[7];          /* D at the start (its quaternion normalised); the prior's measurement is m.motion_prior */
    so_motion m;
} so_solve_optimized_problem;
typedef struct {
    so_solve_result solve;     /* pose = T; radius, decrease factor and gmax of the 12-column loop */
    double motion[7];          /* D */
    double cov[36];            /* T's block of the covariance (so_icp_result.cov) */
} so_solve_optimized_result;
int so_solve_optimized(so_ctx* ctx, const so_solve_row* rows, const float* times, const so_solve_optimized_problem* problems,
                       size_t n_problems, so_solve_optimized_result* out);

/* Sharded-replay plumbing (BASELINE cfg4; SURVEY 8e "K8"): a caller-owned DEVICE buffer of cap_rows x 8 doubles.  Every following
 * so_register / so_register_batch* call appends one row per scan, starting at first_row and advancing: {pose_opt[7] (the
 * optimiser output, so_icp_result.pose_opt), status + 256 * n_iterations}; scans that were not registered (soft statuses) carry
 * their prior.  The rows are written by a kernel on the context stream right after the last optimiser step, so a collective
 * enqueued on that stream (ncclAllGather / torch.distributed.all_gather_into_tensor) gathers the poses of a whole replay without
 * a host round trip.  d_rows == NULL detaches the sink.  The reference has no counterpart (single process, one scan at a time). */
int so_set_pose_sink(so_ctx* ctx, void* d_rows, size_t cap_rows, size_t first_row);

/* Test hook: so_register (surf cloud only) with the neighbour SEARCH replaced by caller-supplied neighbour sets --
 * nn_ids[it][i][0..4] = the five map point ids (so_map_set_points order, ascending distance; 0xFFFFFFFF = no result) that
 * findNearestNeighbors (LidarSlam.cpp:720-747) returned for scan point i in ICP iteration it, n_trace_iters iterations of them.
 * Everything after the search (the 3*planeRes gate on the 5th distance, PCA, plane fit, solve, covariance) runs as in
 * so_register.  Feeding the neighbour sets of the reference's own octree (flann/octree.h:1004-1055, compiled verbatim in
 * oracle/_ref) proves that exactness of the k-NN is the only deviation of this library from the reference path. */
int so_register_injected(so_ctx* ctx, const void* surf_xyzi, size_t n_surf, size_t stride_bytes, size_t intensity_offset,
                         const double pose_in[7], const so_icp_opts* opts, const uint32_t* nn_ids, int32_t n_trace_iters,
                         so_icp_result* out);

/* Stage-level entry points used by the parity tests (same kernels as so_register). */
/* processPlannerFeatures at a fixed pose (LidarSlam.cpp:323-344): fills corr[n], hist_obs[9], hist_rej[7]. */
int so_correspond(so_ctx* ctx, const void* surf_xyzi, size_t n, size_t stride_bytes, size_t intensity_offset,
                  const double pose[7], int32_t max_surface_features, so_corr* corr, int32_t hist_obs[9], int32_t hist_rej[7]);
/* Test hook: the correspondences of ICP iteration 1 -- the search that takes its bound from the previous iteration's neighbours.
 * The scan is ordered at pose_prev, as a registration starting there orders it; iteration 0's search and fit run at pose_prev
 * unreported; then iteration 1's search and fit run at `pose` on the neighbour records iteration 0 left, and fill corr[n],
 * hist_obs[9] and hist_rej[7] as so_correspond does.  The seed only prunes: the result equals so_correspond at `pose`.  so_evaluate
 * then uses iteration 1's correspondences.  Argument errors and side effects are those of so_correspond. */
int so_correspond_seeded(so_ctx* ctx, const void* surf_xyzi, size_t n, size_t stride_bytes, size_t intensity_offset,
                         const double pose[7], int32_t max_surface_features, so_corr* corr, int32_t hist_obs[9], int32_t hist_rej[7],
                         const double pose_prev[7]);
/* Test hook: the first n points of the cell-ordered scan buffer the kernels read, as the last registration left it: packed float4
 * {x, y, z, w} per point, scans at their batch offsets, w = the point's index inside its scan (uint32 bit pattern).  Meaningful after
 * a so_register_batch* call of mode 0 (modes 1 and 2 rewrite x, y, z every ICP iteration); n <= so_config.max_scan_points * max_batch. */
int so_ordered_scans(so_ctx* ctx, float* out_xyzw, size_t n);
/* processEdgeFeatures at a fixed pose (LidarSlam.cpp:310-321): fills corr[n], hist_rej_line[7]. */
int so_correspond_edge(so_ctx* ctx, const void* edge_xyzi, size_t n, size_t stride_bytes, size_t intensity_offset, const double pose[7],
                       so_edge_corr* corr, int32_t hist_rej_line[7]);
/* Robustified normal equations at `pose` over the correspondences of the last so_correspond call:
 * H = sum rho' J^T J (row-major 6x6), g = sum rho' J^T r, cost = 1/2 sum rho (lidarOptimization.cpp:55-80 + Ceres corrector). */
int so_evaluate(so_ctx* ctx, const double pose[7], double H[36], double g[6], double* cost);
/* Test hook: the end of a registration on a given normal matrix -- ceres::Covariance's pseudo-inverse (directions with
 * sqrt(w_i / w_max) < 1e-7 cut, and every smaller one with them) and EstimateRegistrationError's 3x3 analyses (LidarSlam.cpp:854-884),
 * by the device code a registration ends with, in a one-CTA launch.  H: symmetric n x n, row-major, upper triangle read; n = 6
 * (so_register*) or 12 (so_register_optimized*: T's columns first, T's 6x6 block reported).  Fills out->cov, pos_err, pos_dir,
 * pos_inv_cond, ori_err_deg, ori_dir, ori_inv_cond and zeroes the rest.  Replaces the state a preceding so_correspond* left for
 * so_evaluate. */
int so_covariance(so_ctx* ctx, const double* H, int32_t n, so_icp_result* out);

/* ---- neighbour search (LocalMap::nearestKSearchSurf, LocalMap.h:481-525) --------------------------- */
/* k nearest map points IN THE QUERY'S OWN 50 m BLOCK for nq world-frame queries (packed xyz floats, 12 B stride or
 * given stride).  max_d2 > 0: radius-bounded (neighbours with d2 > max_d2 are not returned); max_d2 <= 0: exact,
 * unbounded.  idx = map point id or 0xFFFFFFFF, d2 = squared distance with the reference's rounding
 * (flann/octree.h:95-102).  Ordering: ascending (d2, id).  1 <= k <= 8.
 * so_knn_device takes device pointers for all three arrays (float4 queries). */
int so_knn(so_ctx* ctx, const float* q_xyz, size_t nq, size_t stride_bytes, int k, float max_d2, uint32_t* idx, float* d2);
int so_knn_device(so_ctx* ctx, const void* d_q_xyzw, size_t nq, int k, float max_d2, uint32_t* d_idx, float* d_d2);

/* ---- feature sampling (calculateSamplingRate + shouldProcessPoint, LidarSlam.cpp:346-359) ---------- */
/* The indices of an n-point scan that a registration capped at max_surface_features processes (ascending; all of 0..n-1 when
 * the cap is <= 0 or >= n).  Host-only (needs no device): this is the list so_register uses to upload the processed points of a
 * capped scan ahead of the rest of the cloud.  Writes min(count, cap) indices to out (may be NULL with cap 0) and the count to
 * *n_out.  Returns SO_OK or SO_ERR_ARG. */
int so_sampling_indices(uint32_t n, int32_t max_surface_features, uint32_t* out, size_t cap, size_t* n_out);

/* ---- global localization against the prior map ------------------------------------------------------------------ */
/* extends: localization mode (laserMapping.cpp:163-173 loads the prior map, :306-313 takes the start pose from init_x ... init_yaw
 * unchanged).  Instead of an exact start pose, search a region around a rough centre: every x/y/z voxel shift and yaw step of the
 * scan is a hypothesis, scored against an occupancy bitmap of the surf map; the best hypotheses, found by branch-and-bound (below),
 * are registered with the ordinary ICP path after non-maximum suppression, and the registration with the most accepted plane
 * correspondences wins.  Roll and pitch are taken
 * from the centre (IMU gravity, as initializeFirstFrame does, laserMapping.cpp:281-298).  Zero fields take the defaults shown. */
typedef struct {
    double half_x, half_y, half_z;  /* search half-extents (m) around the centre; 0 = that axis is not searched */
    double yaw_half;                /* yaw half-range (rad) around the centre's yaw; >= pi = the full circle */
    double res;                     /* voxel edge of the bitmap and translation step (m), default 0.25 */
    double yaw_step;                /* yaw step (rad), default 2 deg */
    double max_range;               /* scan points farther than this are not scored (m), default 40 */
    int32_t score_points;           /* scan points scored (shouldProcessPoint decimation), default 1024, at most 4096 */
    int32_t dilate;                 /* bitmap dilation (voxels, cube neighbourhood), default 1, at most 8 */
    int32_t k;                      /* candidates refined, default 16, at most 64 */
    int32_t whole_map;              /* 0: search and refine in the window; 1: the window plus the surf archive (see below); else SO_ERR_ARG */
    double nms_xy;                  /* suppression radius in x/y (m), default 1.0 */
    double nms_yaw;                 /* suppression half-width in yaw (rad), default 10 deg */
} so_global_opts;

/* One refined candidate, in rank order (score descending, hypothesis index ascending). */
typedef struct {
    double prior[7];        /* hypothesis pose the registration started from */
    int32_t score;          /* occupied bitmap cells hit by the score points */
    int32_t n_success;      /* SO_MATCH_SUCCESS correspondences of the final ICP iteration */
    double cost;            /* final cost of the last ICP iteration */
    double pose[7];         /* so_icp_result.pose of its registration */
    int32_t status;         /* so_icp_result.status */
    int32_t pad_;
} so_global_candidate;

typedef struct {
    double pose[7];         /* the winner's refined pose; the centre when status != SO_OK */
    int32_t status;         /* SO_OK / SO_STATUS_NO_CORRESPONDENCES / SO_STATUS_NOT_ENOUGH_FEATURES */
    int32_t winner;         /* index into the candidate list, -1 when none */
    int32_t n_candidates;   /* candidates kept by the suppression and registered */
    int32_t best_score;     /* score of the best hypothesis */
    uint64_t n_hypotheses;  /* NX * NY * NZ * NYAW */
    int32_t n_score_points; /* scan points scored */
    int32_t n_windows;      /* whole_map = 1 with the archive on: distinct windows the candidates were registered in; else 0 */
    double time_raster_ms;  /* device time (CUDA events) of the map bounds and the raster, */
    double time_dilate_ms;  /* of the dilation, pyramid levels and offset table, */
    double time_score_ms;   /* of the branch-and-bound traversal; */
    double time_sort_ms;    /* 0 (the traversal yields the keys in order) */
    double time_refine_ms;  /* candidate read-back, suppression and registrations (host clock) */
    double time_total_ms;   /* whole call (host clock) */
    so_icp_result icp;      /* the winner's registration (zeroed when there is none) */
} so_global_result;

/* Global localization of a sensor-frame surf cloud (layout as so_register) around center_pose7.  Writes up to cap candidates to
 * cands (may be NULL with cap 0).  The map is not modified and not shifted, an attached pose sink gets no rows; afterwards
 * so_map_add_registered_scan inserts this cloud.  Returns SO_OK, a soft status, or an error.  Before any device work: argument
 * errors; SO_ERR_CAPACITY above 2^24 hypotheses, a whole-box bitmap ((NX + 2e) * (NY + 2e) * (NZ + 2e) voxels, e =
 * ceil(max_range / res), rows padded to 32 bits) above 2^32 bits, a cloud above max_scan_points, or an offset table (NYAW * score
 * points * 16 B) above 1 GiB, i.e. NYAW * score points > 2^26 (yaw steps finer than about 0.02 deg at 4096 points).  After the
 * map bounds: SO_ERR_CAPACITY for a pyramid level above 2^32 bits, which takes a box near the bitmap limit with a map filling it. */
int so_localize_global(so_ctx* ctx, const void* xyzi, size_t n, size_t stride_bytes, size_t intensity_offset, const double center_pose7[7],
                       const so_global_opts* gopts, const so_icp_opts* opts, so_global_candidate* cands, size_t cap,
                       so_global_result* out);
/* Stage hook of so_localize_global: the uint16 score of every hypothesis, index ((yaw * NZ + z) * NY + y) * NX + x, and
 * dims = {NX, NY, NZ, NYAW}: level 0 of the pyramid scored densely, with no pruning.  Needs cap >= the hypothesis count
 * (SO_ERR_CAPACITY before any device work); *n_score_points (optional) receives the points scored.  Other errors as
 * so_localize_global. */
int so_localize_scores(so_ctx* ctx, const void* xyzi, size_t n, size_t stride_bytes, size_t intensity_offset, const double center_pose7[7],
                       const so_global_opts* gopts, uint16_t* scores, size_t cap, int32_t dims[4], int32_t* n_score_points);
/* Host-only (needs no device): the argument checks of so_localize_global's options, dims = {NX, NY, NZ, NYAW}, the hypothesis
 * count, and the bytes of an occupancy bitmap over the whole search box, the quantity so_localize_global's bitmap limit bounds
 * (2^32 bits = 512 MiB; the search itself allocates only the pyramid clipped to the map).  Returns SO_OK, SO_ERR_ARG or
 * SO_ERR_CAPACITY for the hypothesis and bitmap limits (dims and counts are filled for the capacity error too). */
int so_localize_global_size(const so_global_opts* gopts, int32_t dims[4], uint64_t* n_hypotheses, uint64_t* bitmap_bytes);

/* ---- the search: exact branch-and-bound ------------------------------------------------------------------------------------ */
/* Every so_localize_global* call finds the sorted key prefix (the best hypotheses, score descending, index ascending) by
 * branch-and-bound over an occupancy pyramid instead of scoring every hypothesis.  Its memory scales with the map, not with the
 * search region.  so_localize_global_bnb is so_localize_global with the limits this allows: up to 2^32 hypotheses, no bitmap
 * limit, so a region may cover a whole prior map (so_map_bounds gives the extent); within so_localize_global's limits the two
 * return the same result bit for bit (every field but the time_* ones, and the candidate list).  Level L of the pyramid is
 * B_L(x, y, z) = OR over a, b in [0, 2^L) of B(x+a, y+b, z); the bound of a level-L node (yaw m, z shift k, x/y shifts
 * [i0, i0+2^L) x [j0, j0+2^L)) is U = sum over score points of B_L at the point's voxel shifted by (i0, j0), at least the score of
 * every hypothesis in the node. */
#define SO_BNB_LEVELS 32
typedef struct {
    int32_t lmax;                           /* coarsest level: the smallest L >= 1 whose root fits 65 536 nodes (DESIGN.md §4) */
    int32_t kstar_score;                    /* score of the last key of the prefix (the final K*) */
    uint64_t root_nodes;                    /* NYAW * NZ * ceil(NX / 2^lmax) * ceil(NY / 2^lmax) */
    uint64_t scored[SO_BNB_LEVELS];         /* per level: nodes whose bound was computed (level 0: hypotheses scored) */
    uint64_t discarded[SO_BNB_LEVELS];      /* per level: nodes discarded by the pruning rule */
    uint64_t leaves_scored;                 /* scored[0] */
    uint64_t steps;                         /* traversal steps (one small read-back each) */
    uint64_t pyramid_bytes;                 /* device bytes of all pyramid levels */
    double time_build_ms;                   /* device time: map bounds, raster, dilation, levels, offset table (CUDA events) */
    double time_search_ms;                  /* device time of the traversal (CUDA events) */
} so_bnb_stats;

/* Arguments and stage times as so_localize_global, plus optional statistics.  Errors before any device work: argument errors as
 * so_localize_global, SO_ERR_CAPACITY above 2^32 hypotheses or an offset table (NYAW * score points * 16 B) above 1 GiB; after the
 * map bounds: SO_ERR_CAPACITY for a pyramid level above 2^32 bits. */
int so_localize_global_bnb(so_ctx* ctx, const void* xyzi, size_t n, size_t stride_bytes, size_t intensity_offset, const double center_pose7[7],
                           const so_global_opts* gopts, const so_icp_opts* opts, so_global_candidate* cands, size_t cap,
                           so_global_result* out, so_bnb_stats* stats);
/* Stage hook: the first min(NX*NY*NZ*NYAW, 64 k) keys (65535 - score) << 32 | index of the ascending order of every hypothesis'
 * key: the prefix so_localize_global refines.  Writes min(*n_keys, cap) keys; *n_keys = the prefix length. */
int so_localize_bnb_keys(so_ctx* ctx, const void* xyzi, size_t n, size_t stride_bytes, size_t intensity_offset, const double center_pose7[7],
                         const so_global_opts* gopts, uint64_t* keys, size_t cap, size_t* n_keys, so_bnb_stats* stats);
/* Stage hook: U of every node of pyramid level `level` (0 .. lmax), index ((yaw * NZ + z) * NBY + by) * NBX + bx with
 * NBX = ceil(NX / 2^level), NBY = ceil(NY / 2^level); dims = {NBX, NBY, NZ, NYAW}.  Level 0 equals so_localize_scores.  dims are
 * also filled when cap is below the node count (SO_ERR_CAPACITY, returned before any device work; out may then be NULL). */
int so_localize_bnb_bounds(so_ctx* ctx, const void* xyzi, size_t n, size_t stride_bytes, size_t intensity_offset, const double center_pose7[7],
                           const so_global_opts* gopts, int level, uint16_t* out, size_t cap, int32_t dims[4]);
/* Bounding box of the surf map, reduced on the device; *n = its point count (lo and hi are zero for an empty map). */
int so_map_bounds(so_ctx* ctx, float lo[3], float hi[3], size_t* n);
/* The same over the surf window plus the surf archive (so_map_archive), read in place on the device; with the archive off it equals
 * so_map_bounds. */
int so_map_bounds_all(so_ctx* ctx, float lo[3], float hi[3], size_t* n);

/* ---- global localization over the whole archived map (so_global_opts.whole_map = 1) ----------------------------------------------
 * Accepted by so_localize_global, so_localize_global_bnb, so_localize_scores, so_localize_bnb_keys and so_localize_bnb_bounds.  With
 * the archive off the call is the whole_map = 0 call, bit for bit (n_windows = 0, the window does not move).  With it on:
 *   - Any pending origin change is applied first; call that origin O0.
 *   - Search: the occupancy bitmap (level 0 of the pyramid) is rastered from the window's points and every point of the archive's
 *     live segments, read in place.  The raster ORs bits and the bounds reduce with min / max, so the scores are a function of the
 *     whole map's point set only; the branch-and-bound clips its window with so_map_bounds_all's box.  Everything after the raster is
 *     unchanged.
 *   - Refinement: O(c) is the origin so_map_shift(c.prior) would leave when called at O0.  The candidates are grouped by O(c), the
 *     groups ordered by their best-ranked member; for each group the window moves to O(c) (the archive evicts and restores blocks)
 *     and the group registers in rank order, max_batch at a time.  Each candidate's registration equals so_map_shift(prior) followed
 *     by so_register_batch(scan, prior) on the same map at O0, bit for bit.  The winner rule is unchanged.
 *   - On return the origin is O(winner), with the window built there, so so_map_add_registered_scan(pose) inserts where the robot
 *     is; with no winner it is O0 again.  Both stores move together (the origin is shared).  A move the archive has no room for fails
 *     the call with SO_ERR_CAPACITY under the archive's rule (the store is left unbuilt; growing the archive recovers it).
 * The limits are unchanged: 2^32 hypotheses, 2^32 bits per pyramid level, the 1 GiB offset table.  A strip 2 km x 100 m at 0.25 m and
 * 2 deg (about 5.8e8 hypotheses) fits; a 1.5 km x 1.5 km square needs a coarser res or yaw_step. */

/* ---- instrumentation ------------------------------------------------------------------------------ */
/* Number of this library's kernels launched since the last reset (bench.py gpu_launches). */
uint64_t so_kernel_launches(so_ctx* ctx, int reset);
/* Bytes this library copied host->device / device->host for scans, poses, optimiser state and results since the
 * last reset (bench.py e2e accounting). */
int so_bytes_copied(so_ctx* ctx, uint64_t* h2d, uint64_t* d2h, int reset);
/* Accumulated device time (ms, CUDA events on the context stream) and launch count of a kernel class since the last
 * reset; classes: 0 k_knn_scan (scan k-NN), 1 k_evaluate +
 * k_lm_step (LM step), 2 k_knn (so_knn*), 3 scan ordering / map build / map insert / free-space clearing / scan preparation (pre-filter, deskew, uniform and edge extraction), 4 first evaluation of
 * a solve (k_evaluate + k_lm_step iteration zero), 5 k_fit (plane fit), 6 global localization search (map bounds, bitmap raster,
 * dilation, pyramid levels, offset table, traversal steps and dense scoring),
 * 7 k_undistort (within-scan motion compensation: per ICP iteration, and the undistorted map insert / so_undistort_points; the
 * per-iteration warp and the map insert of so_register_optimized*), 8 evaluation + trust-region step of so_register_optimized*.
 * Profiling mode serialises kernels; enable only for roofline runs. */
/* Build-time switches of the loaded library.  Bit 0 (SO_BUILD_FUSED_MATCH, search and fit as one kernel) is reserved: this
 * library always runs them as two kernels and returns 0. */
#define SO_BUILD_FUSED_MATCH 1
int so_build_flags(void);
int so_profile_enable(so_ctx* ctx, int on);
int so_profile_get(so_ctx* ctx, int kernel_class, double* ms, uint64_t* launches, int reset);
/* Neighbour graph of the surf store, which so_register_batch* builds by itself when a call's queries number at least 8 times the
 * store's points and answers most neighbour searches from (same results, fewer candidates).  Builds it for the current map when
 * none is valid, then, when the buffers are given, writes for each point of the store in search order its id (point_id[t]), the
 * ids of its *k nearest points of the same 50 m block (nbr_id[t * k + j], ascending (d2, id), 0xFFFFFFFF when the block holds fewer)
 * and radius[t]: 0.99999 x the distance to the last of them, +inf when the block holds at most *k other points, 0 when unused.
 * *n_out = points of the store; cap_points < *n_out is SO_ERR_CAPACITY. */
int so_knn_graph(so_ctx* ctx, uint32_t* point_id, uint32_t* nbr_id, float* radius, size_t cap_points, uint32_t* k, size_t* n_out);
/* Counters of the searches of k_knn_scan per ICP iteration: counts[2 i] = queries searched in iteration i, counts[2 i + 1] = those
 * the neighbour graph answered (counts may be NULL).  Reads them, then on != 0 resets and keeps counting, on == 0 stops. */
int so_knn_graph_stats(so_ctx* ctx, int on, uint64_t* counts);

#ifdef __cplusplus
}
#endif
#endif /* SUPERODOM_B200_H */
