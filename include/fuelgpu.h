/*
 * fuelgpu.h -- C ABI of the H100-native replacement for FUEL's per-replan hot path.
 *
 * The reference (HKUST-Aerial-Robotics/FUEL) exposes no C ABI or plugin interface: its
 * boundary is the public C++ surface of SDFMap / EDTEnvironment / FrontierFinder /
 * BsplineOptimizer linked through catkin shared libraries (SURVEY.md 8b).  Every entry
 * point below cites the reference method (file:line under fuel_planner/) whose body it
 * replaces; INTEGRATION.md shows the C++ shim a maintainer adds on the reference side.
 *
 * Conventions
 *   - extern "C", plain pointers and sizes, no C++/torch types.
 *   - every function returns 0 on success, a negative FUELGPU_E* code otherwise;
 *     fuelgpu_last_error() gives the message (per handle; NULL handle = creation errors).
 *   - host buffers are caller-owned.  Volume buffers use the reference layout
 *     address = x*ny*nz + y*nz + z (SDFMap::toAddress, plan_env/include/plan_env/sdf_map.h:145-147).
 *   - one opaque handle per map; all device state (occupancy byte, ESDF, frontier flags,
 *     scratch) lives in HBM behind it.  Calls on one handle are serialised on its stream
 *     (the reference is single-threaded for these, exploration_node.cpp:19);
 *     fuelgpu_bspline_* calls are re-entrant across handles.
 *   - there is NO CPU fallback: without a CUDA device every call fails with
 *     FUELGPU_ENODEVICE.
 */
#ifndef FUELGPU_H
#define FUELGPU_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(__GNUC__)
#define FUELGPU_API __attribute__((visibility("default")))
#else
#define FUELGPU_API
#endif

#define FUELGPU_OK 0
#define FUELGPU_EINVAL -1    /* bad argument                                  */
#define FUELGPU_ENODEVICE -2 /* no CUDA device / wrong architecture          */
#define FUELGPU_ECUDA -3     /* CUDA runtime error (see fuelgpu_last_error)  */
#define FUELGPU_ENOMEM -4    /* device or host allocation failed             */
#define FUELGPU_EUNSUPPORTED -5

typedef struct FuelMap FuelMap;

/* Grid geometry = the fields of MapParam that the hot path reads
 * (plan_env/include/plan_env/sdf_map.h:86-105; filled by SDFMap::initMap, sdf_map.cpp:12-93). */
typedef struct {
  int32_t n[3];       /* map_voxel_num_                      */
  double resolution;  /* resolution_                         */
  double origin[3];   /* map_origin_ (= map_min_boundary_)   */
  double box_mind[3]; /* box_mind_  exploration box, metres  */
  double box_maxd[3]; /* box_maxd_                           */
  double map_size[3]; /* map_size_ (sdf_map/map_size_x,y,z): map_max_boundary_ = origin + map_size_ (sdf_map.cpp:34-39),
                         which is not always n*resolution in floating point (n = ceil(size/resolution)).
                         All zero = n * resolution. */
} FuelGridDesc;

/* Occupancy tri-state of SDFMap::getOccupancy (sdf_map.h:32,194-200). */
enum { FUELGPU_UNKNOWN = 0, FUELGPU_FREE = 1, FUELGPU_OCCUPIED = 2 };

/* ---- lifetime --------------------------------------------------------------------- */
/* Replaces the allocations of SDFMap::initMap (sdf_map.cpp:62-76) and the frontier_flag_
 * allocation of FrontierFinder::FrontierFinder (active_perception/src/frontier_finder.cpp:23-27). */
FUELGPU_API int fuelgpu_map_create(const FuelGridDesc* grid, int device_id, FuelMap** out);
FUELGPU_API int fuelgpu_map_destroy(FuelMap* map);
FUELGPU_API const char* fuelgpu_last_error(const FuelMap* map);
/* Run all work of this handle on `cuda_stream` (a cudaStream_t; NULL = the handle's own). */
FUELGPU_API int fuelgpu_map_set_stream(FuelMap* map, void* cuda_stream);
FUELGPU_API int fuelgpu_map_synchronize(FuelMap* map);
/* Device pointers of the resident state, for zero-copy callers (torch tensors, NCCL):
 * occ  = uint8 per voxel: bits0-1 tri-state, bit2 occupancy_buffer_inflate_
 * dist = float32 per voxel: distance_buffer_ in metres
 * flag = int8 per voxel: frontier_flag_ */
FUELGPU_API int fuelgpu_map_device_ptrs(FuelMap* map, void** occ, void** dist, void** flag);
/* Milliseconds spent on the device by the last call of each stage (CUDA events on the
 * handle's stream): [0] esdf_update [1] frontier_search [2] bspline batch [3] upload [4] download
 * [5] trajectory check (fuelgpu_bspline_check_batch[_dev]) [6] trajectory parameterization
 * (fuelgpu_bspline_parameterize_batch[_dev]) [7] waypoint polynomial (fuelgpu_poly_waypoints_batch[_dev]) */
FUELGPU_API int fuelgpu_map_last_timing(FuelMap* map, float ms[8]);
/* Where the last call of each stage sat on the device timeline: start and end in milliseconds after the start of the
 * last upload (same stage indices; -1 = stage not run or no upload recorded).  Diagnostic for overlapped sequences. */
FUELGPU_API int fuelgpu_map_last_timeline(FuelMap* map, float start_ms[8], float end_ms[8]);
/* Number of kernels this handle has launched since creation (every <<<>>> is counted). */
FUELGPU_API int fuelgpu_map_launch_count(FuelMap* map, int64_t* count);

/* Page-lock a long-lived caller buffer (e.g. the std::vector storage of occupancy_buffer_inflate_ /
 * distance_buffer_ that SDFMap::initMap sizes once, sdf_map.cpp:62-76) so that the H2D / D2H legs run
 * at full PCIe rate.  Optional; unregistered buffers work, slower.  cudaHostRegister underneath. */
FUELGPU_API int fuelgpu_host_register(void* ptr, uint64_t bytes);
FUELGPU_API int fuelgpu_host_unregister(void* ptr);

/* ---- ingest: host occupancy -> resident occupancy byte ------------------------------
 * Replaces nothing in the reference (its buffers are already in RAM); this is the H2D leg.
 * inflate  : occupancy_buffer_inflate_ (char {0,1}), full volume                (sdf_map.h:110)
 * logodds  : occupancy_buffer_ (double log-odds), full volume, or NULL          (sdf_map.h:109)
 * tristate : precomputed getOccupancy() per voxel, or NULL.  Exactly one of logodds /
 *            tristate must be given.  With logodds the device applies sdf_map.h:196-199:
 *            occ < clamp_min_log-1e-3 -> UNKNOWN, occ > min_occupancy_log -> OCCUPIED.
 * bmin/bmax: inclusive index box to refresh (NULL = whole map).  The x-slab range
 *            [bmin[0],bmax[0]] is copied (x is the slowest axis, so that is contiguous). */
FUELGPU_API int fuelgpu_map_upload_occupancy(FuelMap* map, const int8_t* inflate, const double* logodds,
                                 const uint8_t* tristate, double clamp_min_log,
                                 double min_occupancy_log, const int32_t bmin[3],
                                 const int32_t bmax[3]);
/* Same, but returns as soon as the copies are queued: the caller must leave the host buffers alone until the
 * next fuelgpu_map_synchronize / blocking call on this map (page-locked buffers are read by DMA later). */
FUELGPU_API int fuelgpu_map_upload_occupancy_async(FuelMap* map, const int8_t* inflate, const double* logodds,
                                                   const uint8_t* tristate, double clamp_min_log,
                                                   double min_occupancy_log, const int32_t bmin[3],
                                                   const int32_t bmax[3]);

/* Replaces SDFMap::clearAndInflateLocalMap (plan_env/src/sdf_map.cpp:364-472), the step between the
 * occupancy fusion and updateESDF3d (SURVEY 8f rank 2), on the resident occupancy byte: the inflate bit
 * is cleared inside [bmin,bmax] and every OCCUPIED voxel of the box stamps its (2*inf_step+1)^3
 * neighbourhood (inf_step = ceil(obstacles_inflation_/resolution_), :436), with the reference's
 * linear-address-only bounds check (:452-458).  virtual_ceil_idx >= 0 marks z = idx OCCUPIED for the
 * box's (x,y) (:462-470); pass -1 when virtual_ceil_height_ <= -0.5.  Read the bytes back with
 * fuelgpu_map_download_occupancy. */
FUELGPU_API int fuelgpu_map_inflate(FuelMap* map, const int32_t bmin[3], const int32_t bmax[3], int32_t inf_step,
                        int32_t virtual_ceil_idx);
/* Resident occupancy byte -> host: inflate (int8 {0,1}) and/or tristate (uint8), full volume. */
FUELGPU_API int fuelgpu_map_download_occupancy(FuelMap* map, int8_t* inflate, uint8_t* tristate);

/* ---- occupancy fusion (SURVEY 8f rank 3) ------------------------------------------------ */
/* MapParam's fusion constants as probabilities (sdf_map.cpp:36-47 logit()s them) */
typedef struct {
  double p_hit, p_miss, p_min, p_max, p_occ; /* sdf_map/p_hit, p_miss, p_min, p_max, p_occ */
  double max_ray_length;                     /* sdf_map/max_ray_length */
  double local_bound_inflate;                /* sdf_map/local_bound_inflate */
} FuelFusionParams;

/* Replaces SDFMap::inputPointCloud (plan_env/src/sdf_map.cpp:259-345; setCacheOccupancy :243-257,
 * closetPointInMap :347-362, RayCaster plan_env/src/raycast.cpp:323-407) on a device-resident fp64
 * log-odds volume (occupancy_buffer_, created on first use at clamp_min_log_ - unknown_flag_,
 * sdf_map.cpp:56,64).  points = point_num float32 xyz in host memory, point_stride floats apart: 4 for
 * pcl::PointCloud<pcl::PointXYZ>::points.data() (16-byte points), 3 for packed xyz.  The resident
 * tri-state byte is refreshed for every touched voxel, so fuelgpu_map_inflate / fuelgpu_esdf_update /
 * fuelgpu_frontier_search can follow without any upload.  local_bound_min/max receive
 * md_->local_bound_min_/max_ (:313-318). */
FUELGPU_API int fuelgpu_map_input_point_cloud(FuelMap* map, const float* points, int32_t point_num,
                                              int32_t point_stride, const double camera_pos[3], const FuelFusionParams* params,
                                              int32_t local_bound_min[3], int32_t local_bound_max[3]);
/* MapROS's camera parameters (plan_env/src/map_ros.cpp:24-37; values exploration.launch:38-41, algorithm.xml:61-69) */
typedef struct {
  double fx, fy, cx, cy;
  double k_depth_scaling_factor, depth_filter_maxdist, depth_filter_mindist;
  int32_t depth_filter_margin, skip_pixel;
} FuelCameraParams;

/* Replaces MapROS::proessDepthImage + the inputPointCloud call of depthPoseCallback
 * (plan_env/src/map_ros.cpp:139-140, 176-215): the uint16 depth image (rows x cols, row-major, host memory) is
 * projected on the device (camera_R = row-major camera_q_.toRotationMatrix()) and fused as above; the world points
 * never exist on the host.  proj_points_cnt (may be NULL) receives the number of projected points. */
FUELGPU_API int fuelgpu_map_input_depth_image(FuelMap* map, const uint16_t* depth, int32_t rows, int32_t cols,
                                              const FuelCameraParams* camera, const double camera_R[9],
                                              const double camera_pos[3], const FuelFusionParams* params,
                                              int32_t local_bound_min[3], int32_t local_bound_max[3],
                                              int32_t* proj_points_cnt);
/* SDFMap::getUpdatedBox (sdf_map.cpp:491-495): md_->update_min_/max_ accumulated by the fusion calls
 * since the last reset. */
FUELGPU_API int fuelgpu_map_get_updated_box(FuelMap* map, double bmin[3], double bmax[3], int32_t reset);
/* Whole-volume access to the resident log-odds (tests, map save/restore).  set also re-derives the
 * tri-state byte (getOccupancy, sdf_map.h:194-200) with clamp_min_log_ = logit(p_min),
 * min_occupancy_log_ = logit(p_occ). */
FUELGPU_API int fuelgpu_map_set_logodds(FuelMap* map, const double* logodds, double p_min, double p_occ);
FUELGPU_API int fuelgpu_map_get_logodds(FuelMap* map, double* logodds);

/* ---- ESDF -------------------------------------------------------------------------- */
#define FUELGPU_ESDF_OPTIMISTIC 1 /* mp_->optimistic_  (sdf_map.cpp:156) */
#define FUELGPU_ESDF_SIGNED 2     /* mp_->signed_dist_ (sdf_map.cpp:201) */
/* Replaces SDFMap::updateESDF3d (plan_env/src/sdf_map.cpp:152-241) incl. fillESDF (:116-150).
 * bmin/bmax = md_->local_bound_min_/max_ (inclusive).  Result: distance_buffer_ inside the
 * box, float32 metres.  A voxel with no site anywhere in the box gets +inf (the reference
 * stores resolution*sqrt(DBL_MAX) ~ 1.34e153 there; see DESIGN.md "sentinel"). */
FUELGPU_API int fuelgpu_esdf_update(FuelMap* map, const int32_t bmin[3], const int32_t bmax[3], int flags);
/* distance_buffer_ -> host, for the scattered single-point CPU readers of
 * SDFMap::getDistance (sdf_map.h:228-237).  Exactly one of out_f32/out_f64 non-NULL; full
 * volume layout; the x-slab range of the box is copied. */
FUELGPU_API int fuelgpu_esdf_download(FuelMap* map, const int32_t bmin[3], const int32_t bmax[3],
                          float* out_f32, double* out_f64);
/* Same for float32, without blocking: the copy is queued on the handle's copy stream behind the
 * ESDF update and overlaps whatever runs next on the main stream (the trajectory batch); the host
 * buffer is valid after fuelgpu_map_synchronize().  Later writers of the field on the main stream
 * (fuelgpu_esdf_update, fuelgpu_esdf_set_from_slabs_dev) wait for the copy, so the buffer holds the
 * field as it was when this call was made.  Use with a page-locked buffer. */
FUELGPU_API int fuelgpu_esdf_download_async(FuelMap* map, const int32_t bmin[3], const int32_t bmax[3],
                                float* out_f32);
/* Replaces SDFMap::getDistWithGrad (sdf_map.cpp:497-536) = EDTEnvironment::evaluateEDTWithGrad
 * (plan_env/src/edt_environment.cpp:78-87) for n positions.  pos [n][3], dist [n], grad [n][3]. */
FUELGPU_API int fuelgpu_esdf_sample(FuelMap* map, int64_t n, const double* pos, double* dist, double* grad);

/* ---- frontier ---------------------------------------------------------------------- */
typedef struct {
  int32_t cluster_min;    /* frontier/cluster_min     frontier_finder.cpp:29 */
  double cluster_size_xy; /* frontier/cluster_size_xy frontier_finder.cpp:30 */
  int32_t down_sample;    /* frontier/down_sample     frontier_finder.cpp:38 */
  double min_z;           /* the literal 0.4 of frontier_finder.cpp:152      */
} FuelFrontierParams;

/* Replaces the voxel-scale part of FrontierFinder::searchFrontiers
 * (active_perception/src/frontier_finder.cpp:94-118): the sweep over the inflated updated
 * box, expandFrontier (:123-164), computeFrontierInfo (:374-390), downsample (:757-774)
 * and splitLargeFrontiers / splitHorizontally (:166-242).  upd_min/upd_max = the box
 * returned by SDFMap::getUpdatedBox (metres).  frontier_flag_ stays on the device and is
 * updated exactly as the reference does (cells of dropped small clusters stay flagged).
 * Outputs the sizes needed for fuelgpu_frontier_fetch.  Clusters come in tmp_frontiers_
 * order; cells of a cluster in ascending address order (DESIGN.md "frontier cell order"). */
FUELGPU_API int fuelgpu_frontier_search(FuelMap* map, const double upd_min[3], const double upd_max[3],
                            const FuelFrontierParams* params, int32_t* n_clusters,
                            int32_t* n_cells, int32_t* n_filtered);
/* The same search split in two so that the caller can overlap it with other work: _begin enqueues
 * the sweep and the clustering on the handle's frontier stream and returns at once; _end waits for
 * it and returns the sizes.  fuelgpu_frontier_search == _begin followed by _end.  The frontier
 * subsystem only reads the occupancy byte and owns frontier_flag_, so ESDF updates and B-spline
 * batches may be issued between the two calls (they run on the handle's main stream). */
FUELGPU_API int fuelgpu_frontier_search_begin(FuelMap* map, const double upd_min[3], const double upd_max[3],
                                  const FuelFrontierParams* params);
FUELGPU_API int fuelgpu_frontier_search_end(FuelMap* map, int32_t* n_clusters, int32_t* n_cells,
                                int32_t* n_filtered);
/* cell_offsets [n_clusters+1], cell_addr [n_cells] (toAddress), filt_offsets [n_clusters+1],
 * filtered [n_filtered][3] (Frontier::filtered_cells_), average/box_min/box_max [n_clusters][3]
 * (Frontier::average_/box_min_/box_max_, frontier_finder.h:34-51).  Any pointer may be NULL. */
FUELGPU_API int fuelgpu_frontier_fetch(FuelMap* map, int32_t* cell_offsets, int32_t* cell_addr,
                           int32_t* filt_offsets, double* filtered, double* average,
                           double* box_min, double* box_max);
/* ---- z-sharded frontier sweep (SURVEY 8e row 2) ----------------------------------------------------------
 * The voxel sweep shards on z, the clustering (O(frontier cells)) runs on the union of the candidates:
 *   1. every rank holds the tri-state of its planes [z_lo, z_hi] plus one halo plane on each side
 *      (fuelgpu_map_occupancy_plane_dev moves a plane to / from a contiguous device buffer for the exchange);
 *   2. fuelgpu_frontier_candidates sweeps ITS planes (knownfree && isNeighborUnknown && frontier_flag_ == 0,
 *      frontier_finder.cpp:108-117,862-877) and returns its candidate cells: address + class (1 = may be absorbed
 *      by a region growth, 2 = can only seed one, :146-152);
 *   3. the host program gathers the lists of all ranks and merges them by ascending address (KBs);
 *   4. fuelgpu_frontier_search_from_candidates clusters + splits the full list on every rank: same kernels and the
 *      same result as fuelgpu_frontier_search on one GPU, bit for bit; frontier_flag_ is updated for all cells on
 *      every rank (replicated).  Results through fuelgpu_frontier_fetch as usual. */
FUELGPU_API int fuelgpu_frontier_candidates(FuelMap* map, const double upd_min[3], const double upd_max[3],
                                            const FuelFrontierParams* params, int32_t z_lo, int32_t z_hi,
                                            int32_t* n_candidates);
FUELGPU_API int fuelgpu_frontier_candidates_fetch(FuelMap* map, int32_t n, int32_t* addr, uint8_t* cls);
FUELGPU_API int fuelgpu_frontier_search_from_candidates(FuelMap* map, const double upd_min[3], const double upd_max[3],
                                                        const FuelFrontierParams* params, int32_t n, const int32_t* addr,
                                                        const uint8_t* cls, int32_t* n_clusters, int32_t* n_cells,
                                                        int32_t* n_filtered);
/* plane z of the resident occupancy byte -> plane_dev [nx][ny] (set = 0) or plane_dev -> plane z (set = 1) */
FUELGPU_API int fuelgpu_map_occupancy_plane_dev(FuelMap* map, int32_t z, void* plane_dev, int32_t set);

/* Order of a cluster's cells in fuelgpu_frontier_fetch.  BY_ADDRESS (default): ascending toAddress, straight
 * from the device.  BFS: the reference's own order (expandFrontier's BFS from the seed, :139-156, kept by
 * splitHorizontally, :217-224), re-derived on the host from the fetched cell sets; average_ and filtered_cells_ are
 * then recomputed in that order and equal the reference's to the last bit.  Cluster membership, cluster order and
 * frontier_flag_ are the same in both modes. */
#define FUELGPU_CELLS_BY_ADDRESS 0
#define FUELGPU_CELLS_BFS 1
FUELGPU_API int fuelgpu_frontier_set_cell_order(FuelMap* map, int32_t order);
/* Replaces the resetFlag lambda of searchFrontiers (:62-69): frontier_flag_[addr] = 0. */
FUELGPU_API int fuelgpu_frontier_clear_flags(FuelMap* map, int32_t n, const int32_t* addr);
/* Replaces FrontierFinder::isFrontierChanged (:365-372) for m stored clusters given in CSR
 * form; changed[i] = 1 iff some cell of cluster i stopped being a frontier cell. */
FUELGPU_API int fuelgpu_frontier_is_changed(FuelMap* map, int32_t m, const int32_t* cell_offsets,
                                const int32_t* cell_addr, uint8_t* changed);
/* frontier_flag_ = 0 everywhere: the fill of FrontierFinder::FrontierFinder (frontier_finder.cpp:26-27). */
FUELGPU_API int fuelgpu_frontier_reset_flags(FuelMap* map);
FUELGPU_API int fuelgpu_frontier_download_flags(FuelMap* map, int8_t* out);
FUELGPU_API int fuelgpu_frontier_upload_flags(FuelMap* map, const int8_t* in);

/* ---- viewpoint sampling (SURVEY 8f rank 4) ---------------------------------------------- */
typedef struct {
  double candidate_rmin, candidate_rmax; /* frontier/candidate_rmin, candidate_rmax (frontier_finder.cpp:35-36) */
  int32_t candidate_rnum;                /* frontier/candidate_rnum (:37) */
  double candidate_dphi;                 /* frontier/candidate_dphi (:34) */
  double min_candidate_clearance;        /* frontier/min_candidate_clearance (:33) */
  double top_angle, left_angle, right_angle, max_dist; /* perception_utils params (perception_utils.cpp:7-10) */
} FuelViewParams;

/* Number of (radius, angle) candidates the loops of sampleViewpoints visit (frontier_finder.cpp:664-667);
 * negative on a degenerate parameter set. */
FUELGPU_API int32_t fuelgpu_viewpoint_candidate_count(const FuelViewParams* params);
/* Replaces FrontierFinder::sampleViewpoints (active_perception/src/frontier_finder.cpp:662-695) with
 * isNearUnknown (:721-732), countVisibleCells (:734-755) and PerceptionUtils::setPose/insideFOV
 * (active_perception/src/perception_utils.cpp:49-93) for n_clusters clusters at once, against the resident
 * occupancy byte.  Inputs in the layout fuelgpu_frontier_fetch returns: filt_offsets[n_clusters+1],
 * filtered[3*filt_offsets[n]] (filtered_cells_), average[3*n_clusters].  Outputs, n_cand =
 * fuelgpu_viewpoint_candidate_count() entries per cluster in the reference's loop order:
 *   cand_pos[3*n*n_cand] sample_pos; cand_yaw[n*n_cand] avg_yaw; cand_visib[n*n_cand] = countVisibleCells,
 *   or -1 where the candidate fails isInBox / getInflateOccupancy / isNearUnknown (:671-673).
 * The caller keeps candidates with visib > min_visib_num_ (:688) and sorts them (:404-406). */
FUELGPU_API int fuelgpu_frontier_sample_viewpoints(FuelMap* map, int32_t n_clusters, const int32_t* filt_offsets,
                                                   const double* filtered, const double* average,
                                                   const FuelViewParams* params, int32_t n_cand, double* cand_pos,
                                                   double* cand_yaw, int32_t* cand_visib);
/* isFrontierCovered's per-cluster count (frontier_finder.cpp:697-719): how many of each stored cluster's cells are
 * no longer frontier cells; the caller compares with min_view_finish_fraction_ * size.  Same CSR input as
 * fuelgpu_frontier_is_changed. */
FUELGPU_API int fuelgpu_frontier_changed_counts(FuelMap* map, int32_t n_clusters, const int32_t* cell_offsets,
                                                const int32_t* cell_addr, int32_t* counts);

/* ---- B-spline cost ------------------------------------------------------------------ */
/* cost-term bits = BsplineOptimizer::SMOOTHNESS..MINTIME (bspline_opt/src/bspline_optimizer.cpp:10-18) */
#define FUELGPU_SMOOTHNESS (1 << 0)
#define FUELGPU_DISTANCE (1 << 1)
#define FUELGPU_FEASIBILITY (1 << 2)
#define FUELGPU_START (1 << 3)
#define FUELGPU_END (1 << 4)
#define FUELGPU_GUIDE (1 << 5)
#define FUELGPU_WAYPOINTS (1 << 6)
#define FUELGPU_VIEWCONS (1 << 7) /* calcViewCost :477-502; needs FuelTrajConst.view_idx >= 0 */
#define FUELGPU_MINTIME (1 << 8)
/* not a cost term: evaluate with the solver loop's evaluator (fuelgpu_bspline_optimize_batch runs it: fp32
 * trilinear lerps on the fp32 ESDF samples, reciprocals, FMA contraction) instead of the faithful one; same
 * 1e-4 parity bar, n_pts <= 64 (above 32 points: the two-points-per-lane evaluator of the long-trajectory solver) */
#define FUELGPU_COST_FAST_EVAL (1 << 30)

/* BsplineOptimizer::setParam (bspline_optimizer.cpp:25-57) */
typedef struct {
  double ld_smooth, ld_dist, ld_feasi, ld_start, ld_end, ld_guide, ld_waypt, ld_view, ld_time;
  double dist0, max_vel, max_acc;
  int32_t order; /* order_ = bspline_degree_ */
  double wnl;    /* wnl_ (optimization/wnl, :44): weight of the parallel part of calcViewCost */
} FuelOptParams;

#define FUELGPU_MAX_PTS 64
/* per-trajectory constants frozen by BsplineOptimizer::optimize() before the solver runs
 * (bspline_optimizer.cpp:116-141) plus the setters (:82-108) */
typedef struct {
  double pt_dist;     /* pt_dist_ (:136-140)                     */
  double knot_span;   /* knot_span_, used when MINTIME is off    */
  double start[3][3]; /* start_state_: pos, vel, acc             */
  double end[3][3];   /* end_state_                               */
  int32_t n_end;      /* end_state_.size(), 1..3                  */
  double time_lb;     /* time_lb_                                 */
  int32_t n_guide;    /* guide_pts_.size()                        */
  double guide[FUELGPU_MAX_PTS][3];
  int32_t n_waypt;    /* waypoints_.size()                        */
  double waypt[FUELGPU_MAX_PTS][3];
  int32_t waypt_idx[FUELGPU_MAX_PTS];
  double view_pt[3];  /* view_cons_.pt_  (setViewConstraint :91-93)  */
  double view_dir[3]; /* view_cons_.dir_ (its length = safe distance) */
  int32_t view_idx;   /* view_cons_.idx_; < 0: none set (VIEWCONS then returns FUELGPU_EINVAL) */
} FuelTrajConst;

/* Replaces BsplineOptimizer::combineCost (bspline_optimizer.cpp:518-647) and the calc*Cost
 * it calls (:255-516) for B trajectories of n_pts control points (dim_ == 3) against this
 * map's ESDF.  x [B][nvar], nvar = 3*n_pts (+1 = dt when MINTIME); f [B]; grad [B][nvar].
 * B == 1 is the BsplineOptimizer::costFunction trampoline (:693-706). */
FUELGPU_API int fuelgpu_bspline_cost_batch(FuelMap* map, int32_t B, int32_t n_pts, int32_t cost_mask,
                               const FuelOptParams* params, const FuelTrajConst* traj,
                               const double* x, double* f, double* grad);
/* Same, all pointers in device memory (traj = device array of FuelTrajConst). */
FUELGPU_API int fuelgpu_bspline_cost_batch_dev(FuelMap* map, int32_t B, int32_t n_pts, int32_t cost_mask,
                                   const FuelOptParams* params, const void* traj_dev,
                                   const void* x_dev, void* f_dev, void* grad_dev);

/* Replaces the solver loop of BsplineOptimizer::optimize() (bspline_optimizer.cpp:165-253:
 * clamp to box+-0.1, bounds, maxeval stop, best-x tracking of costFunction :693-706) for a
 * whole batch on the device.  NLopt (third party, LD_LBFGS) is replaced by a projected
 * L-BFGS run per trajectory inside one persistent kernel; iterate-level parity with NLopt
 * is unpinned (SURVEY 8c), the CPU twin is oracle/orc_optimize_batch.
 * x [B][nvar] in/out (best_variable_), f_best [B], n_eval [B].  n_pts <= 64: up to 32 lanes (n_pts + dt) one
 * control point per lane, above that two per lane.  At every n_pts, f_best is exactly (bit for bit) what
 * fuelgpu_bspline_cost_batch returns for the returned x: the faithful evaluator runs on it after the solver, on the
 * same stream. */
typedef struct {
  int32_t max_eval; /* max_iteration_num_[id]  (algorithm.xml:184-187) */
  int32_t lbfgs_m;  /* history pairs, <= 8                              */
  double xtol_rel;  /* 1e-5 (bspline_optimizer.cpp:173)                 */
  int32_t flags;    /* FUELGPU_SOLVE_*                                   */
  int32_t reserved;
} FuelSolveParams;
/* keep evaluating until max_eval is reached: a failed line search restarts from steepest descent and a vanished
 * gradient re-evaluates in place (benchmark mode: exactly B x max_eval combineCost evaluations, like a CPU run that
 * calls the objective max_eval times) */
#define FUELGPU_SOLVE_EXACT_EVALS 1
FUELGPU_API int fuelgpu_bspline_optimize_batch(FuelMap* map, int32_t B, int32_t n_pts, int32_t cost_mask,
                                   const FuelOptParams* params, const FuelTrajConst* traj,
                                   const FuelSolveParams* solve, double* x, double* f_best,
                                   int32_t* n_eval);

/* Same, all pointers in device memory. */
/* The same in two halves, so the caller can do other host work (e.g. fuelgpu_frontier_search_end + fetch) while
 * the solver runs: _begin stages the inputs and enqueues everything, _end waits and copies x / f_best / n_eval
 * out.  One outstanding call per map; other work on the map's main stream queues behind the solver. */
FUELGPU_API int fuelgpu_bspline_optimize_batch_begin(FuelMap* map, int32_t B, int32_t n_pts, int32_t cost_mask,
                                                     const FuelOptParams* p, const FuelTrajConst* traj,
                                                     const FuelSolveParams* solve, const double* x);
FUELGPU_API int fuelgpu_bspline_optimize_batch_end(FuelMap* map, double* x, double* f_best, int32_t* n_eval);
FUELGPU_API int fuelgpu_bspline_optimize_batch_dev(FuelMap* map, int32_t B, int32_t n_pts, int32_t cost_mask,
                                       const FuelOptParams* params, const void* traj_dev,
                                       const FuelSolveParams* solve, void* x_dev, void* f_best_dev,
                                       void* n_eval_dev);

/* ---- trajectory verdicts: NonUniformBspline checks, checkTrajCollision, selectBestTraj -----------------------
 * Uniform cubic B-splines (setUniformBspline(ctrl, 3, dt), bspline/src/non_uniform_bspline.cpp:16-32) in the solver's
 * layout: x [B][nvar] holds the control points of trajectory b as x[b][3*i + axis].  nvar == 3*n_pts + 1: the knot
 * span is x[b][3*n_pts] (MINTIME, what the solver returns) and dt must be NULL; nvar == 3*n_pts: dt [B] holds it.
 * n_pts is 4..FUELGPU_MAX_PTS.  Every output equals the reference's fp64 arithmetic bit for bit (DESIGN.md 4.6). */
typedef struct {
  double max_vel, max_acc; /* setPhysicalLimits(pp_.max_vel_, pp_.max_acc_), non_uniform_bspline.cpp:129-133 */
  double t_now;            /* checkTrajCollision's t_now (planner_manager.cpp:97): seconds since the batch's start; 0 = fresh plan */
} FuelTrajCheckParams;

typedef struct {
  double duration;   /* getTimeSum  (:267-269) */
  double jerk;       /* getJerk     (:283-298) */
  double ratio;      /* checkRatio  (:135-160) */
  double distance;   /* checkTrajCollision's `distance` out-value when unsafe; -1 when safe (the reference leaves it untouched) */
  int32_t safe;      /* checkTrajCollision's return value */
  int32_t feasible;  /* checkFeasibility (:443-487) */
  int32_t n_checked; /* fut_t samples the loop evaluated before it stopped */
  int32_t reserved;
} FuelTrajReport;

/* A collision scan stops after this many samples (20 971 s of trajectory at the reference's 0.02 s step) and reports
 * the trajectory safe; the longest scan of the solver's output (64 points, dt 5 s) is about 15 000 samples. */
#define FUELGPU_CHECK_MAX_SAMPLES (1 << 20)

/* checkTrajCollision (planner_manager.cpp:96-118) samples the spline every 0.02 s from t_now, up to 6 m from
 * evaluateDeBoorT(t_now) or the end, and fails on the first sample whose voxel has the inflate bit (bit 2 of the
 * resident occupancy byte, getInflateOccupancy, sdf_map.h:217-226; outside the map is not a hit).
 * best[0] = selectBestTraj (planner_manager.cpp:476-482): index of the least jerk (ties: lowest index; NaN never wins).
 * best[1] = the same among trajectories with safe && feasible; -1 if none.
 * Runs on the map's main stream, so the _dev form can be enqueued straight after fuelgpu_bspline_optimize_batch_dev
 * on its x.  Device time: slot 5 of fuelgpu_map_last_timing. */
FUELGPU_API int fuelgpu_bspline_check_batch(FuelMap* map, int32_t B, int32_t n_pts, int32_t nvar, const double* x,
                                            const double* dt, const FuelTrajCheckParams* params, FuelTrajReport* report,
                                            int32_t best[2]);
FUELGPU_API int fuelgpu_bspline_check_batch_dev(FuelMap* map, int32_t B, int32_t n_pts, int32_t nvar, const void* x_dev,
                                                const void* dt_dev, const FuelTrajCheckParams* params, void* report_dev,
                                                void* best_dev);
/* evaluateDeBoorT (:73-75) of the spline (deriv 0) or of getDerivative() once / twice (deriv 1, 2; :77-106), at
 * t [B][n_t] per trajectory (clamped to [0, duration] like the reference); out [B][n_t][3]. */
FUELGPU_API int fuelgpu_bspline_evaluate_batch(FuelMap* map, int32_t B, int32_t n_pts, int32_t nvar, const double* x,
                                               const double* dt, int32_t n_t, const double* t, int32_t deriv, double* out);

/* ---- trajectory parameterization: the solver's batch from sampled paths ---------------------------------------------
 * Replaces NonUniformBspline::parameterizeToBspline (bspline/src/non_uniform_bspline.cpp:178-265, degree 3), the
 * getBoundaryStates(2, 0) that follows it (:108-123; planner_manager.cpp:308, :561) and the pt_dist_ that
 * BsplineOptimizer::optimize() freezes (bspline_optimizer.cpp:136-140), for B trajectories of K = n_pts - 2 samples.
 *   points [B][n_pts-2][3]  the sampled positions (point_set)
 *   derivs [B][4][3]        start vel, end vel, start acc, end acc (start_end_derivative)
 *   dt [B]                  ts, the knot span of the result
 *   time_lb [B] or NULL     copied to traj[b].time_lb (NULL: -1, none)
 * Outputs, in the solver's layout: x [B][nvar] = the n_pts control points (nvar == 3*n_pts + 1: dt in the last column);
 * traj [B] = pt_dist, knot_span = dt, start = getBoundaryStates(2, 0) start (pos, vel, acc), end[0] = its end position
 * (n_end = 1), time_lb, n_guide = n_waypt = 0, view_idx = -1, every other byte 0.  The control points solve the
 * reference's (K+4) x (K+2) least-squares system (same entries, rows and right-hand sides) by Givens rotations on its
 * band; they agree with an exact solve to about cond(A) * 1e-16 (DESIGN.md 4.7).  Given those control points, every
 * other output equals the reference's fp64 arithmetic bit for bit.  n_pts is 4..FUELGPU_MAX_PTS.
 * Runs on the map's main stream, so parameterize_batch_dev -> fuelgpu_bspline_optimize_batch_dev ->
 * fuelgpu_bspline_check_batch_dev needs no host sync.  Device time: slot 6 of fuelgpu_map_last_timing.
 * The host entry returns FUELGPU_EINVAL and writes nothing when a dt is not finite and positive (the reference prints
 * and returns, :181-184).  The _dev entry cannot read dt before the launch: such a trajectory gets NaN in x and in its
 * pt_dist, knot_span, start and end[0], and the other trajectories are unaffected. */
FUELGPU_API int fuelgpu_bspline_parameterize_batch(FuelMap* map, int32_t B, int32_t n_pts, int32_t nvar,
                                                   const double* points, const double* derivs, const double* dt,
                                                   const double* time_lb, double* x, FuelTrajConst* traj);
FUELGPU_API int fuelgpu_bspline_parameterize_batch_dev(FuelMap* map, int32_t B, int32_t n_pts, int32_t nvar,
                                                       const void* points_dev, const void* derivs_dev, const void* dt_dev,
                                                       const void* time_lb_dev, void* x_dev, void* traj_dev);

/* ---- waypoint polynomial: the head of planExploreTraj on the device ---------------------------------------------------
 * Replaces FastPlannerManager::planExploreTraj's lines 270-297 (plan_manage/src/planner_manager.cpp) for B tours: the
 * segment times (:276-278), PolynomialTraj::waypointsTraj (poly_traj/src/polynomial_traj.cpp:5-175), getTotalTime and
 * getLength (polynomial_traj.h:83-124), seg_num = max(min_seg_num, (int)(length / ctrl_pt_dist)), dt = duration /
 * seg_num (:285-288), the samples at ts = 0, dt, ... while ts <= duration + 1e-4 and the four boundary derivatives
 * (:292-297), laid out as the input of fuelgpu_bspline_parameterize_batch.
 *   n_wp [B]                      waypoints of tour b, 3..FUELGPU_MAX_WAYPTS (S = n_wp - 1 segments)
 *   waypts [B][w_max][3]          the tours, padded to w_max rows
 *   start_vel, start_acc [B][3]   cur_vel, cur_acc
 *   end_vel, end_acc [B][3]       or NULL: zero, what planExploreTraj passes
 *   times [B][w_max-1]            segment times, or NULL: |p[i+1] - p[i]| / (max_vel * 0.5), the norm taken as
 *                                 sqrt((dx*dx + dy*dy) + dz*dz) (Eigen's order is unpinned)
 * Outputs: info [B]; coeffs [B][w_max-1][3][6] or NULL (segment k, axis j: cx[i] multiplies t^i, as
 * Polynomial(cx, cy, cz, T) stores it; rows >= S zero); points [B][FUELGPU_MAX_PTS-2][3] (the K = n_pts - 2 samples,
 * rows >= K zero); derivs [B][4][3] (start vel, end vel, start acc, end acc).
 * The coefficients solve the reference's minimum-jerk problem without its dense inverses (a block-tridiagonal LDL^T in
 * the inner velocities and accelerations, DESIGN.md 4.8); they agree with an exact solve to
 * within 1e-11 relative on the test grid (S up to 31, times 0.05 to 5 s).
 * duration, dt, the sample times, K and the times computed from the waypoints equal the reference's fp64 arithmetic
 * bit for bit; length, the samples and derivs agree to rounding, and so seg_num does except where length /
 * ctrl_pt_dist lies within rounding of an integer.  A tour whose n_pts would exceed FUELGPU_MAX_PTS gets status
 * FUELGPU_POLY_TOO_LONG, its info and coefficients, zero points and its derivs.
 * Tours of two waypoints are refused: the reference's waypointsTraj writes Ct(3, 2S+4) and Ct(5, 2S+5) there, columns 6
 * and 7 of a 6-column matrix; shortenPath (fast_exploration_manager.cpp:321-323) never hands it such a tour.
 * Runs on the map's main stream, so fuelgpu_poly_waypoints_batch_dev -> fuelgpu_bspline_parameterize_batch_dev -> ...
 * needs no host sync except to read info[].n_pts.  Device time: slot 7 of fuelgpu_map_last_timing.
 * The host entry returns FUELGPU_EINVAL and writes nothing when an n_wp is outside 3..FUELGPU_MAX_WAYPTS or above w_max,
 * a segment time (given or computed) is not finite and positive (a repeated waypoint makes A singular), max_vel or
 * ctrl_pt_dist is not finite and positive, or min_seg_num < 1.  The _dev entry checks the parameters alone; a tour with
 * a bad n_wp or time gets status FUELGPU_POLY_BAD_INPUT, NaN in every double it outputs and seg_num = n_pts = 0, and the
 * other tours are unaffected. */
#define FUELGPU_MAX_WAYPTS 32
#define FUELGPU_POLY_TOO_LONG 1
#define FUELGPU_POLY_BAD_INPUT 2
typedef struct {
  double max_vel;      /* pp_.max_vel_: times = |p[i+1]-p[i]| / (max_vel*0.5) when times == NULL (planner_manager.cpp:276-278) */
  double ctrl_pt_dist; /* pp_.ctrl_pt_dist (manager/control_points_distance, 0.35 in algorithm.xml) */
  int32_t min_seg_num; /* 8 in planExploreTraj (:287) */
  int32_t reserved;
} FuelPolyParams;
typedef struct {
  double duration, length, dt; /* getTotalTime, getLength, duration / seg_num */
  int32_t seg_num, n_pts;      /* n_pts = K + 2: the point count to hand to parameterize / optimize / check */
  int32_t status;              /* 0, FUELGPU_POLY_TOO_LONG (n_pts > FUELGPU_MAX_PTS), FUELGPU_POLY_BAD_INPUT (_dev only) */
  int32_t reserved;
} FuelPolyInfo;
FUELGPU_API int fuelgpu_poly_waypoints_batch(FuelMap* map, int32_t B, int32_t w_max, const int32_t* n_wp,
                                             const double* waypts, const double* start_vel, const double* start_acc,
                                             const double* end_vel, const double* end_acc, const double* times,
                                             const FuelPolyParams* params, FuelPolyInfo* info, double* coeffs,
                                             double* points, double* derivs);
FUELGPU_API int fuelgpu_poly_waypoints_batch_dev(FuelMap* map, int32_t B, int32_t w_max, const void* n_wp_dev,
                                                 const void* waypts_dev, const void* start_vel_dev,
                                                 const void* start_acc_dev, const void* end_vel_dev,
                                                 const void* end_acc_dev, const void* times_dev,
                                                 const FuelPolyParams* params, void* info_dev, void* coeffs_dev,
                                                 void* points_dev, void* derivs_dev);

/* ---- exploration yaw: planYawExplore on the device ----------------------------------------------------------------------
 * Replaces FastPlannerManager::planYawExplore(start_yaw, end_yaw, lookfwd, relax_time) (plan_manage/src/
 * planner_manager.cpp:774-865, calcNextYaw :867-885) for every trajectory of a batch in the solver's layout (x [B][nvar]
 * with n_pts 4..FUELGPU_MAX_PTS, dt in the last column when nvar == 3*n_pts + 1, else dt [B]; see the trajectory
 * verdicts above).  Per trajectory: dt_yaw = getTimeSum() / FUELGPU_YAW_SEG_NUM; the start yaw wrapped into [-pi, pi];
 * the look-ahead waypoints atan2 of evaluateDeBoorT(min(duration, tc + 2)) - evaluateDeBoorT(tc) at tc = i * dt_yaw,
 * i = 1 .. 11 - (int)(relax_time / dt_yaw), chained through calcNextYaw; the 15 x 1 initial guess and pt_dist_ that
 * BsplineOptimizer::optimize() freezes from it; and the minimizer of its SMOOTHNESS | START | END | WAYPOINTS objective
 * (combineCost with dim_ == 1, bspline_optimizer.cpp:518-630).  That objective is a strictly convex quadratic: the device
 * solves its normal equations (half-bandwidth 3) by a banded Cholesky factorization in fp64 instead of running NLopt
 * (DESIGN.md 4.9).  dt_yaw and the waypoint count equal the reference's fp64 arithmetic bit for bit; the waypoints agree
 * to atan2's rounding (2 ulp), and given them so do the end yaw, the initial guess and pt_dist.
 *   start_yaw [B][3]   yaw, yawdot, yawddot (finite, |yaw| <= 1000: this library's bound on the reference's wrapping loops)
 *   end_yaw [B]        finite
 *   params             ld_smooth, ld_start, ld_end and ld_waypt are read (ld_smooth and ld_start finite and > 0)
 *   yaw_params         relax_time (finite, >= 0) and lookfwd (0: no waypoints)
 * Outputs: yaw [B][FUELGPU_YAW_PTS] (the yaw control points, knot span info[b].dt_yaw); info [B]; waypt
 * [B][FUELGPU_YAW_MAX_WAYPT] or NULL (waypoint k constrains control points k+1..k+3; zero past n_waypt).
 * Where the reference's behaviour is undefined a trajectory gets a status and NaN yaw.  What the reference computed
 * before that point is written (dt_yaw always; pt_dist, n_waypt and the waypoints for FUELGPU_YAW_ZERO_PT_DIST and
 * FUELGPU_YAW_NOT_SPD), the rest is NaN, n_waypt 0:
 *   FUELGPU_YAW_BAD_INPUT       (_dev only) a dt, start yaw or end yaw the host entry refuses, or dt_yaw not finite and > 0
 *   FUELGPU_YAW_RELAX_OVERFLOW  relax_time / dt_yaw >= 2^31: the reference's int conversion is undefined
 *   FUELGPU_YAW_NO_LOOKAHEAD    the first look-ahead difference is <= 1e-6 m: the reference reads waypts.back() of an
 *                               empty vector
 *   FUELGPU_YAW_ZERO_PT_DIST    pt_dist_ == 0 (all start and end states 0): every cost of the reference is NaN
 *   FUELGPU_YAW_NOT_SPD         a non-positive or non-finite pivot in the factorization
 * Runs on the map's main stream, so fuelgpu_bspline_check_batch_dev -> fuelgpu_yaw_explore_batch_dev needs no host sync.
 * The host entry returns FUELGPU_EINVAL and writes nothing on a bad n_pts or nvar, B < 0, a dt that is not finite and
 * positive, a bad start or end yaw, or a bad parameter; the _dev entry checks the parameters alone and marks a bad
 * trajectory FUELGPU_YAW_BAD_INPUT, leaving the others unaffected.  Not timed in fuelgpu_map_last_timing. */
#define FUELGPU_YAW_SEG_NUM 12
#define FUELGPU_YAW_PTS (FUELGPU_YAW_SEG_NUM + 3)
#define FUELGPU_YAW_MAX_WAYPT (FUELGPU_YAW_SEG_NUM - 1)
#define FUELGPU_YAW_MAX_START 1000.0
#define FUELGPU_YAW_BAD_INPUT 1
#define FUELGPU_YAW_RELAX_OVERFLOW 2
#define FUELGPU_YAW_NO_LOOKAHEAD 3
#define FUELGPU_YAW_ZERO_PT_DIST 4
#define FUELGPU_YAW_NOT_SPD 5
typedef struct {
  double relax_time; /* ep_->relax_time_ (exploration_manager/launch/algorithm.xml: 1.0) */
  int32_t lookfwd;   /* planYawExplore's lookfwd; planExploreMotion passes true */
  int32_t reserved;
} FuelYawParams;
typedef struct {
  double dt_yaw, pt_dist; /* knot span of the yaw spline; pt_dist_ of the initial guess */
  int32_t n_waypt;        /* look-ahead waypoints, 0..FUELGPU_YAW_MAX_WAYPT */
  int32_t status;         /* 0 or FUELGPU_YAW_* */
} FuelYawInfo;
FUELGPU_API int fuelgpu_yaw_explore_batch(FuelMap* map, int32_t B, int32_t n_pts, int32_t nvar, const double* x,
                                          const double* dt, const double* start_yaw, const double* end_yaw,
                                          const FuelOptParams* params, const FuelYawParams* yaw_params, double* yaw,
                                          FuelYawInfo* info, double* waypt);
FUELGPU_API int fuelgpu_yaw_explore_batch_dev(FuelMap* map, int32_t B, int32_t n_pts, int32_t nvar, const void* x_dev,
                                              const void* dt_dev, const void* start_yaw_dev, const void* end_yaw_dev,
                                              const FuelOptParams* params, const FuelYawParams* yaw_params,
                                              void* yaw_dev, void* info_dev, void* waypt_dev);

/* ---- kinodynamic-replan yaw: planYaw on the device ---------------------------------------------------------------------
 * Replaces FastPlannerManager::planYaw(start_yaw) (plan_manage/src/planner_manager.cpp:695-772, calcNextYaw :867-885),
 * the last stage of KinoReplanFSM::callKinodynamicReplan (kino_replan_fsm.cpp:280-300), for every trajectory of a batch
 * in the solver's layout (as fuelgpu_yaw_explore_batch: x [B][nvar], n_pts 4..FUELGPU_MAX_PTS, dt in the last column
 * when nvar == 3*n_pts + 1, else dt [B]).  Per trajectory, with duration = getTimeSum():
 *   seg_num = ceil(duration / 0.3), dt_yaw = duration / seg_num;
 *   waypoint i = 0 .. seg_num - 1: atan2 of evaluateDeBoorT(min(duration, tc + 2)) - evaluateDeBoorT(tc) at
 *   tc = i * dt_yaw, chained through calcNextYaw from start_yaw[0] as given (not wrapped), or the previous waypoint
 *   where |pd| <= 1e-6; waypoint i constrains control points i..i+2;
 *   end yaw: atan2 of the velocity spline (getDerivative(), updateTrajInfo :518-526) at evaluateDeBoorT(duration - 0.1),
 *   clamped to the spline's first knot as evaluateDeBoor does when duration < 0.1, then calcNextYaw;
 *   the (seg_num + 3) x 1 initial guess: states2pts * start_yaw in rows 0-2, states2pts * (end, 0, 0) in rows
 *   seg_num..seg_num+2, written second (for seg_num 1 and 2 the blocks overlap and the end block wins); pt_dist_ of it;
 *   the minimizer of SMOOTHNESS | START | END | WAYPOINTS with three end states (end velocity and acceleration 0, so
 *   calcEndCost's acceleration term is active, bspline_optimizer.cpp:393-431), combineCost with dim_ == 1.
 * Divergences from the reference, as for planYawExplore (DESIGN.md 4.15): the strictly convex quadratic objective is
 * solved by a banded Cholesky factorization in fp64 instead of NLopt (NLopt parity unpinned); |pd| is summed
 * (dx*dx + dy*dy) + dz*dz and states2pts * v left to right per row; the device's atan2 is within 2 ulp of the C
 * library's, so the waypoints agree to that rounding, and given them the end yaw, the initial guess and pt_dist are bit
 * for bit.  seg_num, dt_yaw and the waypoint count equal the reference's fp64 arithmetic bit for bit.
 *   start_yaw [B][3]   yaw, yawdot, yawddot (finite, |yaw| <= FUELGPU_YAW_MAX_START)
 *   params             ld_smooth, ld_start, ld_end and ld_waypt are read (ld_smooth and ld_start finite and > 0)
 * Outputs: yaw [B][FUELGPU_PLANYAW_MAX_PTS] (control points of the yaw spline, knot span info[b].dt_yaw; NaN past
 * seg_num + 3); info [B]; waypt [B][FUELGPU_PLANYAW_MAX_SEG] or NULL (plan_data_.path_yaw_, zero past n_waypt).
 * Where the reference's behaviour is undefined, or the trajectory is longer than this library's cap, a trajectory gets a
 * status and NaN yaw.  What the reference computed before that point is written (seg_num and dt_yaw from
 * FUELGPU_YAW_NO_LOOKAHEAD on; pt_dist, n_waypt and the waypoints for FUELGPU_YAW_ZERO_PT_DIST and FUELGPU_YAW_NOT_SPD),
 * the rest is NaN, seg_num and n_waypt 0:
 *   FUELGPU_YAW_BAD_INPUT       (_dev only) a dt or start yaw the host entry refuses; also (either entry) a duration that
 *                               is not finite and positive (the reference's seg_num is 0 and dt_yaw 0/0)
 *   FUELGPU_YAW_TOO_LONG        duration / 0.3 > FUELGPU_PLANYAW_MAX_SEG (tested before the int conversion)
 *   FUELGPU_YAW_NO_LOOKAHEAD    |pd| <= 1e-6 at i = 0 (a hovering start): the reference reads waypts.back() of an empty
 *                               vector
 *   FUELGPU_YAW_ZERO_PT_DIST    pt_dist_ == 0 (start yaw, rate and acceleration 0 and an end velocity along +x): every
 *                               cost of the reference is NaN
 *   FUELGPU_YAW_NOT_SPD         a pivot that is not finite and positive in the factorization
 * Runs on the map's main stream, so fuelgpu_bspline_optimize_batch_dev -> fuelgpu_plan_yaw_batch_dev needs no host sync.
 * The host entry returns FUELGPU_EINVAL and writes nothing on B < 0, a bad n_pts or nvar, a dt that is not finite and
 * positive, a start yaw that is not finite or has |yaw| > FUELGPU_YAW_MAX_START, or a bad parameter; the _dev entry
 * checks the parameters alone and marks a bad trajectory FUELGPU_YAW_BAD_INPUT, leaving the others unaffected.  Not timed
 * in fuelgpu_map_last_timing. */
#define FUELGPU_PLANYAW_MAX_SEG 128 /* 38.4 s of trajectory at 0.3 s per segment */
#define FUELGPU_PLANYAW_MAX_PTS (FUELGPU_PLANYAW_MAX_SEG + 3)
#define FUELGPU_YAW_TOO_LONG 6
typedef struct {
  double dt_yaw, pt_dist; /* knot span of the yaw spline; pt_dist_ of the initial guess */
  int32_t seg_num;        /* 1..FUELGPU_PLANYAW_MAX_SEG; the yaw spline has seg_num + 3 control points */
  int32_t n_waypt;        /* waypoints (= seg_num when planned) */
  int32_t status;         /* 0 or FUELGPU_YAW_* */
  int32_t reserved;
} FuelPlanYawInfo;
FUELGPU_API int fuelgpu_plan_yaw_batch(FuelMap* map, int32_t B, int32_t n_pts, int32_t nvar, const double* x,
                                       const double* dt, const double* start_yaw, const FuelOptParams* params,
                                       double* yaw, FuelPlanYawInfo* info, double* waypt);
FUELGPU_API int fuelgpu_plan_yaw_batch_dev(FuelMap* map, int32_t B, int32_t n_pts, int32_t nvar, const void* x_dev,
                                           const void* dt_dev, const void* start_yaw_dev, const FuelOptParams* params,
                                           void* yaw_dev, void* info_dev, void* waypt_dev);

/* ---- geometric path to the next viewpoint: Astar::search, shortenPath and the goal branch on the device -------------
 * Replaces, for B (start, goal) queries, the head of FastExplorationManager::planExploreMotion
 * (exploration_manager/src/fast_exploration_manager.cpp:238-263): path_finder_->reset(), Astar::search(pos, next_pos)
 * (path_searching/src/astar2.cpp:47-149) with getPath / backtrack (:177-190), shortenPath (:295-325, dist_thresh 3.0,
 * its ray test the RayCaster walk of the viewpoint visibility), Astar::pathLength (:169-175) and the radius_close = 1.5 /
 * radius_far = 5.0 branch with the far-goal truncation (:253-262).  Every search reads the resident occupancy byte (the
 * inflate bit and the tri-state) with the reference's tests: isInBox, getInflateOccupancy == 1 || getOccupancy ==
 * UNKNOWN, the check points every 0.1 m along each step; A* nodes are keyed by floor((p - origin) / resolution) on the
 * map's origin.  The open set is libstdc++'s std::priority_queue restated over node ids (its stale, re-pushed entries
 * included), so every output equals the reference's fp64 arithmetic bit for bit (DESIGN.md 4.10).
 *   start, goal [B][3]   pos and next_pos (finite)
 *   params               resolution (finite and > 1e-3: the reference's neighbour loop then has its 26 steps),
 *                        lambda_heu (finite), allocate_num (>= 2: the node pool), max_iter (>= 1)
 * The reference's wall-clock cut (max_search_time_) is replaced by an iteration cap: the search ends with NO_PATH at
 * loop iteration max_iter + 1, with early_terminate_cost = g + getDiagHeu(pos, end) of the open set's top.  The open
 * set holds at most 2 * allocate_num entries on the device (the reference's is unbounded): a push beyond that ends the
 * search with NO_PATH and reason FUELGPU_ASTAR_HEAP_FULL, never silently.
 * Outputs: info [B]; path [B][path_max][3] or NULL: getPath() (start ... end node, goal), its first path_max rows, zero
 * past them; waypts [B][w_max][3] and n_wp [B]: the tour planExploreTraj receives (the shortened path for CLOSE and
 * MID, the truncated one for FAR), exactly the input of fuelgpu_poly_waypoints_batch[_dev].  n_wp[b] is the tour's
 * count when tour_status is 0 and 0 otherwise (no path, a tour of fewer than 3 points -- start == goal hands
 * planExploreTraj a single point -- or one longer than FUELGPU_MAX_WAYPTS or w_max); the poly entry's _dev form marks
 * an n_wp of 0 FUELGPU_POLY_BAD_INPUT and leaves the other rows alone, so fuelgpu_astar_batch_dev ->
 * fuelgpu_poly_waypoints_batch_dev -> ... needs no host sync.  A MID tour (1.5 <= length <= 5.0) is written too: the
 * reference calls kinodynamicReplan there instead, which fuelgpu_kino_search_batch_dev runs on exactly these rows.
 * Scratch: one map-owned device buffer, grown on demand: W warps search at once, W = min(B, 32 * SM count,
 * max(1, 4 GiB / S)), with S = 80 * allocate_num + 16 * T + 24 bytes per warp (each array rounded up to 256 bytes), T the
 * least power of two >= max(64, 2 * allocate_num), and 256 bytes more; FUELGPU_ENOMEM if it cannot be allocated.  Runs on the map's main stream;
 * not timed in fuelgpu_map_last_timing.  The host entry returns FUELGPU_EINVAL and writes nothing on a non-finite start
 * or goal or a bad parameter; the _dev entry checks the parameters alone and marks a row with a non-finite start or goal
 * FUELGPU_ASTAR_BAD_INPUT, leaving the other rows unaffected. */
#define FUELGPU_ASTAR_REACH_END 1 /* Astar::REACH_END */
#define FUELGPU_ASTAR_NO_PATH 2   /* Astar::NO_PATH */
/* FuelPathInfo.reason */
#define FUELGPU_ASTAR_FOUND 0
#define FUELGPU_ASTAR_OPEN_EMPTY 1 /* the open set ran empty (:144-148) */
#define FUELGPU_ASTAR_POOL 2       /* use_node_num_ == allocate_num_ right after an allocation (:127-130) */
#define FUELGPU_ASTAR_ITER_CAP 3   /* loop iteration max_iter + 1 (the reference's time cut, :75-79) */
#define FUELGPU_ASTAR_HEAP_FULL 4  /* more than 2 * allocate_num open-set entries (device only) */
#define FUELGPU_ASTAR_BAD_INPUT 5  /* _dev only: a non-finite start or goal */
/* FuelPathInfo.branch (fast_exploration_manager.cpp:243-275) */
#define FUELGPU_ASTAR_NONE 0
#define FUELGPU_ASTAR_CLOSE 1 /* length < 1.5: the whole tour, next_goal = goal */
#define FUELGPU_ASTAR_MID 2   /* otherwise: the reference runs kinodynamicReplan (fuelgpu_kino_search_batch_dev); the
                                 whole tour, next_goal = goal */
#define FUELGPU_ASTAR_FAR 3   /* length > 5.0: the tour truncated past 5 m, next_goal = its last point */
/* FuelPathInfo.tour_status */
#define FUELGPU_ASTAR_TOO_LONG 1   /* more than FUELGPU_MAX_WAYPTS or w_max points */
#define FUELGPU_ASTAR_DEGENERATE 2 /* fewer than 3 points */
typedef struct {
  double resolution;    /* astar/resolution_astar */
  double lambda_heu;    /* astar/lambda_heu */
  int32_t allocate_num; /* astar/allocate_num: the node pool */
  int32_t max_iter;     /* stands for astar/max_search_time: loop iterations instead of seconds */
} FuelAstarParams;
typedef struct {
  int32_t status;       /* FUELGPU_ASTAR_REACH_END or FUELGPU_ASTAR_NO_PATH */
  int32_t reason;       /* FUELGPU_ASTAR_FOUND ... FUELGPU_ASTAR_BAD_INPUT */
  int32_t iter_num, use_node_num, n_path; /* iter_num_, use_node_num_, getPath().size() */
  int32_t n_wp;         /* points of the tour (0 without a path) */
  int32_t branch;       /* FUELGPU_ASTAR_NONE / CLOSE / MID / FAR */
  int32_t tour_status;  /* 0, FUELGPU_ASTAR_TOO_LONG, FUELGPU_ASTAR_DEGENERATE */
  double early_terminate_cost; /* getEarlyTerminateCost() after FUELGPU_ASTAR_ITER_CAP, else 0 */
  double length;               /* pathLength of the shortened path (0 without a path) */
  double next_goal[3];         /* ed_->next_goal_ (0 without a path) */
} FuelPathInfo;
FUELGPU_API int fuelgpu_astar_batch(FuelMap* map, int32_t B, const double* start, const double* goal,
                                    const FuelAstarParams* params, FuelPathInfo* info, int32_t path_max, double* path,
                                    int32_t w_max, int32_t* n_wp, double* waypts);
FUELGPU_API int fuelgpu_astar_batch_dev(FuelMap* map, int32_t B, const void* start_dev, const void* goal_dev,
                                        const FuelAstarParams* params, void* info_dev, int32_t path_max, void* path_dev,
                                        int32_t w_max, void* n_wp_dev, void* waypts_dev);

/* ---- kinodynamic path to a mid-range goal: kinodynamicReplan's search on the device --------------------------------
 * Replaces, for B queries, FastPlannerManager::kinodynamicReplan(start, vel, acc, goal, 0, time_lb) up to its
 * parameterization (plan_manage/src/planner_manager.cpp:131-164): the "Close goal" refusal (|start - goal| < 1e-2),
 * KinodynamicAstar::reset and the non-dynamic search(start, vel, acc, goal, 0, init = true) with the retry at
 * init = false after NO_PATH (path_searching/src/kinodynamic_astar.cpp:15-263), computeShotTraj and getSamples at
 * ts = ctrl_pt_dist / manager_max_vel, laid out as the input of fuelgpu_bspline_parameterize_batch[_dev] (with the
 * caller's time_lb).  Every search reads the resident occupancy byte with the reference's tests: isInBox, the inflate bit,
 * UNKNOWN unless optimistic; the shot's samples are bounded by origin below and by the map's SIZE above (the reference's
 * getRegion) and tested against the inflate bit alone.  Nodes are keyed by floor((p - origin) / resolution) on the map's
 * origin; the open set is libstdc++'s std::priority_queue restated over node ids, compared through each node's current
 * f_score.  Arithmetic (DESIGN.md 4.14): the search's powers are host tables of 0.5 * pow(t, 2) computed with the host's
 * pow in the reference's loops, and cbrt is glibc's routine restated, so the search equals the reference's glibc build
 * bit for bit except where cubic()'s three-real-root branch (D < 0) runs: there acos and cos are correctly rounded.  Outside
 * the search (the shot and getSamples) pow(t, 2) and pow(t, 3) are correctly rounded.
 *   start, vel, acc, goal [B][3]   finite; end_v is 0, as planExploreMotion passes it
 *   params                        the search/ parameters (max_vel without vel_margin: the search adds it), ctrl_pt_dist and
 *                                 manager_max_vel (pp_.max_vel_).  The duration and acceleration lists follow the
 *                                 reference's loops; at most 32 init durations and 8 steps per axis (the loop of
 *                                 the other durations always yields max_tau alone).
 * Outputs: info [B]; points [B][FUELGPU_MAX_PTS-2][3] (the K = n_pts - 2 samples of getSamples, rows >= K zero); derivs
 * [B][4][3] (start vel, end vel, start acc, end acc); dt [B] (getSamples' ts; NaN without samples, so that
 * fuelgpu_bspline_parameterize_batch_dev marks the row); nodes [B][node_max][12] or NULL (state, input, duration, g, f of
 * the path root .. end node; the root's input and duration 0); shot [B][3][4] or NULL (coef_shot_, zero without a shot).
 * A path of more than FUELGPU_MAX_PTS - 2 samples gets traj_status FUELGPU_KINO_TOO_LONG and no samples.
 * The _dev entry takes gate, the info of fuelgpu_astar_batch_dev, or NULL: rows whose branch is not FUELGPU_ASTAR_MID get
 * status FUELGPU_KINO_SKIPPED, so astar_batch_dev -> kino_search_batch_dev -> parameterize_batch_dev needs no host sync
 * except to read info[].n_pts.  A node pool of allocate_num per search; use_node_num_ reaching it ends the search with
 * NO_PATH, reason FUELGPU_KINO_POOL.
 * Scratch: one map-owned device buffer, grown on demand: W warps search at once, W = min(B, 32 * SM count,
 * max(1, 4 GiB / S)), S about 153 * allocate_num + 56 KiB per warp; FUELGPU_ENOMEM if it cannot be allocated.  Runs on the
 * map's main stream; not timed in fuelgpu_map_last_timing.  The host entry returns FUELGPU_EINVAL and writes nothing on a
 * non-finite input or a bad parameter; the _dev entry checks the parameters alone and marks a row with a non-finite input
 * FUELGPU_KINO_BAD_INPUT, leaving the other rows unaffected. */
/* FuelKinoInfo.status: KinodynamicAstar's codes for the attempt that counted, then the rows not searched */
#define FUELGPU_KINO_REACH_HORIZON 1
#define FUELGPU_KINO_REACH_END 2
#define FUELGPU_KINO_NO_PATH 3
#define FUELGPU_KINO_NEAR_END 4
#define FUELGPU_KINO_SKIPPED 5   /* _dev with gate: not a MID row */
#define FUELGPU_KINO_BAD_INPUT 6 /* _dev only: a non-finite start, vel, acc or goal */
/* FuelKinoInfo.reason */
#define FUELGPU_KINO_FOUND 0
#define FUELGPU_KINO_OPEN_EMPTY 1     /* the open set ran empty (:259-262) */
#define FUELGPU_KINO_POOL 2           /* use_node_num_ == allocate_num_ right after an allocation (:235-239) */
#define FUELGPU_KINO_START_NEAR_END 3 /* the start node lies within the goal tolerance and has no shot (:90-93) */
#define FUELGPU_KINO_CLOSE_GOAL 4     /* |start - goal| < 1e-2: kinodynamicReplan returns before searching */
/* FuelKinoInfo.traj_status */
#define FUELGPU_KINO_TOO_LONG 1 /* more than FUELGPU_MAX_PTS - 2 samples */
#define FUELGPU_KINO_NO_TRAJ 2  /* no samples: NO_PATH, skipped or bad input */
typedef struct {
  double max_tau, init_max_tau; /* search/max_tau, search/init_max_tau */
  double max_vel, vel_margin;   /* search/max_vel, search/vel_margin: the search's max_vel_ is their sum */
  double max_acc, w_time, horizon, lambda_heu;
  double resolution;            /* search/resolution_astar */
  double ctrl_pt_dist;          /* manager/control_points_distance */
  double manager_max_vel;       /* manager/max_vel: ts = ctrl_pt_dist / manager_max_vel */
  int32_t allocate_num, check_num, optimistic, reserved;
} FuelKinoParams;
typedef struct {
  int32_t status, reason, retried, traj_status; /* retried: the init = false search ran */
  int32_t iter_num, use_node_num;               /* iter_num_, use_node_num_ after the attempt that counted */
  int32_t n_nodes, shot;                        /* path_nodes_.size(), is_shot_succ_ */
  int32_t seg_num, n_pts;                       /* getSamples' seg_num; n_pts = K + 2 (0 without samples) */
  double t_shot, T_sum;
} FuelKinoInfo;
FUELGPU_API int fuelgpu_kino_search_batch(FuelMap* map, int32_t B, const double* start, const double* vel,
                                          const double* acc, const double* goal, const FuelKinoParams* params,
                                          FuelKinoInfo* info, double* points, double* derivs, double* dt,
                                          int32_t node_max, double* nodes, double* shot);
FUELGPU_API int fuelgpu_kino_search_batch_dev(FuelMap* map, int32_t B, const void* start_dev, const void* vel_dev,
                                              const void* acc_dev, const void* goal_dev, const void* gate_dev,
                                              const FuelKinoParams* params, void* info_dev, void* points_dev,
                                              void* derivs_dev, void* dt_dev, int32_t node_max, void* nodes_dev,
                                              void* shot_dev);

/* ---- tour cost between viewpoints: ViewNode::searchPath and ViewNode::computeCost on the device -------------------
 * For P pairs (p1, p2, y1, y2, v1), what ViewNode::computeCost(p1, p2, y1, y2, v1, 0, path)
 * (active_perception/src/graph_node.cpp:63-85) returns and the path ViewNode::searchPath (:32-61) leaves: the edge cost
 * of FrontierFinder::updateFrontierCostMatrix (frontier_finder.cpp:260-326, v1 = 0) and of getFullCostMatrix's first
 * row (:562-591, v1 = the current velocity).  Per pair:
 *   1. the straight line p1 -> p2: the RayCaster walk of the viewpoint visibility (input, then nextId until the end
 *      voxel), blocked by an inflated-occupied, UNKNOWN or outside-the-box voxel (!isInBox(idx)).  Clear: kind LINE,
 *      path {p1, p2}, length (p1 - p2).norm().  Like every ray walk of this library it gives up after 4096 voxels and
 *      counts the line clear (the reference's loop has no bound);
 *   2. a blocked line: Astar::search(p1, p2) at params->astar (as fuelgpu_astar_batch searches, iteration cap and all;
 *      the reference sets resolution 0.4).  REACH_END: kind ASTAR, path getPath() (start ... end node, goal; no
 *      shortenPath), length Astar::pathLength of it.  Otherwise kind NO_PATH, path {p1, p2}, length 1000;
 *   3. cost = max(length / vm [+ w_dir * acos(v1.normalized() . (p2 - p1).normalized()) when |v1| > 1e-3],
 *      min(|y2 - y1|, 2 pi - |y2 - y1|) / yd), std::max's NaN behaviour included.
 * Every output but cost equals the reference's fp64 arithmetic bit for bit; cost too wherever |v1| <= 1e-3.  acos is
 * the device's (within 2 ulp of the correctly rounded value), so with a velocity the cost may differ in its last bits.
 *   p1, p2, v1 [P][3], y1, y2 [P]; params: vm, yd finite and > 0, w_dir finite, astar as fuelgpu_astar_batch checks it
 * Outputs: info [P]; path [P][path_max][3] or NULL: its first path_max rows, zero past them.  A row with a non-finite
 * input gets kind 0, reason FUELGPU_ASTAR_BAD_INPUT and zeros; the other rows are unaffected (both entries).
 * Scratch: the search's (fuelgpu_astar_batch) with the node pool clamped to min(allocate_num, 26 * max_iter + 2) -- a
 * search never uses more, so the results are those of allocate_num -- plus about 256 + 76 * P bytes.  Runs on the map's main
 * stream with no host synchronisation inside (the search reads the blocked pairs' count from device memory); the host
 * entry waits once, at the end. */
#define FUELGPU_VIEW_LINE 1    /* the straight line is clear */
#define FUELGPU_VIEW_ASTAR 2   /* the line is blocked, A* reached the goal */
#define FUELGPU_VIEW_NO_PATH 3 /* the line is blocked, A* did not reach it: length 1000 */
typedef struct {
  double vm, yd, w_dir;  /* ViewNode::vm_, yd_, w_dir_ (exploration/vm, exploration/yd, exploration/w_dir) */
  FuelAstarParams astar; /* ViewNode::astar_: the astar/ parameters, resolution as searchPath sets it (0.4) */
} FuelViewCostParams;
typedef struct {
  int32_t kind;                     /* FUELGPU_VIEW_LINE / ASTAR / NO_PATH, 0 on a bad row */
  int32_t reason;                   /* the search's FuelPathInfo.reason (ASTAR, NO_PATH), FUELGPU_ASTAR_BAD_INPUT */
  int32_t iter_num, use_node_num;   /* the search's (ASTAR, NO_PATH), else 0 */
  int32_t n_path, reserved;         /* path.size() */
  double length;                    /* searchPath's return value */
  double cost;                      /* computeCost's return value */
} FuelViewCostInfo;
FUELGPU_API int fuelgpu_view_cost_batch(FuelMap* map, int32_t P, const double* p1, const double* p2, const double* y1,
                                        const double* y2, const double* v1, const FuelViewCostParams* params,
                                        FuelViewCostInfo* info, int32_t path_max, double* path);
FUELGPU_API int fuelgpu_view_cost_batch_dev(FuelMap* map, int32_t P, const void* p1_dev, const void* p2_dev,
                                            const void* y1_dev, const void* y2_dev, const void* v1_dev,
                                            const FuelViewCostParams* params, void* info_dev, int32_t path_max,
                                            void* path_dev);

/* ---- local tour refinement: FastExplorationManager::refineLocalTour on the device ---------------------------------
 * B independent refineLocalTour(cur_pos, cur_vel, cur_yaw, n_points, n_yaws, refined_pts, refined_yaws) problems
 * (exploration_manager/src/fast_exploration_manager.cpp:429-503).  Problem b has groups prob_off[b] .. prob_off[b+1]
 * (n_points / n_yaws, in order); group g has viewpoints vp_pos / vp_yaw [group_off[g] .. group_off[g+1]).  As the
 * reference builds it: node 0 is the current state (vel_ = cur_vel, yaw cur_yaw[b]), every viewpoint of a group is a
 * node with zero velocity, except that the last group keeps only its first viewpoint (final_node); each node of a group
 * has an edge from every node of the group before (node 0 for the first group), in addEdge order: group, new node,
 * then previous-group node.  Each edge costs ViewNode::computeCost (fuelgpu_view_cost_batch, eagerly, all at once);
 * DijkstraSearch (graph_search.h:76-118) then runs over that table exactly as the reference's std::priority_queue does
 * it (g_value_ from 1e6, strict <, neighbours in order, stale entries popped and expanded again).  refined holds the
 * viewpoints of path[1..] as indices into vp_*; the tour is ed_->refined_tour_: cur_pos, then for each refined point
 * ViewNode::searchPath from the tour's end with astar.lambda_heu = tour_lambda_heu, its path appended when searchPath
 * returns nonzero (NaN and 1000 included), the point alone otherwise.
 * The reference evaluates costTo lazily, as Dijkstra expands nodes; costTo is a pure function of its pair, so every
 * output is the reference's given the same edge costs.  n_evals is the number of costTo calls the reference makes.
 * Divergences are those of fuelgpu_view_cost_batch: the iteration cap for max_search_time, the 4096-voxel ray guard,
 * and the device's acos on node 0's edges when |cur_vel| > 1e-3 (g may then differ in its last bits).
 *   prob_off [B + 1], group_off [G + 1]: HOST memory in both entries, starting at 0 and nondecreasing.
 *   cur_pos, cur_vel [B][3], cur_yaw [B], vp_pos [N][3], vp_yaw [N]: host arrays, device pointers in _dev.
 *   params: view as fuelgpu_view_cost_batch checks it (resolution 0.4 as searchPath sets it), tour_lambda_heu finite
 *   (refineLocalTour sets 1.0 for the tour's searches).
 * Outputs (host arrays, device pointers in _dev): info [B]; refined [B][kmax], -1 past n_refined; tour
 * [B][tour_max][3], zero past n_tour; edge_cost [E] or NULL: every edge's cost in addEdge order, problem by problem.
 * Status per problem:
 *   FUELGPU_TOUR_OK;
 *   FUELGPU_TOUR_UNREACHABLE: the open set ran empty before final_node was popped (an empty middle group, or edges of
 *     NaN or >= 1e6 cost): n_refined 0, g 1e6, tour [cur_pos] -- the reference then indexes refined_points_[0], which
 *     is undefined behaviour;
 *   FUELGPU_TOUR_BAD_INPUT: a non-finite cur_pos / cur_vel / cur_yaw or graph node coordinate: everything zero, refined
 *     -1; the other problems are unaffected.  Its tour segments go to the searches as non-finite rows, which cost none;
 *   FUELGPU_TOUR_TRUNCATED: as OK, but the tour needs n_tour > tour_max rows; the first tour_max are written.  Call
 *     again with tour_max >= n_tour.
 * FUELGPU_EINVAL, nothing written: B < 0, a problem with no group or an empty last group (the reference dereferences a
 * null final_node), more than FUELGPU_TOUR_MAX_NODES nodes or more than kmax groups in one problem, tour_max < 1, a
 * bad parameter or a null argument.
 * Runs on the map's main stream with no host synchronisation inside: the edge enumeration, the edge costs
 * (fuelgpu_view_cost_batch's three launches), the search (one warp per problem), the tour's segment costs (again the
 * view-cost launches), the tour assembly.  The host entry waits once, at the end.
 * Scratch: one map-owned device buffer grown on demand, about 164 E + 16 N' + 28 B + 188 G + 24 G tour_max bytes
 * (E edges, N' graph nodes, G groups), plus the view-cost scratch of fuelgpu_view_cost_batch. */
#define FUELGPU_TOUR_MAX_NODES 1024
#define FUELGPU_TOUR_OK 0
#define FUELGPU_TOUR_UNREACHABLE 1
#define FUELGPU_TOUR_BAD_INPUT 2
#define FUELGPU_TOUR_TRUNCATED 3
typedef struct {
  FuelViewCostParams view; /* ViewNode's statics: the edge costs and the tour's searches */
  double tour_lambda_heu;  /* ViewNode::astar_->lambda_heu_ for the tour's searches (refineLocalTour :490: 1.0) */
} FuelLocalTourParams;
typedef struct {
  int32_t status;          /* FUELGPU_TOUR_OK ... FUELGPU_TOUR_TRUNCATED */
  int32_t n_nodes, n_edges; /* the graph's node_num_ and edge_num_ */
  int32_t n_evals;         /* costTo calls the reference's lazy search makes */
  int32_t n_refined;       /* refined_pts.size() */
  int32_t n_tour;          /* ed_->refined_tour_.size() (the rows needed when TRUNCATED) */
  int32_t pops, pushes;    /* open-set pops and pushes (the start's push included) */
  double g;                /* final_node's g_value_ */
} FuelLocalTourInfo;
FUELGPU_API int fuelgpu_local_tour_batch(FuelMap* map, int32_t B, const int32_t* prob_off, const int32_t* group_off,
                                         const double* cur_pos, const double* cur_vel, const double* cur_yaw,
                                         const double* vp_pos, const double* vp_yaw, const FuelLocalTourParams* params,
                                         FuelLocalTourInfo* info, int32_t kmax, int32_t* refined, int32_t tour_max,
                                         double* tour, double* edge_cost);
FUELGPU_API int fuelgpu_local_tour_batch_dev(FuelMap* map, int32_t B, const int32_t* prob_off,
                                             const int32_t* group_off, const void* cur_pos_dev,
                                             const void* cur_vel_dev, const void* cur_yaw_dev, const void* vp_pos_dev,
                                             const void* vp_yaw_dev, const FuelLocalTourParams* params,
                                             void* info_dev, int32_t kmax, void* refined_dev, int32_t tour_max,
                                             void* tour_dev, void* edge_cost_dev);

/* ---- global tour: the ATSP of FastExplorationManager::findGlobalTour, solved exactly on the device -----------------
 * findGlobalTour (exploration_manager/src/fast_exploration_manager.cpp:327-427) writes getFullCostMatrix's
 * (n + 1) x (n + 1) matrix as a TSPLIB ATSP, solves it with LKH and reads the tour back.  These entries solve the same
 * problem for B instances exactly (Held-Karp dynamic programming over subsets), so no tour is worse than LKH's.
 * Instance b has dimension d_b = dims[b] = n + 1: node 0 is the current state, nodes 1 .. n the clusters; its matrix
 * is d_b x d_b row-major doubles in `cost`, the instances concatenated.
 *   - Integer costs as the reference makes them: int(cost(i, j) * 100), the double product truncated toward zero
 *     (:357-376).  The diagonal is never read.
 *   - Objective: LKH's cycle cost c[0][t1] + c[t1][t2] + ... + c[tn][0], summed in int64.  getFullCostMatrix's column 0
 *     is zero, so in FUEL this is the open tour from the current state.
 *   - Output: indices (the instance's n entries in the concatenation) are the 0-based cluster ids t1 - 1 .. tn - 1, as
 *     findGlobalTour pushes id - 2 for LKH's 1-based node id.  Among optimal tours, the lexicographically smallest
 *     sequence.  info.cost is the optimal cost, info.n_optimal the number of optimal tours (saturating at INT32_MAX).
 *   - n = 1 gives [0] (the reference calls findGlobalTour only for more than one cluster; LKH rejects dimension < 3).
 * Status per instance; the others are unaffected:
 *   FUELGPU_GTOUR_OK;
 *   FUELGPU_GTOUR_BAD_INPUT: an off-diagonal product that is NaN, infinite or whose truncation does not fit int32
 *     (undefined behaviour in the reference's conversion);
 *   FUELGPU_GTOUR_TOO_LARGE: n > FUELGPU_GTOUR_MAX_CLUSTERS; such a caller keeps LKH.
 *   For both, info holds only status and n, and the indices are -1.
 * FUELGPU_EINVAL, nothing written: B < 0, a dims[b] < 2 (n < 1), or a null argument while B > 0.
 *   dims [B]: HOST memory in both entries, so the host sizes everything without a read-back.
 *   cost [sum d_b^2], info [B], indices [sum (d_b - 1)]: host arrays, device pointers in _dev.
 * Runs on the map's main stream with no host synchronisation inside; the host entry waits once, at the end.  Scratch:
 * one map-owned device buffer grown on demand: a 32 B descriptor and a 4 B status per instance (each array rounded up
 * to 256 B), plus, per group of instances, the sum of 4 (n+1)^2 + 12 n 2^n bytes per instance (each part rounded up to
 * 256 B; about 252 MB at n = 20, 2.8 MB at n = 14), groups of at most 4 GiB. */
#define FUELGPU_GTOUR_MAX_CLUSTERS 20
#define FUELGPU_GTOUR_OK 0
#define FUELGPU_GTOUR_BAD_INPUT 1
#define FUELGPU_GTOUR_TOO_LARGE 2
typedef struct {
  int32_t status;    /* FUELGPU_GTOUR_OK ... FUELGPU_GTOUR_TOO_LARGE */
  int32_t n;         /* clusters: dims[b] - 1 */
  int32_t n_optimal; /* optimal tours, saturating at INT32_MAX */
  int32_t reserved;  /* 0 */
  int64_t cost;      /* the optimal tour's cost in the integer units above */
} FuelGlobalTourInfo;
FUELGPU_API int fuelgpu_global_tour_batch(FuelMap* map, int32_t B, const int32_t* dims, const double* cost,
                                          FuelGlobalTourInfo* info, int32_t* indices);
FUELGPU_API int fuelgpu_global_tour_batch_dev(FuelMap* map, int32_t B, const int32_t* dims, const void* cost_dev,
                                              void* info_dev, void* indices_dev);

/* ---- multi-GPU: the z-sharded ESDF update (BASELINE config 4; SURVEY 8e row 1) ---------------------------
 * Multi-GPU form of SDFMap::updateESDF3d (plan_env/src/sdf_map.cpp:152-241) over the whole map.  One process
 * (or thread) per GPU; rank r owns planes [r*nz/G, (r+1)*nz/G) of every (x,y) column, z fastest like the
 * reference (sdf_map.h:145-147).  NCCL is called from inside the library (bound at run time with dlopen, no
 * link-time dependency).  Bootstrap like any NCCL application: rank 0 calls fuelgpu_comm_get_unique_id, the
 * host program ships the 128 bytes to the other ranks (ROS topic, MPI, torch.distributed, a file), every rank
 * calls fuelgpu_comm_init.  nx and nz must be multiples of 32 * ranks. */
typedef struct FuelComm FuelComm;
typedef struct FuelShardedEsdf FuelShardedEsdf;
FUELGPU_API int fuelgpu_comm_get_unique_id(uint8_t id[128]);
FUELGPU_API int fuelgpu_comm_init(int32_t nranks, int32_t rank, const uint8_t id[128], int32_t device_id, FuelComm** out);
FUELGPU_API int fuelgpu_comm_info(const FuelComm* comm, int32_t* nranks, int32_t* rank);
FUELGPU_API int fuelgpu_comm_destroy(FuelComm* comm);
FUELGPU_API int fuelgpu_sharded_esdf_create(FuelComm* comm, const int32_t n[3], double resolution, FuelShardedEsdf** out);
/* occ_slab_dev: [nx][ny][nz/G] occupancy byte of this rank (bits0-1 tri-state, bit2 inflate, as the resident
 * byte of a FuelMap); dist_slab_dev: [nx][ny][nz/G] float32 metres out (+inf where the map has no site).
 * flags: FUELGPU_ESDF_OPTIMISTIC or 0.  Collective: every rank of the communicator must call it.  Enqueued on
 * cuda_stream (plus an internal stream for the exchange rounds); returns without waiting. */
FUELGPU_API int fuelgpu_sharded_esdf_update(FuelShardedEsdf* s, void* cuda_stream, const void* occ_slab_dev, int flags,
                                            void* dist_slab_dev);
/* device times (ms) of the last update on this rank: [0] occupancy exchange, [1] z records + zy tiles (the
 * exchange rounds of the 2-D partial overlap them), [2] wait for the last rounds, [3] x tiles, [4] total */
FUELGPU_API int fuelgpu_sharded_esdf_last_timing(FuelShardedEsdf* s, float ms[5]);
FUELGPU_API int64_t fuelgpu_sharded_esdf_bytes_exchanged(const FuelShardedEsdf* s);
/* 1 when the 2-D partial travels by direct stores of the zy tile kernels into the peers' receive buffers (CUDA-IPC
 * mapped at creation; one process per GPU, peer access available), 0 when it goes through ncclSend/ncclRecv rounds
 * (FUELGPU_SHARDED_P2P=0 or no peer mapping).  In the peer-memory mode fuelgpu_sharded_esdf_destroy is collective. */
FUELGPU_API int fuelgpu_sharded_esdf_uses_peer_memory(const FuelShardedEsdf* s);
/* every rank gets all z-slabs: out_dev [G][nx][ny][nz/G] float32 (what a trajectory batch split over the ranks
 * samples, SURVEY 8e row 3) */
FUELGPU_API int fuelgpu_sharded_esdf_allgather(FuelShardedEsdf* s, void* cuda_stream, const void* dist_slab_dev,
                                               void* out_dev);
FUELGPU_API int fuelgpu_sharded_esdf_destroy(FuelShardedEsdf* s);
/* Replace the map's distance_buffer_ by a field computed elsewhere: n_slabs == 1: slabs_dev is [nx][ny][nz] float32;
 * n_slabs == G: slabs_dev is the all-gather buffer [G][nx][ny][nz/G] of fuelgpu_sharded_esdf_allgather.  Device to
 * device on the map's stream.  This is the "broadcast the ESDF once" step of a planner that splits its trajectory
 * batch over several GPUs (SURVEY 8e row 3; precedent: the reference's per-thread optimizers share one read-only map,
 * plan_manage/src/planner_manager.cpp:444-453). */
FUELGPU_API int fuelgpu_esdf_set_from_slabs_dev(FuelMap* map, const void* slabs_dev, int32_t n_slabs);
#define FUELGPU_EDT_INF 0x3fffffff

/* Library / device info.  Fills name with the device name; returns the SM count or <0. */
FUELGPU_API int fuelgpu_device_info(int device_id, char* name, int name_len, int* cc_major, int* cc_minor);
FUELGPU_API const char* fuelgpu_version(void);

#ifdef __cplusplus
}
#endif
#endif /* FUELGPU_H */
