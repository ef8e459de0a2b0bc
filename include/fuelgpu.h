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
 * handle's stream): [0] esdf_update [1] frontier_search [2] bspline batch [3] upload [4] download */
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
 * buffer is valid after fuelgpu_map_synchronize().  Use with a page-locked buffer. */
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
 * control point per lane, above that two per lane (and f_best is then exactly what fuelgpu_bspline_cost_batch returns
 * for the returned x). */
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
