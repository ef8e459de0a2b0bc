// common.cuh -- shared state and helpers of libfuelgpu (sm_90a only).
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include <vector>
#ifdef FUEL_PROF
#include <chrono>
#endif

#include "fuelgpu.h"

#define FUELGPU_EDT_INF_I 0x3fffffff

// Grid geometry as the kernels see it (plain, passed by value).
struct Geom {
  int nx, ny, nz;
  double res, res_inv;
  double origin[3];
  double map_max[3];  // map_origin_ + map_size_ (map_max_boundary_, sdf_map.cpp:34-39)
  int box_min[3];     // posToIndex(box_mind_), sdf_map.cpp:83
  int box_max[3];     // posToIndex(box_maxd_), sdf_map.cpp:84
  double box_mind[3], box_maxd[3];
};

enum { T_ESDF = 0, T_FRONTIER = 1, T_BSPLINE = 2, T_UPLOAD = 3, T_DOWNLOAD = 4, T_CHECK = 5, T_PARAM = 6, T_POLY = 7, T_COUNT = 8 };

struct FrontierState;  // frontier.cu
struct FusionState;    // fusion.cu
struct FuelMap;

// A scratch block that grows on demand: device memory, or page-locked host memory when Pinned.  Growing first waits
// for the whole device, since any stream may still use the old block; steady-state calls never wait.
template <typename T, bool Pinned = false>
struct DevBuf {
  T* p = nullptr;
  size_t cap = 0;  // elements
  // at least n elements at p; *grew (if given) tells whether the block was replaced (its contents are then undefined)
  int ensure(FuelMap* m, size_t n, bool* grew = nullptr);
  void release() {
    if (p) Pinned ? cudaFreeHost(p) : cudaFree(p);
    p = nullptr;
    cap = 0;
  }
};

struct FuelMap {
  FuelGridDesc desc;
  Geom g;
  int dev;
  int sm_count;
  int64_t nvox;
  // resident volumes
  uint8_t* occ;     // bits0-1 tri-state, bit2 inflate
  float* dist;      // distance_buffer_ (metres)
  float* dist_neg;  // distance_buffer_neg_ (lazy, signed mode only)
  int8_t* flag;     // frontier_flag_
  // ESDF scratch (esdf_tile.cu): z records, two chunk buffers of the 2-D partial, second stream
  void* esdf_rec;
  void* esdf_p[2];
  size_t esdf_p_bytes;
  cudaStream_t esdf_aux;
  cudaEvent_t esdf_ev[2];
  // Grow-on-demand scratch.  Each block belongs to one stream (or one pending call); calls that may overlap never
  // share a block.
  DevBuf<uint8_t> stage;  // main-stream ingest and downloads
  cudaStream_t own_stream, stream;
  cudaStream_t copy_stream;  // D2H mirror copies that may overlap the main stream
  cudaEvent_t copy_ev;
  bool dist_ev_ok;           // ev1[T_ESDF] marks the last write of `dist` (a mirror download waits on it, not on later work)
  cudaEvent_t mirror_ev;     // end of the last mirror download on copy_stream: writers of `dist` on the main stream wait for it
  bool mirror_pending;
  cudaStream_t in_stream;    // H2D of the solver inputs: goes out at once, not behind the ESDF kernels of the main stream
  cudaEvent_t in_ev;
  cudaEvent_t ev0[T_COUNT], ev1[T_COUNT];
  bool ev_valid[T_COUNT];
  FrontierState* fs;
  FusionState* fus;  // lazily created by the first fusion call
  DevBuf<uint8_t> bs_buf;       // host-facing cost / optimize calls (owned by a pending optimize_batch_begin)
  DevBuf<uint8_t, true> bs_pin;  // their page-locked bounce buffer
  DevBuf<double> bs_grad;  // gradient output of the faithful re-evaluation after the long-trajectory solver (discarded)
  DevBuf<uint8_t> fr_scr;  // small frontier-stream calls (is_changed, viewpoints, clear_flags)
  int bs_pend_B, bs_pend_nvar;  // optimize_batch_begin issued, _end outstanding (B == 0: none)
  size_t bs_pend_off;           // offset of the result block inside bs_pin
  long long launches;  // kernels launched so far
  char err[512];
  DevBuf<uint8_t> tc_buf;  // the other host-facing batch calls (check, evaluate, parameterize, poly, yaw, A*, esdf_sample)
  DevBuf<uint8_t> as_buf;  // A* search scratch (astar.cu)
  DevBuf<uint8_t> vc_buf;  // view cost: the blocked-line list and the searches' results (view_cost.cu)
  DevBuf<uint8_t> lt_buf;  // local tour: the graph, its edges and their costs, the search state, the tour segments
  DevBuf<uint8_t> gt_buf;  // global tour: the instance table and the Held-Karp tables of one group (global_tour.cu)
  size_t as_stride, as_warps;  // layout whose key tables are known empty: per-warp bytes, warps
  DevBuf<uint8_t> ks_buf;      // kinodynamic search scratch (kino_astar.cu)
  size_t ks_stride, ks_warps;  // its layout whose key tables are known empty
#ifdef FUEL_PROF
  double end_prof_us[3];  // the last fuelgpu_frontier_search_end: stream wait, result assembly, closing event (host µs)
#endif
};

extern thread_local char g_fuelgpu_err[512];

static inline int fuel_fail(FuelMap* m, int code, const char* fmt, const char* a = "", long long b = 0) {
  char* dst = m ? m->err : g_fuelgpu_err;
  snprintf(dst, 512, fmt, a, b);
  return code;
}

#define FUEL_CUDA(m, expr)                                                                     \
  do {                                                                                         \
    cudaError_t _e = (expr);                                                                   \
    if (_e != cudaSuccess) {                                                                   \
      char* _dst = (m) ? ((FuelMap*)(m))->err : g_fuelgpu_err;                                 \
      snprintf(_dst, 512, "CUDA error %s at %s:%d: %s", cudaGetErrorName(_e), __FILE__,        \
               __LINE__, cudaGetErrorString(_e));                                              \
      return _e == cudaErrorMemoryAllocation ? FUELGPU_ENOMEM : FUELGPU_ECUDA;                 \
    }                                                                                          \
  } while (0)

template <typename T, bool Pinned>
int DevBuf<T, Pinned>::ensure(FuelMap* m, size_t n, bool* grew) {
  if (grew) *grew = false;
  if (n <= cap) return 0;
  if (p) {
    FUEL_CUDA(m, cudaDeviceSynchronize());
    release();
  }
  const size_t want = n + n / 4 + 1024;
  T* q = nullptr;
  FUEL_CUDA(m, Pinned ? cudaMallocHost((void**)&q, want * sizeof(T)) : cudaMalloc((void**)&q, want * sizeof(T)));
  p = q;
  cap = want;
  if (grew) *grew = true;
  return 0;
}

static inline void tbegin(FuelMap* m, int t, cudaStream_t s = nullptr) { cudaEventRecord(m->ev0[t], s ? s : m->stream); }
static inline void tend(FuelMap* m, int t, cudaStream_t s = nullptr) {
  cudaEventRecord(m->ev1[t], s ? s : m->stream);
  m->ev_valid[t] = true;
}
#define FUEL_LAUNCHES(m, n) __atomic_fetch_add(&(m)->launches, (long long)(n), __ATOMIC_RELAXED)
#ifdef FUEL_PROF
static inline double prof_now_us() {
  return 1e-3 * (double)std::chrono::duration_cast<std::chrono::nanoseconds>(
                    std::chrono::steady_clock::now().time_since_epoch()).count();
}
#endif

__host__ __device__ static inline int64_t addr_of(const Geom& g, int x, int y, int z) {
  return ((int64_t)x * g.ny + y) * g.nz + z;
}

// ---- stage entry points implemented per .cu file ----
int esdf_update_impl(FuelMap* m, const int bmin[3], const int bmax[3], int flags);
void esdf_tile_scratch_sizes(int nx, int ny, int nz, size_t* rec_bytes, size_t* p_bytes, int* wc);
int esdf_tile_transform(FuelMap* m, const int lo[3], const int hi[3], int mode, float* out);
int edt_stage_zpack(cudaStream_t st, const uint8_t* occ, void* rec, int nxl, int ny, int nzc, int G, int64_t chunk_stride,
                    int mode);
int edt_stage_zy(cudaStream_t st, const void* rec, int nxl, int ny, int NW, int w0, int wn, int32_t* P, int64_t out_o,
                 int64_t out_bx, int64_t out_q);
int edt_stage_zy_scatter(cudaStream_t st, const void* rec, int nxl, int ny, int NW, int32_t* const* tab, int ntab, int wl,
                         int64_t out_o, int64_t out_bx, int64_t out_q);
int edt_stage_x(cudaStream_t st, const int32_t* P, int64_t in_o, int64_t in_bx, int64_t piece_stride, int piece_rows, int nx,
                int ny, int wn, float* out, int64_t out_o, int64_t out_bx, int64_t out_q, int lanes_total, float res,
                int discard);
int map_inflate_impl(FuelMap* m, const int bmin[3], const int bmax[3], int step, int ceil_id);
int esdf_sample_impl(FuelMap* m, int64_t n, const double* pos_dev, double* dist_dev, double* grad_dev);

int fusion_input_impl(FuelMap* m, const float* pts_host, int stride, int n, const double cam[3], const FuelFusionParams* p,
                      int32_t lbmin[3], int32_t lbmax[3]);
int fusion_input_depth_impl(FuelMap* m, const uint16_t* img_host, int rows, int cols, const FuelCameraParams* cp,
                            const double R[9], const double cam[3], const FuelFusionParams* p, int32_t lbmin[3],
                            int32_t lbmax[3], int32_t* proj_cnt);
int fusion_set_logodds(FuelMap* m, const double* logodds_host, double p_min, double p_occ);
int fusion_get_logodds(FuelMap* m, double* out);
void fusion_get_updated_box(FuelMap* m, double bmin[3], double bmax[3], int reset);
void fusion_state_destroy(FuelMap* m);
double* fusion_logodds_ptr(FuelMap* m, double* clamp_max_log);
void frontier_order_writer(FuelMap* m);
// main-stream writers of `dist` wait for an enqueued mirror download (fuelgpu_esdf_download_async)
static inline void esdf_order_writer(FuelMap* m) {
  if (m->mirror_pending) cudaStreamWaitEvent(m->stream, m->mirror_ev, 0);
}
int frontier_set_cell_order(FuelMap* m, int order);
int frontier_candidates_impl(FuelMap* m, const double umin[3], const double umax[3], const FuelFrontierParams* p, int z_lo,
                             int z_hi, int32_t* n_out);
int frontier_candidates_fetch_impl(FuelMap* m, int32_t n, int32_t* addr, uint8_t* cls);
int frontier_search_from_candidates_impl(FuelMap* m, const double umin[3], const double umax[3], const FuelFrontierParams* p,
                                         int32_t n, const int32_t* addr, const uint8_t* cls, int32_t* n_clusters,
                                         int32_t* n_cells, int32_t* n_filtered);  // main-stream writers of `occ` wait for an enqueued frontier search

int frontier_state_create(FuelMap* m);
// The frontier subsystem runs on its own stream (it only reads `occ` and owns `flag`), so a host
// thread can search frontiers while another updates the ESDF / runs the B-spline batch on the
// map's main stream.  frontier_stream() orders it after everything already queued on the main stream.
cudaStream_t frontier_stream(FuelMap* m);
cudaStream_t frontier_stream_raw(FuelMap* m);
void frontier_state_destroy(FuelMap* m);
int frontier_search_impl(FuelMap* m, const double umin[3], const double umax[3],
                         const FuelFrontierParams* p, int32_t* n_clusters, int32_t* n_cells,
                         int32_t* n_filtered);
int frontier_search_begin_impl(FuelMap* m, const double umin[3], const double umax[3],
                               const FuelFrontierParams* p);
int frontier_search_end_impl(FuelMap* m, int32_t* n_clusters, int32_t* n_cells, int32_t* n_filtered);
int frontier_fetch_impl(FuelMap* m, int32_t* cell_offsets, int32_t* cell_addr, int32_t* filt_offsets,
                        double* filtered, double* average, double* box_min, double* box_max);
int frontier_is_changed_impl(FuelMap* m, int32_t mcl, const int32_t* offs, const int32_t* addr,
                             uint8_t* changed, int32_t* counts = nullptr);
int viewpoint_candidates_host(const FuelViewParams* vp, std::vector<double>* off);
int sample_viewpoints_impl(FuelMap* m, int ncl, const int32_t* filt_off, const double* filt, const double* avg,
                           const FuelViewParams* vp, int ncand, double* cand_pos, double* cand_yaw, int32_t* cand_visib);

int bspline_cost_batch_dev_impl(FuelMap* m, int B, int n_pts, int mask, const FuelOptParams* p,
                                const FuelTrajConst* tc_dev, const double* x_dev, double* f_dev,
                                double* grad_dev);
int bspline_optimize_batch_dev_impl(FuelMap* m, int B, int n_pts, int mask, const FuelOptParams* p,
                                    const FuelTrajConst* tc_dev, const FuelSolveParams* sp,
                                    double* x_dev, double* fbest_dev, int32_t* neval_dev);
int bspline_optimize_long_impl(FuelMap* m, int B, int n_pts, int mask, const FuelOptParams* p,
                               const FuelTrajConst* tc_dev, const FuelSolveParams* sp, double* x_dev,
                               int32_t* neval_dev);
// traj_check.cu: NonUniformBspline checks / checkTrajCollision / selectBestTraj, and evaluateDeBoorT
int traj_check_impl(FuelMap* m, int B, int n_pts, int nvar, const double* x_dev, const double* dt_dev,
                    const FuelTrajCheckParams* p, FuelTrajReport* rep_dev, int32_t* best_dev);
int traj_evaluate_impl(FuelMap* m, int B, int n_pts, int nvar, const double* x_dev, const double* dt_dev, int n_t,
                       const double* t_dev, int deriv, double* out_dev);
// parameterizeToBspline + the constants optimize() freezes from its control points
int traj_param_impl(FuelMap* m, int B, int n_pts, int nvar, const double* pts_dev, const double* der_dev,
                    const double* dt_dev, const double* tlb_dev, double* x_dev, FuelTrajConst* tc_dev);
// planYawExplore (planner_manager.cpp:774-865) on each trajectory of a batch
int yaw_explore_impl(FuelMap* m, int B, int n_pts, int nvar, const double* x_dev, const double* dt_dev,
                     const double* syaw_dev, const double* eyaw_dev, const FuelOptParams* p, const FuelYawParams* yp,
                     double* yaw_dev, FuelYawInfo* info_dev, double* wpt_dev);
int plan_yaw_impl(FuelMap* m, int B, int n_pts, int nvar, const double* x_dev, const double* dt_dev,
                  const double* syaw_dev, const FuelOptParams* p, double* yaw_dev, FuelPlanYawInfo* info_dev,
                  double* wpt_dev);
// poly_traj.cu: waypointsTraj + getLength + planExploreTraj's sampling (planner_manager.cpp:270-297)
int poly_waypoints_impl(FuelMap* m, int B, int w_max, const int32_t* n_wp_dev, const double* wp_dev,
                        const double* sv_dev, const double* sa_dev, const double* ev_dev, const double* ea_dev,
                        const double* times_dev, const FuelPolyParams* p, FuelPolyInfo* info_dev, double* coeffs_dev,
                        double* points_dev, double* derivs_dev);
// astar.cu: Astar::search + shortenPath + planExploreMotion's goal branch (fast_exploration_manager.cpp:238-263)
int astar_impl(FuelMap* m, int B, const double* start_dev, const double* goal_dev, const FuelAstarParams* p,
               FuelPathInfo* info_dev, int path_max, double* path_dev, int w_max, int32_t* nwp_dev, double* wp_dev);
// the same search as ViewNode::searchPath runs it, over the queries list_dev[0 .. *n_list_dev) of P pairs: getPath() and
// its pathLength, no shortenPath or branch; the node pool is clamped to what max_iter can use
int astar_raw_impl(FuelMap* m, int P, const int* n_list_dev, const int* list_dev, const double* p1_dev,
                   const double* p2_dev, const FuelAstarParams* p, FuelPathInfo* info_dev, int path_max,
                   double* path_dev);
// kino_astar.cu: kinodynamicReplan's search, retry and getSamples (planner_manager.cpp:131-164) for B queries
int kino_check_params(FuelMap* m, const FuelKinoParams* p);
int kino_search_impl(FuelMap* m, int B, const double* start, const double* vel, const double* acc, const double* goal,
                     const FuelPathInfo* gate, const FuelKinoParams* p, FuelKinoInfo* info, double* points,
                     double* derivs, double* dt, int node_max, double* nodes, double* shot);
// view_cost.cu: ViewNode::searchPath + computeCost (graph_node.cpp:32-85) for P pairs
int view_cost_impl(FuelMap* m, int P, const double* p1, const double* p2, const double* y1, const double* y2,
                   const double* v1, const FuelViewCostParams* vp, FuelViewCostInfo* info_dev, int path_max,
                   double* path_dev);
// local_tour.cu: refineLocalTour (fast_exploration_manager.cpp:429-503) for B problems; prob_off / group_off on the host
struct LocalTourIO {
  const double *cur_pos, *cur_vel, *cur_yaw, *vp_pos, *vp_yaw;  // device
  FuelLocalTourInfo* info;
  int32_t* refined;
  double *tour, *edge_cost;  // edge_cost may be null
  int kmax, tour_max;
};
int local_tour_impl(FuelMap* m, int B, const int32_t* prob_off, const int32_t* group_off, const FuelLocalTourParams* p,
                    const LocalTourIO& io);
// global_tour.cu: findGlobalTour's ATSP (fast_exploration_manager.cpp:327-427) for B instances; dims on the host
int global_tour_impl(FuelMap* m, int B, const int32_t* dims, const double* cost_dev, FuelGlobalTourInfo* info_dev,
                     int32_t* indices_dev);

// getDistWithGrad on the device (sdf_map.cpp:497-536); shared by esdf.cu and bspline.cu
__device__ __forceinline__ double dev_get_distance(const Geom& g, const float* __restrict__ dist,
                                                   int x, int y, int z) {
  // getDistance(idx), sdf_map.h:228-231: -1 outside the map
  if (x < 0 || y < 0 || z < 0 || x > g.nx - 1 || y > g.ny - 1 || z > g.nz - 1) return -1.0;
  float v = __ldg(dist + addr_of(g, x, y, z));
  // "no site in the box" is +inf on the device; the reference holds resolution*sqrt(DBL_MAX)
  // there (sdf_map.cpp:196 on a DBL_MAX line).  Restore that finite value so the trilinear
  // arithmetic (inf-inf) matches the reference's.
  if (isinf(v)) return v > 0 ? g.res * sqrt(1.7976931348623157e308) : -(g.res * sqrt(1.7976931348623157e308));
  return (double)v;
}

__device__ __forceinline__ double dev_dist_with_grad(const Geom& g, const float* __restrict__ dist,
                                                     const double pos[3], double grad[3]) {
  // isInMap(pos), sdf_map.h:153-161
  if (pos[0] < g.origin[0] + 1e-4 || pos[1] < g.origin[1] + 1e-4 || pos[2] < g.origin[2] + 1e-4 ||
      pos[0] > g.map_max[0] - 1e-4 || pos[1] > g.map_max[1] - 1e-4 || pos[2] > g.map_max[2] - 1e-4) {
    grad[0] = grad[1] = grad[2] = 0.0;
    return 0.0;
  }
  int idx[3];
  double diff[3];
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    double pm = pos[i] - 0.5 * g.res * 1.0;
    idx[i] = (int)floor((pm - g.origin[i]) * g.res_inv);
    double ip = (idx[i] + 0.5) * g.res + g.origin[i];
    diff[i] = (pos[i] - ip) * g.res_inv;
  }
  double v[2][2][2];
#pragma unroll
  for (int x = 0; x < 2; x++)
#pragma unroll
    for (int y = 0; y < 2; y++)
#pragma unroll
      for (int z = 0; z < 2; z++) v[x][y][z] = dev_get_distance(g, dist, idx[0] + x, idx[1] + y, idx[2] + z);

  // no FMA contraction here: keep the reference's rounding sequence
  double v00 = __dadd_rn(__dmul_rn(1 - diff[0], v[0][0][0]), __dmul_rn(diff[0], v[1][0][0]));
  double v01 = __dadd_rn(__dmul_rn(1 - diff[0], v[0][0][1]), __dmul_rn(diff[0], v[1][0][1]));
  double v10 = __dadd_rn(__dmul_rn(1 - diff[0], v[0][1][0]), __dmul_rn(diff[0], v[1][1][0]));
  double v11 = __dadd_rn(__dmul_rn(1 - diff[0], v[0][1][1]), __dmul_rn(diff[0], v[1][1][1]));
  double v0 = __dadd_rn(__dmul_rn(1 - diff[1], v00), __dmul_rn(diff[1], v10));
  double v1 = __dadd_rn(__dmul_rn(1 - diff[1], v01), __dmul_rn(diff[1], v11));
  double d = __dadd_rn(__dmul_rn(1 - diff[2], v0), __dmul_rn(diff[2], v1));

  grad[2] = __dmul_rn(v1 - v0, g.res_inv);
  grad[1] = __dmul_rn(
      __dadd_rn(__dmul_rn(1 - diff[2], v10 - v00), __dmul_rn(diff[2], v11 - v01)), g.res_inv);
  double g0 = __dmul_rn(__dmul_rn(1 - diff[2], 1 - diff[1]), v[1][0][0] - v[0][0][0]);
  g0 = __dadd_rn(g0, __dmul_rn(__dmul_rn(1 - diff[2], diff[1]), v[1][1][0] - v[0][1][0]));
  g0 = __dadd_rn(g0, __dmul_rn(__dmul_rn(diff[2], 1 - diff[1]), v[1][0][1] - v[0][0][1]));
  g0 = __dadd_rn(g0, __dmul_rn(__dmul_rn(diff[2], diff[1]), v[1][1][1] - v[0][1][1]));
  grad[0] = __dmul_rn(g0, g.res_inv);
  return d;
}
