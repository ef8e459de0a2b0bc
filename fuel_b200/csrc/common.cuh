// common.cuh -- shared state and helpers of libfuelgpu (sm_90a only).
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include <vector>

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

enum { T_ESDF = 0, T_FRONTIER = 1, T_BSPLINE = 2, T_UPLOAD = 3, T_DOWNLOAD = 4, T_COUNT = 8 };

struct FrontierState;  // frontier.cu
struct FusionState;    // fusion.cu

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
  // staging for ingest
  void* stage;
  size_t stage_bytes;
  cudaStream_t own_stream, stream;
  cudaStream_t copy_stream;  // D2H mirror copies that may overlap the main stream
  cudaEvent_t copy_ev;
  bool dist_ev_ok;           // ev1[T_ESDF] marks the last write of `dist` (a mirror download waits on it, not on later work)
  cudaStream_t in_stream;    // H2D of the solver inputs: goes out at once, not behind the ESDF kernels of the main stream
  cudaEvent_t in_ev;
  cudaEvent_t ev0[T_COUNT], ev1[T_COUNT];
  bool ev_valid[T_COUNT];
  FrontierState* fs;
  FusionState* fus;  // lazily created by the first fusion call
  // bspline scratch (device)
  void* bs_buf;
  size_t bs_bytes;
  void* bs_pin;  // page-locked bounce buffer for the host-facing B-spline calls
  size_t bs_pin_bytes;
  void* bs_grad;  // gradient output of the faithful re-evaluation after the long-trajectory solver (discarded)
  size_t bs_grad_bytes;
  void* fr_scr;  // device scratch of the small frontier-side calls (is_changed, viewpoints), grown on demand
  size_t fr_scr_bytes;
  int bs_pend_B, bs_pend_nvar;  // optimize_batch_begin issued, _end outstanding (B == 0: none)
  size_t bs_pend_off;           // offset of the result block inside bs_pin
  long long launches;  // kernels launched so far
  char err[512];
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

static inline void tbegin(FuelMap* m, int t, cudaStream_t s = nullptr) { cudaEventRecord(m->ev0[t], s ? s : m->stream); }
static inline void tend(FuelMap* m, int t, cudaStream_t s = nullptr) {
  cudaEventRecord(m->ev1[t], s ? s : m->stream);
  m->ev_valid[t] = true;
}
#define FUEL_LAUNCHES(m, n) __atomic_fetch_add(&(m)->launches, (long long)(n), __ATOMIC_RELAXED)

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
int frontier_set_cell_order(FuelMap* m, int order);
int frontier_candidates_impl(FuelMap* m, const double umin[3], const double umax[3], const FuelFrontierParams* p, int z_lo,
                             int z_hi, int32_t* n_out);
int frontier_candidates_fetch_impl(FuelMap* m, int32_t n, int32_t* addr, uint8_t* cls);
int frontier_search_from_candidates_impl(FuelMap* m, const double umin[3], const double umax[3], const FuelFrontierParams* p,
                                         int32_t n, const int32_t* addr, const uint8_t* cls, int32_t* n_clusters,
                                         int32_t* n_cells, int32_t* n_filtered);  // main-stream writers of `occ` wait for an enqueued frontier search

int ensure_fr_scratch(FuelMap* m, size_t bytes);
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
                               double* fbest_dev, int32_t* neval_dev);

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
