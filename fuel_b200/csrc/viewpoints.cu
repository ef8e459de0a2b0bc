// viewpoints.cu -- viewpoint sampling and visibility for new frontier clusters on sm_90a (SURVEY.md 8f rank 4).
//
// Replaces FrontierFinder::sampleViewpoints / countVisibleCells / isNearUnknown / wrapYaw
// (active_perception/src/frontier_finder.cpp:662-695,721-755,776-781) and PerceptionUtils::setPose / insideFOV
// (active_perception/src/perception_utils.cpp:49-93).  One thread block per (cluster, candidate): the reference's
// ~100 candidates per cluster x |filtered_cells_| raycasts are independent, and all of them read the resident
// occupancy byte (inflate bit + tri-state) the ESDF and frontier kernels already use.
#include "common.cuh"
#include "raycast.cuh"

#include <math.h>

#include <vector>

namespace {

struct ViewConsts {
  double ta, tb, lc, ld, re, rf;  // FOV plane normals in the camera frame (perception_utils.cpp:13-17)
  double max_dist;
  int clear_vox;  // floor(min_candidate_clearance_ / resolution_), frontier_finder.cpp:722
};

__device__ __forceinline__ void pos_to_idx(const Geom& g, const double p[3], int id[3]) {  // sdf_map.h:127-130
#pragma unroll
  for (int k = 0; k < 3; ++k) id[k] = (int)floor((p[k] - g.origin[k]) * g.res_inv);
}

__device__ __forceinline__ void normalized3(const double v[3], double out[3]) {  // Eigen normalized()
  const double z = __dadd_rn(__dadd_rn(__dmul_rn(v[0], v[0]), __dmul_rn(v[1], v[1])), __dmul_rn(v[2], v[2]));
  if (z > 0) {
    const double n = sqrt(z);
    out[0] = v[0] / n, out[1] = v[1] / n, out[2] = v[2] / n;
  } else
    out[0] = v[0], out[1] = v[1], out[2] = v[2];
}
__device__ __forceinline__ double dot3(const double a[3], const double b[3]) {
  return __dadd_rn(__dadd_rn(__dmul_rn(a[0], b[0]), __dmul_rn(a[1], b[1])), __dmul_rn(a[2], b[2]));
}

constexpr int VP_THREADS = 128;

// HOSTYAW = false: one block per (candidate, cluster); the average yaw comes from the device's acos/atan2 (<= 2 ulp
// per call, so the yaw and the FOV plane normals are within ~1e-12 of the host's) and cand_unc[out] is raised when a
// FOV plane test of some cell comes closer to zero than 1e-9: only then could the host's libm decide otherwise.
// HOSTYAW = true: second pass over the raised candidates (redo[blockIdx.x] = out index) with yaw, cos(yaw), sin(yaw)
// computed by the host's libm exactly as the reference does, so that the visible count is the reference's integer.
constexpr double FOV_EPS = 1e-9;

template <bool HOSTYAW>
__global__ void __launch_bounds__(VP_THREADS)
sample_viewpoints_kernel(Geom g, const uint8_t* __restrict__ occ, ViewConsts vc, int ncand, const double* __restrict__ off_xy,
                         const int* __restrict__ filt_off, const double* __restrict__ filt, const double* __restrict__ avg,
                         double* __restrict__ cand_pos, double* __restrict__ cand_yaw, int* __restrict__ cand_visib,
                         int* __restrict__ cand_unc, const int* __restrict__ redo, const double* __restrict__ host_yaw) {
  const int t = threadIdx.x;
  const int out = HOSTYAW ? redo[blockIdx.x] : (int)(blockIdx.y * ncand + blockIdx.x);
  const int c = out % ncand, cl = out / ncand;
  const double* cells = filt + 3 * (int64_t)filt_off[cl];
  const int n_cells = filt_off[cl + 1] - filt_off[cl];
  // sample_pos = average_ + rc * (cos phi, sin phi, 0): the products come from the host's libm (api side)
  const double pos[3] = { __dadd_rn(avg[3 * cl], off_xy[2 * c]), __dadd_rn(avg[3 * cl + 1], off_xy[2 * c + 1]),
                          __dadd_rn(avg[3 * cl + 2], 0.0) };
  __shared__ int s_reject, s_visib, s_unc;
  __shared__ double s_term[VP_THREADS];
  __shared__ double s_ref[3], s_yaw, s_nrm[4][3];
  if (t == 0) {
    s_reject = 0;
    s_visib = 0;
    s_unc = 0;
    cand_pos[3 * out] = pos[0], cand_pos[3 * out + 1] = pos[1], cand_pos[3 * out + 2] = pos[2];
    // isInBox(pos) (sdf_map.h:180-187) and getInflateOccupancy(pos) == 1 (:222-226), frontier_finder.cpp:671-672
    bool inbox = true;
#pragma unroll
    for (int k = 0; k < 3; ++k)
      if (pos[k] <= g.box_mind[k] || pos[k] >= g.box_maxd[k]) inbox = false;
    int id[3];
    pos_to_idx(g, pos, id);
    if (!inbox || (idx_in_map(g, id[0], id[1], id[2]) && (occ[addr_of(g, id[0], id[1], id[2])] & 4))) s_reject = 1;
  }
  __syncthreads();
  // isNearUnknown (:721-732): (2v+1)^2 x 3 probes
  {
    const int w = 2 * vc.clear_vox + 1, total = w * w * 3;
    for (int i = t; i < total && !s_reject; i += VP_THREADS) {
      const int zz = i % 3 - 1, yy = (i / 3) % w - vc.clear_vox, xx = i / (3 * w) - vc.clear_vox;
      const double v[3] = { __dadd_rn(pos[0], __dmul_rn(xx, g.res)), __dadd_rn(pos[1], __dmul_rn(yy, g.res)),
                            __dadd_rn(pos[2], __dmul_rn(zz, g.res)) };
      int id[3];
      pos_to_idx(g, v, id);
      if (idx_in_map(g, id[0], id[1], id[2]) && (occ[addr_of(g, id[0], id[1], id[2])] & 3) == FUELGPU_UNKNOWN) s_reject = 1;
    }
  }
  __syncthreads();
  if (s_reject || n_cells <= 0) {
    if (t == 0) {
      cand_yaw[out] = 0.0;
      cand_visib[out] = -1;
      if (!HOSTYAW) cand_unc[out] = 0;
    }
    return;
  }
  // average yaw (:675-685): per-cell terms in parallel, summed by one thread in the reference's order
  if (!HOSTYAW) {
    if (t == 0) {
      const double d0[3] = { cells[0] - pos[0], cells[1] - pos[1], cells[2] - pos[2] };
      double r[3];
      normalized3(d0, r);
      s_ref[0] = r[0], s_ref[1] = r[1], s_ref[2] = r[2];
      s_yaw = 0.0;
    }
    __syncthreads();
    for (int base = 1; base < n_cells; base += VP_THREADS) {
      const int i = base + t;
      if (i < n_cells) {
        const double d[3] = { cells[3 * i] - pos[0], cells[3 * i + 1] - pos[1], cells[3 * i + 2] - pos[2] };
        double dir[3];
        normalized3(d, dir);
        const double ref[3] = { s_ref[0], s_ref[1], s_ref[2] };
        double yaw = acos(dot3(dir, ref));
        if (__dadd_rn(__dmul_rn(ref[0], dir[1]), -__dmul_rn(ref[1], dir[0])) < 0) yaw = -yaw;
        s_term[t] = yaw;
      }
      __syncthreads();
      if (t == 0) {
        double a = s_yaw;
        const int m = min(VP_THREADS, n_cells - base);
        for (int k = 0; k < m; ++k) a = __dadd_rn(a, s_term[k]);
        s_yaw = a;
      }
      __syncthreads();
    }
  }
  if (t == 0) {
    double a, cy, sy;
    if (HOSTYAW) {
      a = host_yaw[3 * blockIdx.x], cy = host_yaw[3 * blockIdx.x + 1], sy = host_yaw[3 * blockIdx.x + 2];
    } else {
      a = __dadd_rn(s_yaw / n_cells, atan2(s_ref[1], s_ref[0]));
      const double PI = 3.14159265358979323846;
      for (int it = 0; it < 64 && a < -PI; ++it) a = __dadd_rn(a, 2 * PI);  // wrapYaw :776-781 (bounded; NaN falls through)
      for (int it = 0; it < 64 && a > PI; ++it) a = __dadd_rn(a, -(2 * PI));
      cy = cos(a), sy = sin(a);
    }
    s_yaw = a;
    cand_yaw[out] = a;
    // setPose (perception_utils.cpp:49-66): normals_ = R_wc * {n_top, n_bottom, n_left, n_right}
    s_nrm[0][0] = __dmul_rn(cy, vc.tb), s_nrm[0][1] = __dmul_rn(sy, vc.tb), s_nrm[0][2] = vc.ta;
    s_nrm[1][0] = __dmul_rn(cy, vc.tb), s_nrm[1][1] = __dmul_rn(sy, vc.tb), s_nrm[1][2] = -vc.ta;
    s_nrm[2][0] = __dadd_rn(__dmul_rn(sy, vc.lc), __dmul_rn(cy, vc.ld));
    s_nrm[2][1] = __dadd_rn(__dmul_rn(-cy, vc.lc), __dmul_rn(sy, vc.ld));
    s_nrm[2][2] = 0.0;
    s_nrm[3][0] = __dadd_rn(__dmul_rn(sy, -vc.re), __dmul_rn(cy, vc.rf));
    s_nrm[3][1] = __dadd_rn(__dmul_rn(-cy, -vc.re), __dmul_rn(sy, vc.rf));
    s_nrm[3][2] = 0.0;
  }
  __syncthreads();
  // countVisibleCells (:734-755)
  int mine = 0;
  for (int i = t; i < n_cells; i += VP_THREADS) {
    const double cell[3] = { cells[3 * i], cells[3 * i + 1], cells[3 * i + 2] };
    const double dir[3] = { cell[0] - pos[0], cell[1] - pos[1], cell[2] - pos[2] };
    const double nn = sqrt(dot3(dir, dir));  // insideFOV, perception_utils.cpp:83-93
    if (nn > vc.max_dist) continue;
    double u[3];
    normalized3(dir, u);
    bool inside = true, close = false;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const double nk[3] = { s_nrm[k][0], s_nrm[k][1], s_nrm[k][2] };
      const double dk = dot3(u, nk);
      if (dk < 0.0) inside = false;
      if (fabs(dk) <= FOV_EPS) close = true;
    }
    if (!HOSTYAW && close) s_unc = 1;  // benign race: every writer stores 1
    if (!inside) continue;
    if (ray_is_clear(g, occ, cell, pos)) ++mine;
  }
  if (mine) atomicAdd(&s_visib, mine);
  __syncthreads();
  if (t == 0) {
    cand_visib[out] = s_visib;
    if (!HOSTYAW) cand_unc[out] = s_unc;
  }
}

}  // namespace

int viewpoint_candidates_host(const FuelViewParams* vp, std::vector<double>* off) {
  // the two loops of sampleViewpoints (:664-667); cos/sin from the host libm, like the reference
  int n = 0;
  for (double rc = vp->candidate_rmin, dr = (vp->candidate_rmax - vp->candidate_rmin) / vp->candidate_rnum;
       rc <= vp->candidate_rmax + 1e-3; rc += dr) {
    for (double phi = -M_PI; phi < M_PI; phi += vp->candidate_dphi) {
      if (off) {
        off->push_back(rc * cos(phi));
        off->push_back(rc * sin(phi));
      }
      if (++n > 65535) return -1;
    }
    if (!(dr > 0)) break;  // rnum/rmax misconfigured: do not spin
  }
  return n;
}

int sample_viewpoints_impl(FuelMap* m, int ncl, const int32_t* filt_off, const double* filt, const double* avg,
                           const FuelViewParams* vp, int ncand, double* cand_pos, double* cand_yaw, int32_t* cand_visib) {
  std::vector<double> off;
  const int nc = viewpoint_candidates_host(vp, &off);
  if (nc <= 0 || nc != ncand) return fuel_fail(m, FUELGPU_EINVAL, "candidate count does not match fuelgpu_viewpoint_candidate_count");
  if (ncl <= 0) return 0;
  const int nfilt = filt_off[ncl];
  ViewConsts vc;
  vc.ta = sin(M_PI_2 - vp->top_angle), vc.tb = cos(M_PI_2 - vp->top_angle);
  vc.lc = sin(M_PI_2 - vp->left_angle), vc.ld = cos(M_PI_2 - vp->left_angle);
  vc.re = sin(M_PI_2 - vp->right_angle), vc.rf = cos(M_PI_2 - vp->right_angle);
  vc.max_dist = vp->max_dist;
  vc.clear_vox = (int)floor(vp->min_candidate_clearance / m->g.res);
  if (vc.clear_vox < 0 || vc.clear_vox > 64) return fuel_fail(m, FUELGPU_EINVAL, "min_candidate_clearance out of range");
  cudaStream_t s = frontier_stream(m);
  const size_t n_out = (size_t)ncl * nc;
  // one staging allocation: [off 2nc][avg 3ncl][filt 3nfilt][pos 3n_out][yaw n_out][host yaw 3n_out] doubles, then ints
  const size_t nd = 2 * (size_t)nc + 3 * (size_t)ncl + 3 * (size_t)(nfilt > 0 ? nfilt : 1) + 7 * n_out;
  const size_t ni = (size_t)ncl + 1 + 3 * n_out;
  const size_t dbytes = (sizeof(double) * nd + 255) & ~(size_t)255;
  int rc = m->fr_scr.ensure(m, dbytes + sizeof(int) * ni);
  if (rc) return rc;
  double* d_d = (double*)m->fr_scr.p;
  int* d_i = (int*)(m->fr_scr.p + dbytes);
  double *d_off = d_d, *d_avg = d_off + 2 * nc, *d_filt = d_avg + 3 * ncl, *d_pos = d_filt + 3 * (size_t)(nfilt > 0 ? nfilt : 1),
         *d_yaw = d_pos + 3 * n_out, *d_hyaw = d_yaw + n_out;
  int *d_fo = d_i, *d_vis = d_i + ncl + 1, *d_unc = d_vis + n_out, *d_redo = d_unc + n_out;
  FUEL_CUDA(m, cudaMemcpyAsync(d_off, off.data(), sizeof(double) * 2 * nc, cudaMemcpyHostToDevice, s));
  FUEL_CUDA(m, cudaMemcpyAsync(d_avg, avg, sizeof(double) * 3 * ncl, cudaMemcpyHostToDevice, s));
  if (nfilt > 0) FUEL_CUDA(m, cudaMemcpyAsync(d_filt, filt, sizeof(double) * 3 * nfilt, cudaMemcpyHostToDevice, s));
  FUEL_CUDA(m, cudaMemcpyAsync(d_fo, filt_off, sizeof(int) * (ncl + 1), cudaMemcpyHostToDevice, s));
  sample_viewpoints_kernel<false><<<dim3(nc, ncl), VP_THREADS, 0, s>>>(m->g, m->occ, vc, nc, d_off, d_fo, d_filt, d_avg, d_pos,
                                                                       d_yaw, d_vis, d_unc, nullptr, nullptr);
  FUEL_LAUNCHES(m, 1);
  FUEL_CUDA(m, cudaGetLastError());
  std::vector<int> unc(n_out);
  FUEL_CUDA(m, cudaMemcpyAsync(cand_pos, d_pos, sizeof(double) * 3 * n_out, cudaMemcpyDeviceToHost, s));
  FUEL_CUDA(m, cudaMemcpyAsync(cand_yaw, d_yaw, sizeof(double) * n_out, cudaMemcpyDeviceToHost, s));
  FUEL_CUDA(m, cudaMemcpyAsync(cand_visib, d_vis, sizeof(int) * n_out, cudaMemcpyDeviceToHost, s));
  FUEL_CUDA(m, cudaMemcpyAsync(unc.data(), d_unc, sizeof(int) * n_out, cudaMemcpyDeviceToHost, s));
  FUEL_CUDA(m, cudaStreamSynchronize(s));
  // candidates with a FOV test on the edge: the yaw again, with the host's libm and the reference's operation order
  // (frontier_finder.cpp:675-685, wrapYaw :776-781), and the visibility count with the normals it implies
  std::vector<int> redo;
  std::vector<double> hy;
  for (size_t o = 0; o < n_out; ++o) {
    if (!unc[o]) continue;
    const int cl = (int)(o / nc);
    const double* cells = filt + 3 * (size_t)filt_off[cl];
    const int n_cells = filt_off[cl + 1] - filt_off[cl];
    const double* pos = cand_pos + 3 * o;
    auto normalized = [](const double v[3], double out[3]) {
      const double z = (v[0] * v[0] + v[1] * v[1]) + v[2] * v[2];
      if (z > 0) {
        const double nrm = sqrt(z);
        out[0] = v[0] / nrm, out[1] = v[1] / nrm, out[2] = v[2] / nrm;
      } else
        out[0] = v[0], out[1] = v[1], out[2] = v[2];
    };
    const double d0[3] = { cells[0] - pos[0], cells[1] - pos[1], cells[2] - pos[2] };
    double ref[3];
    normalized(d0, ref);
    double a = 0.0;
    for (int i = 1; i < n_cells; ++i) {
      const double d[3] = { cells[3 * i] - pos[0], cells[3 * i + 1] - pos[1], cells[3 * i + 2] - pos[2] };
      double dir[3];
      normalized(d, dir);
      double yaw = acos((dir[0] * ref[0] + dir[1] * ref[1]) + dir[2] * ref[2]);
      if (ref[0] * dir[1] - ref[1] * dir[0] < 0) yaw = -yaw;
      a += yaw;
    }
    a = a / n_cells + atan2(ref[1], ref[0]);
    for (int it = 0; it < 64 && a < -M_PI; ++it) a += 2 * M_PI;
    for (int it = 0; it < 64 && a > M_PI; ++it) a -= 2 * M_PI;
    redo.push_back((int)o);
    hy.push_back(a);
    hy.push_back(cos(a));
    hy.push_back(sin(a));
  }
  if (!redo.empty()) {
    FUEL_CUDA(m, cudaMemcpyAsync(d_redo, redo.data(), sizeof(int) * redo.size(), cudaMemcpyHostToDevice, s));
    FUEL_CUDA(m, cudaMemcpyAsync(d_hyaw, hy.data(), sizeof(double) * hy.size(), cudaMemcpyHostToDevice, s));
    sample_viewpoints_kernel<true><<<(unsigned)redo.size(), VP_THREADS, 0, s>>>(m->g, m->occ, vc, nc, d_off, d_fo, d_filt, d_avg,
                                                                               d_pos, d_yaw, d_vis, d_unc, d_redo, d_hyaw);
    FUEL_LAUNCHES(m, 1);
    FUEL_CUDA(m, cudaGetLastError());
    FUEL_CUDA(m, cudaMemcpyAsync(cand_yaw, d_yaw, sizeof(double) * n_out, cudaMemcpyDeviceToHost, s));
    FUEL_CUDA(m, cudaMemcpyAsync(cand_visib, d_vis, sizeof(int) * n_out, cudaMemcpyDeviceToHost, s));
    FUEL_CUDA(m, cudaStreamSynchronize(s));
  }
  return 0;
}
