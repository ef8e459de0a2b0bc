// view_cost.cu -- ViewNode::searchPath and ViewNode::computeCost (active_perception/src/graph_node.cpp:32-85) on sm_90a
// for a batch of viewpoint pairs, the edge cost behind FrontierFinder::updateFrontierCostMatrix / getFullCostMatrix.
//
// Three launches on the map's main stream, with no host synchronisation between them:
//   1. vc_line_kernel: the straight-line test, one pair per thread -- the RayCaster walk of raycast.cuh with the box
//      test of searchPath; a pair whose line is blocked is appended to a list on the device;
//   2. astar_kernel<true> (astar.cu) over that list, its length read from device memory: Astar::search at the given
//      resolution, getPath() and Astar::pathLength;
//   3. vc_cost_kernel: searchPath's result (the line, the search's path, or 1000 without one) and computeCost.
// Built with -fmad=false: every double operation rounds as the reference's does, except acos (the device's libm).
#include "common.cuh"
#include "raycast.cuh"

#include <math.h>

namespace {

constexpr int VC_THREADS = 128;

struct VcPairs {
  const double *p1, *p2, *y1, *y2, *v1;
};

__device__ __forceinline__ double vc_norm3(double x, double y, double z) { return sqrt((x * x + y * y) + z * z); }

__global__ void __launch_bounds__(VC_THREADS)
vc_line_kernel(Geom g, const uint8_t* __restrict__ occ, int P, VcPairs in, FuelViewCostInfo* __restrict__ info,
               int* __restrict__ n_list, int* __restrict__ list) {
  const int q = blockIdx.x * VC_THREADS + threadIdx.x;
  if (q >= P) return;
  const double a[3] = { in.p1[3 * q], in.p1[3 * q + 1], in.p1[3 * q + 2] };
  const double b[3] = { in.p2[3 * q], in.p2[3 * q + 1], in.p2[3 * q + 2] };
  bool finite = isfinite(in.y1[q]) && isfinite(in.y2[q]);
#pragma unroll
  for (int k = 0; k < 3; ++k) finite = finite && isfinite(a[k]) && isfinite(b[k]) && isfinite(in.v1[3 * q + k]);
  FuelViewCostInfo r;
  memset(&r, 0, sizeof(r));
  if (!finite) {
    r.reason = FUELGPU_ASTAR_BAD_INPUT;
  } else if (ray_is_clear<true>(g, occ, a, b)) {
    r.kind = FUELGPU_VIEW_LINE;
  } else {
    r.kind = FUELGPU_VIEW_ASTAR;  // until the search says otherwise
    list[atomicAdd(n_list, 1)] = q;
  }
  info[q] = r;
}

__global__ void __launch_bounds__(VC_THREADS)
vc_cost_kernel(int P, VcPairs in, double vm, double yd, double w_dir, const FuelPathInfo* __restrict__ search,
               FuelViewCostInfo* __restrict__ info, int path_max, double* __restrict__ path) {
  const int q = blockIdx.x * VC_THREADS + threadIdx.x;
  if (q >= P) return;
  FuelViewCostInfo r = info[q];
  const double a[3] = { in.p1[3 * q], in.p1[3 * q + 1], in.p1[3 * q + 2] };
  const double b[3] = { in.p2[3 * q], in.p2[3 * q + 1], in.p2[3 * q + 2] };
  int rows = 0;  // rows of `path` this kernel writes: {p1, p2}, or nothing on a bad row
  if (r.kind == FUELGPU_VIEW_LINE) {
    r.n_path = 2;
    r.length = vc_norm3(a[0] - b[0], a[1] - b[1], a[2] - b[2]);  // (p1 - p2).norm()
    rows = 2;
  } else if (r.kind == FUELGPU_VIEW_ASTAR) {
    const FuelPathInfo s = search[q];
    r.reason = s.reason;
    r.iter_num = s.iter_num;
    r.use_node_num = s.use_node_num;
    if (s.status == FUELGPU_ASTAR_REACH_END) {  // the search wrote its path rows
      r.n_path = s.n_path;
      r.length = s.length;
      rows = -1;
    } else {  // "early termination cost as an estimate" (graph_node.cpp:58-60)
      r.kind = FUELGPU_VIEW_NO_PATH;
      r.n_path = 2;
      r.length = 1000.0;
      rows = 2;
    }
  }
  if (r.kind) {
    double pos_cost = r.length / vm;
    const double v[3] = { in.v1[3 * q], in.v1[3 * q + 1], in.v1[3 * q + 2] };
    if (vc_norm3(v[0], v[1], v[2]) > 1e-3) {
      double dir[3] = { b[0] - a[0], b[1] - a[1], b[2] - a[2] };  // (p2 - p1).normalized(): unchanged when zero
      double vdir[3] = { v[0], v[1], v[2] };
      const double zd = (dir[0] * dir[0] + dir[1] * dir[1]) + dir[2] * dir[2];
      if (zd > 0.0) {
        const double n = sqrt(zd);
        dir[0] = dir[0] / n, dir[1] = dir[1] / n, dir[2] = dir[2] / n;
      }
      const double zv = (vdir[0] * vdir[0] + vdir[1] * vdir[1]) + vdir[2] * vdir[2];
      const double n = sqrt(zv);
      vdir[0] = vdir[0] / n, vdir[1] = vdir[1] / n, vdir[2] = vdir[2] / n;
      const double diff = acos((vdir[0] * dir[0] + vdir[1] * dir[1]) + vdir[2] * dir[2]);
      pos_cost += w_dir * diff;
    }
    double diff = fabs(in.y2[q] - in.y1[q]);
    const double other = 2 * M_PI - diff;
    diff = other < diff ? other : diff;  // std::min(diff, 2 * M_PI - diff)
    const double yaw_cost = diff / yd;
    r.cost = pos_cost < yaw_cost ? yaw_cost : pos_cost;  // std::max: a NaN pos_cost stays
  }
  info[q] = r;
  if (path && rows >= 0) {
    double* dst = path + (size_t)q * path_max * 3;
    for (int i = 0; i < path_max; ++i) {
      const bool on = i < rows, first = i == 0;
      dst[3 * i] = on ? (first ? a[0] : b[0]) : 0.0;
      dst[3 * i + 1] = on ? (first ? a[1] : b[1]) : 0.0;
      dst[3 * i + 2] = on ? (first ? a[2] : b[2]) : 0.0;
    }
  }
}

}  // namespace

int view_cost_impl(FuelMap* m, int P, const double* p1, const double* p2, const double* y1, const double* y2,
                   const double* v1, const FuelViewCostParams* vp, FuelViewCostInfo* info_dev, int path_max,
                   double* path_dev) {
  if (P == 0) return 0;
  auto al = [](size_t b) { return (b + 255) & ~(size_t)255; };
  const size_t off_list = 256, off_search = off_list + al(sizeof(int) * (size_t)P);
  const int rc = m->vc_buf.ensure(m, off_search + sizeof(FuelPathInfo) * (size_t)P);
  if (rc) return rc;
  int* n_list = (int*)m->vc_buf.p;
  int* list = (int*)(m->vc_buf.p + off_list);
  FuelPathInfo* search = (FuelPathInfo*)(m->vc_buf.p + off_search);
  const VcPairs in{ p1, p2, y1, y2, v1 };
  const unsigned blocks = (unsigned)((P + VC_THREADS - 1) / VC_THREADS);
  FUEL_CUDA(m, cudaMemsetAsync(n_list, 0, sizeof(int), m->stream));
  vc_line_kernel<<<blocks, VC_THREADS, 0, m->stream>>>(m->g, m->occ, P, in, info_dev, n_list, list);
  FUEL_LAUNCHES(m, 1);
  FUEL_CUDA(m, cudaGetLastError());
  const int r = astar_raw_impl(m, P, n_list, list, p1, p2, &vp->astar, search, path_max, path_dev);
  if (r) return r;
  vc_cost_kernel<<<blocks, VC_THREADS, 0, m->stream>>>(P, in, vp->vm, vp->yd, vp->w_dir, search, info_dev, path_max,
                                                       path_dev);
  FUEL_LAUNCHES(m, 1);
  FUEL_CUDA(m, cudaGetLastError());
  return 0;
}
