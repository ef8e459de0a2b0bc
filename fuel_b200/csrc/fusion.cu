// fusion.cu -- occupancy fusion of one depth frame on sm_90a (SURVEY.md 8f rank 3).
//
// Replaces SDFMap::inputPointCloud (plan_env/src/sdf_map.cpp:259-345) with setCacheOccupancy
// (:243-257), closetPointInMap (:347-362) and RayCaster::input/nextId
// (plan_env/src/raycast.cpp:6-23,323-407).  The reference walks the points one by one; nothing
// in it is order-dependent except WHICH point of several that end in the same voxel gets its ray
// traced (the first, :303-306).  Here:
//   1. one thread per point: clip to the map / to max_ray_length, classify hit/miss, mark the end
//      voxel, fold the point into the updated box, and elect the first point of every end voxel
//      (atomicMin of the point index);
//   2. one thread per elected point: the reference's integer-delta DDA from the point back to the
//      camera, marking every traversed voxel "missed";
//   3. one thread per voxel of the updated box: voxels touched this frame get the log-odds update
//      (hit iff count_hit >= count_miss, i.e. iff it was hit at least once) with the reference's
//      unknown -> min_occupancy_log initialisation and clamps, in fp64 like occupancy_buffer_; the
//      tri-state byte is refreshed; the per-frame marks are cleared.
#include "common.cuh"

#include <math.h>

namespace {

struct FusionConsts {
  double max_ray_length;
  double clamp_min, clamp_max, hit, miss, min_occ;
};

// double <-> order-preserving unsigned 64-bit (for atomicMin/Max on coordinates)
__host__ __device__ inline unsigned long long d2o(double d) {
  unsigned long long u;
  memcpy(&u, &d, 8);
  return (u & 0x8000000000000000ull) ? ~u : (u | 0x8000000000000000ull);
}
__host__ __device__ inline double o2d(unsigned long long u) {
  u = (u & 0x8000000000000000ull) ? (u & 0x7fffffffffffffffull) : ~u;
  double d;
  memcpy(&d, &u, 8);
  return d;
}

__device__ __forceinline__ bool in_map_pos(const Geom& g, const double p[3]) {  // sdf_map.h:153-161
  return !(p[0] < g.origin[0] + 1e-4 || p[1] < g.origin[1] + 1e-4 || p[2] < g.origin[2] + 1e-4 ||
           p[0] > g.map_max[0] - 1e-4 || p[1] > g.map_max[1] - 1e-4 || p[2] > g.map_max[2] - 1e-4);
}

// marks: one byte per voxel, bit0 = hit this frame, bit1 = missed this frame.  Byte-wise OR through a
// 32-bit atomic on the containing word.
__device__ __forceinline__ void mark_or(uint8_t* mark, int64_t adr, unsigned bits) {
  unsigned* w = (unsigned*)(mark + (adr & ~(int64_t)3));
  const unsigned v = bits << (8 * (unsigned)(adr & 3));
  if ((*(volatile unsigned*)w & v) != v) atomicOr(w, v);
}

// One point of the cloud (index i in the reference's iteration order): sdf_map.cpp:273-306 up to the ray election.
__device__ __forceinline__ void classify_point(const Geom& g, const FusionConsts& fc, int i, double p0, double p1, double p2,
                                               double cx, double cy, double cz, double* __restrict__ ptw,
                                               int* __restrict__ end_adr, uint8_t* __restrict__ mark,
                                               int* __restrict__ rayend, unsigned long long* __restrict__ bounds) {
  const double cam[3] = { cx, cy, cz };
  double p[3] = { p0, p1, p2 };
  int flag;
  end_adr[i] = -1;
  if (!in_map_pos(g, p)) {
    // closetPointInMap, sdf_map.cpp:347-362
    double diff[3], min_t = 1000000;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      diff[k] = p[k] - cam[k];
      if (fabs(diff[k]) > 0) {
        const double t1 = (g.map_max[k] - cam[k]) / diff[k];
        if (t1 > 0 && t1 < min_t) min_t = t1;
        const double t2 = (g.origin[k] - cam[k]) / diff[k];
        if (t2 > 0 && t2 < min_t) min_t = t2;
      }
    }
#pragma unroll
    for (int k = 0; k < 3; ++k) p[k] = __dadd_rn(cam[k], __dmul_rn(min_t - 1e-3, diff[k]));
    const double d[3] = { p[0] - cam[0], p[1] - cam[1], p[2] - cam[2] };
    const double len = sqrt(__dadd_rn(__dadd_rn(__dmul_rn(d[0], d[0]), __dmul_rn(d[1], d[1])), __dmul_rn(d[2], d[2])));
    if (len > fc.max_ray_length) {
#pragma unroll
      for (int k = 0; k < 3; ++k) p[k] = __dadd_rn(__dmul_rn(d[k] / len, fc.max_ray_length), cam[k]);
    }
    if (p[2] < 0.2) return;
    flag = 0;
  } else {
    const double d[3] = { p[0] - cam[0], p[1] - cam[1], p[2] - cam[2] };
    const double len = sqrt(__dadd_rn(__dadd_rn(__dmul_rn(d[0], d[0]), __dmul_rn(d[1], d[1])), __dmul_rn(d[2], d[2])));
    if (len > fc.max_ray_length) {
#pragma unroll
      for (int k = 0; k < 3; ++k) p[k] = __dadd_rn(__dmul_rn(d[k] / len, fc.max_ray_length), cam[k]);
      if (p[2] < 0.2) return;
      flag = 0;
    } else
      flag = 1;
  }
  int idx[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) idx[k] = (int)floor((p[k] - g.origin[k]) * g.res_inv);
  if (idx[0] < 0 || idx[1] < 0 || idx[2] < 0 || idx[0] >= g.nx || idx[1] >= g.ny || idx[2] >= g.nz) return;
  const int64_t adr = addr_of(g, idx[0], idx[1], idx[2]);
  mark_or(mark, adr, flag ? 1u : 2u);  // setCacheOccupancy(vox_adr, tmp_flag), :243-257
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    atomicMin(&bounds[k], d2o(p[k]));
    atomicMax(&bounds[3 + k], d2o(p[k]));
    ptw[3 * i + k] = p[k];
  }
  end_adr[i] = (int)adr;
  atomicMin(&rayend[adr], i);  // the first point of this end voxel traces the ray (:303-306)
}

__global__ void classify_points_kernel(Geom g, FusionConsts fc, const float* __restrict__ pts, int stride, int n,
                                       double cx, double cy, double cz, double* __restrict__ ptw,
                                       int* __restrict__ end_adr, uint8_t* __restrict__ mark,
                                       int* __restrict__ rayend, unsigned long long* __restrict__ bounds) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float* q = pts + (int64_t)stride * i;
  classify_point(g, fc, i, (double)q[0], (double)q[1], (double)q[2], cx, cy, cz, ptw, end_adr, mark, rayend, bounds);
}

struct CamConsts {
  double fx, fy, cx, cy, inv_factor, maxdist, mindist;
  double R[9];
  int margin, skip, rows, cols, nu, nv;  // nu x nv sampled pixels
};

// MapROS::proessDepthImage (plan_env/src/map_ros.cpp:176-215) fused with the per-point part of inputPointCloud.
// Thread i = sampled pixel (v-major, then u): that order is the reference's point order with the skipped pixels
// (depth < mindist) left out, and leaving elements out does not change who is FIRST in a voxel.
__global__ void classify_depth_kernel(Geom g, FusionConsts fc, CamConsts cc, const uint16_t* __restrict__ img, double cx,
                                      double cy, double cz, double* __restrict__ ptw, int* __restrict__ end_adr,
                                      uint8_t* __restrict__ mark, int* __restrict__ rayend,
                                      unsigned long long* __restrict__ bounds, int* __restrict__ count) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= cc.nu * cc.nv) return;
  end_adr[i] = -1;
  const int v = cc.margin + (i / cc.nu) * cc.skip, u = cc.margin + (i % cc.nu) * cc.skip;
  const int64_t at = (int64_t)v * cc.cols + u;
  double depth = img[at] * cc.inv_factor;
  // the reference tests the pixel `skip` to the right of the one it just read (row_ptr advanced first, :190-198)
  const int64_t nx = at + cc.skip;
  const unsigned nxt = nx < (int64_t)cc.rows * cc.cols ? img[nx] : 0u;
  if (nxt == 0 || depth > cc.maxdist)
    depth = cc.maxdist;
  else if (depth < cc.mindist)
    return;
  atomicAdd(count, 1);
  const double pc[3] = { __dmul_rn(u - cc.cx, depth) / cc.fx, __dmul_rn(v - cc.cy, depth) / cc.fy, depth };
  float w[3];
#pragma unroll
  for (int k = 0; k < 3; ++k)
    w[k] = (float)__dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(cc.R[3 * k], pc[0]), __dmul_rn(cc.R[3 * k + 1], pc[1])),
                                      __dmul_rn(cc.R[3 * k + 2], pc[2])),
                            k == 0 ? cx : (k == 1 ? cy : cz));
  classify_point(g, fc, i, (double)w[0], (double)w[1], (double)w[2], cx, cy, cz, ptw, end_adr, mark, rayend, bounds);
}

__device__ __forceinline__ double intbound(double s, double ds) {  // raycast.cpp:14-23
  if (ds < 0) {
    s = -s;
    ds = -ds;
  }
  s = fmod(fmod(s, 1.0) + 1.0, 1.0);
  return (1 - s) / ds;
}

__global__ void raycast_kernel(Geom g, const double* __restrict__ ptw, const int* __restrict__ end_adr,
                               const int* __restrict__ rayend, int n, double cx, double cy, double cz,
                               uint8_t* __restrict__ mark) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int adr0 = end_adr[i];
  if (adr0 < 0 || rayend[adr0] != i) return;
  // RayCaster::input(pt_w, camera_pos), raycast.cpp:329-372
  const double res = g.res;
  const double s[3] = { ptw[3 * i] / res, ptw[3 * i + 1] / res, ptw[3 * i + 2] / res };
  const double e[3] = { cx / res, cy / res, cz / res };
  int x = (int)floor(s[0]), y = (int)floor(s[1]), z = (int)floor(s[2]);
  const int ex = (int)floor(e[0]), ey = (int)floor(e[1]), ez = (int)floor(e[2]);
  const double dx = ex - x, dy = ey - y, dz = ez - z;
  const int sx = dx == 0 ? 0 : (dx < 0 ? -1 : 1), sy = dy == 0 ? 0 : (dy < 0 ? -1 : 1), sz = dz == 0 ? 0 : (dz < 0 ? -1 : 1);
  double tmx = intbound(s[0], dx), tmy = intbound(s[1], dy), tmz = intbound(s[2], dz);
  const double tdx = ((double)sx) / dx, tdy = ((double)sy) / dy, tdz = ((double)sz) / dz;
  const double off[3] = { 0.5 - g.origin[0] / res, 0.5 - g.origin[1] / res, 0.5 - g.origin[2] / res };  // :323-327
  bool first = true;
  // caster_->nextId(idx); while (caster_->nextId(idx)) setCacheOccupancy(toAddress(idx), 0);  (:308-311)
  for (int guard = 0; guard < 4096; ++guard) {
    const int ix = (int)(x + off[0]), iy = (int)(y + off[1]), iz = (int)(z + off[2]);
    if (x == ex && y == ey && z == ez) break;  // nextId returns false at the camera voxel
    if (tmx < tmy) {
      if (tmx < tmz) {
        x += sx;
        tmx += tdx;
      } else {
        z += sz;
        tmz += tdz;
      }
    } else {
      if (tmy < tmz) {
        y += sy;
        tmy += tdy;
      } else {
        z += sz;
        tmz += tdz;
      }
    }
    if (!first && !(ix < 0 || iy < 0 || iz < 0 || ix >= g.nx || iy >= g.ny || iz >= g.nz))
      mark_or(mark, addr_of(g, ix, iy, iz), 2u);
    first = false;  // the first nextId (the end voxel itself) is discarded, :308
  }
}

__global__ void apply_kernel(Geom g, FusionConsts fc, int lo0, int lo1, int lo2, int n0, int n1, int n2,
                             uint8_t* __restrict__ mark, int* __restrict__ rayend, double* __restrict__ logodds,
                             uint8_t* __restrict__ occ) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (int64_t)n0 * n1 * n2) return;
  const int z = lo2 + (int)(t % n2), y = lo1 + (int)((t / n2) % n1), x = lo0 + (int)(t / ((int64_t)n2 * n1));
  const int64_t a = addr_of(g, x, y, z);
  const uint8_t mk = mark[a];
  if (!mk) return;
  mark[a] = 0;
  rayend[a] = 0x7fffffff;
  // :326-344: count_hit >= count_miss  <=>  the voxel was hit at least once
  const double upd = (mk & 1) ? fc.hit : fc.miss;
  double v = logodds[a];
  if (v < fc.clamp_min - 1e-3) v = fc.min_occ;
  v = fmin(fmax(__dadd_rn(v, upd), fc.clamp_min), fc.clamp_max);
  logodds[a] = v;
  int tri = FUELGPU_FREE;  // getOccupancy, sdf_map.h:194-200
  if (v < fc.clamp_min - 1e-3)
    tri = FUELGPU_UNKNOWN;
  else if (v > fc.min_occ)
    tri = FUELGPU_OCCUPIED;
  occ[a] = (uint8_t)((occ[a] & ~3u) | tri);
}

__global__ void fill_f64_kernel(double* p, int64_t n, double v) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) p[i] = v;
}
__global__ void fill_i32_kernel(int* p, int64_t n, int v) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) p[i] = v;
}
__global__ void logodds_to_occ_kernel(const double* __restrict__ lo, uint8_t* __restrict__ occ, int64_t n, double unk_thr,
                                      double occ_thr) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const double v = lo[i];
  int t = FUELGPU_FREE;
  if (v < unk_thr)
    t = FUELGPU_UNKNOWN;
  else if (v > occ_thr)
    t = FUELGPU_OCCUPIED;
  occ[i] = (uint8_t)((occ[i] & ~3u) | t);
}

}  // namespace

struct FusionState {
  double* logodds = nullptr;  // occupancy_buffer_ (fp64 log-odds), sdf_map.h:109
  int* rayend = nullptr;      // per voxel: first point index ending there this frame (flag_rayend_ analogue)
  uint8_t* mark = nullptr;    // per voxel: bit0 hit, bit1 missed this frame (count_hit_/count_miss_ analogue)
  unsigned long long* d_bounds = nullptr;
  int* d_count = nullptr;
  DevBuf<float> d_pts;  // per-frame points (or the depth image), grown on demand
  DevBuf<double> d_ptw;
  DevBuf<int> d_end;
  double update_min[3] = { 0, 0, 0 }, update_max[3] = { 0, 0, 0 };  // md_->update_min_/max_
  bool reset_updated_box = true;
  double clamp_max_log = 2.1972245773362196;  // logit(p_max = 0.90, algorithm.xml:48) until a frame says otherwise
};

static double logit(double p) { return log(p / (1 - p)); }

// log-odds consistent with an occupancy byte that was uploaded before the first fused frame (setOccupancyBuffer
// + upload): UNKNOWN -> clamp_min - unknown_flag, FREE -> clamp_min, OCCUPIED -> clamp_max (sdf_map.h:194-200 read
// backwards); a map that never saw an upload is all UNKNOWN, i.e. exactly initMap (sdf_map.cpp:56,64)
__global__ void seed_logodds_kernel(double* __restrict__ lo, const uint8_t* __restrict__ occ, int64_t n, double cmin,
                                    double cmax) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int t = occ[i] & 3;
  lo[i] = t == FUELGPU_OCCUPIED ? cmax : (t == FUELGPU_FREE ? cmin : cmin - 0.01);
}

int fusion_state_ensure(FuelMap* m, double p_min, double p_max) {
  if (m->fus) {
    m->fus->clamp_max_log = logit(p_max);
    return 0;
  }
  FusionState* f = new FusionState();
  m->fus = f;
  FUEL_CUDA(m, cudaMalloc(&f->logodds, sizeof(double) * m->nvox));
  FUEL_CUDA(m, cudaMalloc(&f->rayend, sizeof(int) * m->nvox));
  FUEL_CUDA(m, cudaMalloc(&f->mark, (m->nvox + 3) / 4 * 4));
  FUEL_CUDA(m, cudaMalloc(&f->d_bounds, sizeof(unsigned long long) * 6));
  FUEL_CUDA(m, cudaMalloc(&f->d_count, sizeof(int)));
  const unsigned nb = (unsigned)((m->nvox + 255) / 256);
  // initMap: occupancy_buffer_ = clamp_min_log_ - unknown_flag_ (sdf_map.cpp:56,64)
  f->clamp_max_log = logit(p_max);
  seed_logodds_kernel<<<nb, 256, 0, m->stream>>>(f->logodds, m->occ, m->nvox, logit(p_min), logit(p_max));
  fill_i32_kernel<<<nb, 256, 0, m->stream>>>(f->rayend, m->nvox, 0x7fffffff);
  FUEL_CUDA(m, cudaMemsetAsync(f->mark, 0, (m->nvox + 3) / 4 * 4, m->stream));
  FUEL_LAUNCHES(m, 2);
  FUEL_CUDA(m, cudaGetLastError());
  return 0;
}

// device log-odds volume (nullptr before the first fused frame) and the clamp the virtual ceiling writes
double* fusion_logodds_ptr(FuelMap* m, double* clamp_max_log) {
  if (!m->fus) return nullptr;
  if (clamp_max_log) *clamp_max_log = m->fus->clamp_max_log;
  return m->fus->logodds;
}

void fusion_state_destroy(FuelMap* m) {
  FusionState* f = m->fus;
  if (!f) return;
  void* ptrs[] = { f->logodds, f->rayend, f->mark, f->d_bounds, f->d_count };
  for (void* p : ptrs)
    if (p) cudaFree(p);
  f->d_pts.release();
  f->d_ptw.release();
  f->d_end.release();
  delete f;
  m->fus = nullptr;
}

int fusion_set_logodds(FuelMap* m, const double* logodds_host, double p_min, double p_occ) {
  int rc = fusion_state_ensure(m, p_min, 0.90);
  if (rc) return rc;
  FusionState* f = m->fus;
  FUEL_CUDA(m, cudaMemcpyAsync(f->logodds, logodds_host, sizeof(double) * m->nvox, cudaMemcpyHostToDevice, m->stream));
  logodds_to_occ_kernel<<<(unsigned)((m->nvox + 255) / 256), 256, 0, m->stream>>>(f->logodds, m->occ, m->nvox,
                                                                                 logit(p_min) - 1e-3, logit(p_occ));
  FUEL_LAUNCHES(m, 1);
  FUEL_CUDA(m, cudaGetLastError());
  FUEL_CUDA(m, cudaStreamSynchronize(m->stream));
  return 0;
}

int fusion_get_logodds(FuelMap* m, double* out) {
  if (!m->fus) return fuel_fail(m, FUELGPU_EINVAL, "no fused occupancy on the device yet");
  FUEL_CUDA(m, cudaMemcpyAsync(out, m->fus->logodds, sizeof(double) * m->nvox, cudaMemcpyDeviceToHost, m->stream));
  FUEL_CUDA(m, cudaStreamSynchronize(m->stream));
  return 0;
}

void fusion_get_updated_box(FuelMap* m, double bmin[3], double bmax[3], int reset) {
  FusionState* f = m->fus;
  for (int k = 0; k < 3; ++k) {
    bmin[k] = f ? f->update_min[k] : 0.0;
    bmax[k] = f ? f->update_max[k] : 0.0;
  }
  if (f && reset) f->reset_updated_box = true;  // getUpdatedBox(reset), sdf_map.cpp:491-495
}

// One frame.  Source = a point cloud (pts_host, stride, n) or, when cp != nullptr, a depth image (img_host, rows x cols)
// projected on the device; n is then the number of sampled pixels and *proj_cnt receives proj_points_cnt.
static int fusion_frame(FuelMap* m, const float* pts_host, int stride, int n, const uint16_t* img_host,
                        const FuelCameraParams* cp, int rows, int cols, const double* Rm, int32_t* proj_cnt,
                        const double cam[3], const FuelFusionParams* p, int32_t lbmin[3], int32_t lbmax[3]) {
  int rc = fusion_state_ensure(m, p->p_min, p->p_max);
  if (rc) return rc;
  FusionState* f = m->fus;
  const Geom& g = m->g;
  cudaStream_t s = m->stream;
  if (n == 0) return 0;  // :262
  int need = n;
  if (cp) {  // the image is staged in d_pts: 16 bytes per slot hold 8 pixels
    const int64_t px = ((int64_t)rows * cols + 7) / 8;
    need = px > n ? (int)px : n;
  }
  rc = f->d_pts.ensure(m, 4 * (size_t)need);  // also holds a uint16 image of <= 8 * need pixels
  if (!rc) rc = f->d_ptw.ensure(m, 3 * (size_t)need);
  if (!rc) rc = f->d_end.ensure(m, need);
  if (rc) return rc;
  FusionConsts fc;
  fc.max_ray_length = p->max_ray_length;
  fc.clamp_min = logit(p->p_min);
  fc.clamp_max = logit(p->p_max);
  fc.hit = logit(p->p_hit);
  fc.miss = logit(p->p_miss);
  fc.min_occ = logit(p->p_occ);
  // update box of this call starts at the camera position (:265-266)
  unsigned long long hb[6];
  for (int k = 0; k < 3; ++k) hb[k] = hb[3 + k] = d2o(cam[k]);
  FUEL_CUDA(m, cudaMemcpyAsync(f->d_bounds, hb, sizeof(hb), cudaMemcpyHostToDevice, s));
  const unsigned nb = (unsigned)((n + 127) / 128);
  if (!cp) {
    FUEL_CUDA(m, cudaMemcpyAsync(f->d_pts.p, pts_host, sizeof(float) * ((size_t)stride * (n - 1) + 3), cudaMemcpyHostToDevice, s));
    classify_points_kernel<<<nb, 128, 0, s>>>(g, fc, f->d_pts.p, stride, n, cam[0], cam[1], cam[2], f->d_ptw.p, f->d_end.p, f->mark,
                                              f->rayend, f->d_bounds);
  } else {
    CamConsts cc;
    cc.fx = cp->fx, cc.fy = cp->fy, cc.cx = cp->cx, cc.cy = cp->cy;
    cc.inv_factor = 1.0 / cp->k_depth_scaling_factor;  // :185
    cc.maxdist = cp->depth_filter_maxdist, cc.mindist = cp->depth_filter_mindist;
    for (int k = 0; k < 9; ++k) cc.R[k] = Rm[k];
    cc.margin = cp->depth_filter_margin, cc.skip = cp->skip_pixel, cc.rows = rows, cc.cols = cols;
    cc.nu = (cols - 2 * cc.margin + cc.skip - 1) / cc.skip;
    cc.nv = (rows - 2 * cc.margin + cc.skip - 1) / cc.skip;
    FUEL_CUDA(m, cudaMemsetAsync(f->d_count, 0, sizeof(int), s));
    FUEL_CUDA(m, cudaMemcpyAsync(f->d_pts.p, img_host, sizeof(uint16_t) * (size_t)rows * cols, cudaMemcpyHostToDevice, s));
    classify_depth_kernel<<<nb, 128, 0, s>>>(g, fc, cc, (const uint16_t*)f->d_pts.p, cam[0], cam[1], cam[2], f->d_ptw.p, f->d_end.p,
                                             f->mark, f->rayend, f->d_bounds, f->d_count);
  }
  raycast_kernel<<<nb, 128, 0, s>>>(g, f->d_ptw.p, f->d_end.p, f->rayend, n, cam[0], cam[1], cam[2], f->mark);
  FUEL_LAUNCHES(m, 2);
  // Every voxel touched this frame lies within max_ray_length of the camera (clipped points, :277-297) and
  // inside the map, so the dense sweep needs no device round trip for its extent.
  const int nmax[3] = { g.nx, g.ny, g.nz };
  int blo[3], bhi[3];
  for (int k = 0; k < 3; ++k) {
    const int tlo = (int)floor((cam[k] - p->max_ray_length - g.origin[k]) * g.res_inv) - 1;
    const int thi = (int)floor((cam[k] + p->max_ray_length - g.origin[k]) * g.res_inv) + 1;
    blo[k] = tlo > 0 ? tlo : 0;
    bhi[k] = thi < nmax[k] - 1 ? thi : nmax[k] - 1;
  }
  const int n0 = bhi[0] - blo[0] + 1, n1 = bhi[1] - blo[1] + 1, n2 = bhi[2] - blo[2] + 1;
  if (n0 > 0 && n1 > 0 && n2 > 0) {
    const int64_t nv = (int64_t)n0 * n1 * n2;
    apply_kernel<<<(unsigned)((nv + 255) / 256), 256, 0, s>>>(g, fc, blo[0], blo[1], blo[2], n0, n1, n2, f->mark, f->rayend,
                                                             f->logodds, m->occ);
    FUEL_LAUNCHES(m, 1);
  }
  FUEL_CUDA(m, cudaMemcpyAsync(hb, f->d_bounds, sizeof(hb), cudaMemcpyDeviceToHost, s));
  int cnt = n;
  if (cp) FUEL_CUDA(m, cudaMemcpyAsync(&cnt, f->d_count, sizeof(int), cudaMemcpyDeviceToHost, s));
  FUEL_CUDA(m, cudaStreamSynchronize(s));
  if (proj_cnt) *proj_cnt = cnt;
  if (cnt == 0) return 0;  // inputPointCloud returns before touching any box when point_num == 0 (:262)
  double umin[3], umax[3];
  for (int k = 0; k < 3; ++k) {
    umin[k] = o2d(hb[k]);
    umax[k] = o2d(hb[3 + k]);
  }
  if (f->reset_updated_box) {  // :267-271
    for (int k = 0; k < 3; ++k) f->update_min[k] = f->update_max[k] = cam[k];
    f->reset_updated_box = false;
  }
  // local bound (:313-318) and accumulated updated box (:321-324)
  for (int k = 0; k < 3; ++k) {
    const double infl = k < 2 ? p->local_bound_inflate : 0.0;
    int hi = (int)floor((umax[k] + infl - g.origin[k]) * g.res_inv);
    int lo = (int)floor((umin[k] - infl - g.origin[k]) * g.res_inv);
    hi = hi < nmax[k] - 1 ? hi : nmax[k] - 1;
    hi = hi > 0 ? hi : 0;
    lo = lo < nmax[k] - 1 ? lo : nmax[k] - 1;
    lo = lo > 0 ? lo : 0;
    lbmin[k] = lo;
    lbmax[k] = hi;
    f->update_min[k] = umin[k] < f->update_min[k] ? umin[k] : f->update_min[k];
    f->update_max[k] = umax[k] > f->update_max[k] ? umax[k] : f->update_max[k];
  }
  FUEL_CUDA(m, cudaGetLastError());
  return 0;
}

int fusion_input_impl(FuelMap* m, const float* pts_host, int stride, int n, const double cam[3], const FuelFusionParams* p,
                      int32_t lbmin[3], int32_t lbmax[3]) {
  return fusion_frame(m, pts_host, stride, n, nullptr, nullptr, 0, 0, nullptr, nullptr, cam, p, lbmin, lbmax);
}

int fusion_input_depth_impl(FuelMap* m, const uint16_t* img_host, int rows, int cols, const FuelCameraParams* cp,
                            const double R[9], const double cam[3], const FuelFusionParams* p, int32_t lbmin[3],
                            int32_t lbmax[3], int32_t* proj_cnt) {
  const int nu = (cols - 2 * cp->depth_filter_margin + cp->skip_pixel - 1) / cp->skip_pixel;
  const int nv = (rows - 2 * cp->depth_filter_margin + cp->skip_pixel - 1) / cp->skip_pixel;
  if (proj_cnt) *proj_cnt = 0;
  if (nu <= 0 || nv <= 0) return 0;
  return fusion_frame(m, nullptr, 0, nu * nv, img_host, cp, rows, cols, R, proj_cnt, cam, p, lbmin, lbmax);
}
