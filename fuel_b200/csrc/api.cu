// api.cu -- the extern "C" boundary of libfuelgpu (see include/fuelgpu.h).
#include "common.cuh"

#include <vector>

#include <math.h>
#include <stddef.h>
#include <new>

thread_local char g_fuelgpu_err[512] = "";

namespace {

// host occupancy -> resident byte: bits0-1 tri-state (sdf_map.h:194-200), bit2 inflate
__global__ void ingest_logodds_kernel(const int8_t* __restrict__ inflate, const double* __restrict__ lo,
                                      uint8_t* __restrict__ occ, int64_t n, double unknown_thr,
                                      double occ_thr) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const double v = lo[i];
  int t = FUELGPU_FREE;
  if (v < unknown_thr)
    t = FUELGPU_UNKNOWN;
  else if (v > occ_thr)
    t = FUELGPU_OCCUPIED;
  occ[i] = (uint8_t)(t | ((inflate[i] == 1) ? 4 : 0));
}

__global__ void ingest_tri_kernel(const int8_t* __restrict__ inflate, const uint8_t* __restrict__ tri,
                                  uint8_t* __restrict__ occ, int64_t n) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  occ[i] = (uint8_t)((tri[i] & 3) | ((inflate[i] == 1) ? 4 : 0));
}

__global__ void f32_to_f64_kernel(const float* __restrict__ in, double* __restrict__ out, int64_t n,
                                  double inf_value) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float v = in[i];
  out[i] = isinf(v) ? (v > 0 ? inf_value : -inf_value) : (double)v;
}

// [G][nx][ny][nzl] z-slabs (the all-gather of a z-sharded ESDF) -> [nx][ny][G*nzl]
__global__ void slabs_to_volume_kernel(const float* __restrict__ slabs, float* __restrict__ dist, int64_t nxy, int nzl,
                                       int G) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t total = nxy * nzl * G;
  if (i >= total) return;
  const int nz = nzl * G;
  const int z = (int)(i % nz);
  const int64_t xy = i / nz;
  const int gsl = z / nzl;
  dist[i] = slabs[((int64_t)gsl * nxy + xy) * nzl + (z - gsl * nzl)];
}

__global__ void clear_flags_kernel(int8_t* flag, const int* __restrict__ addr, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) flag[addr[i]] = 0;
}

int ensure_stage(FuelMap* m, size_t bytes) {
  if (bytes <= m->stage_bytes) return 0;
  if (m->stage) cudaFree(m->stage);
  m->stage = nullptr;
  m->stage_bytes = 0;
  FUEL_CUDA(m, cudaMalloc(&m->stage, bytes));
  m->stage_bytes = bytes;
  return 0;
}

int ensure_bs(FuelMap* m, size_t bytes) {
  if (bytes <= m->bs_bytes) return 0;
  if (m->bs_buf) cudaFree(m->bs_buf);
  m->bs_buf = nullptr;
  m->bs_bytes = 0;
  FUEL_CUDA(m, cudaMalloc(&m->bs_buf, bytes));
  m->bs_bytes = bytes;
  return 0;
}

static int ensure_bs_pin(FuelMap* m, size_t bytes) {
  if (bytes <= m->bs_pin_bytes) return 0;
  if (m->bs_pin) cudaFreeHost(m->bs_pin);
  m->bs_pin = nullptr;
  m->bs_pin_bytes = 0;
  FUEL_CUDA(m, cudaMallocHost(&m->bs_pin, bytes + bytes / 4));
  m->bs_pin_bytes = bytes + bytes / 4;
  return 0;
}

int check_box(FuelMap* m, const int32_t bmin[3], const int32_t bmax[3], int lo[3], int hi[3]) {
  const int n[3] = { m->g.nx, m->g.ny, m->g.nz };
  for (int i = 0; i < 3; ++i) {
    lo[i] = bmin ? bmin[i] : 0;
    hi[i] = bmax ? bmax[i] : n[i] - 1;
    if (lo[i] < 0 || hi[i] >= n[i] || lo[i] > hi[i])
      return fuel_fail(m, FUELGPU_EINVAL, "box outside the map or empty on axis %s%lld", "", i);
  }
  return 0;
}

}  // namespace

extern "C" {

const char* fuelgpu_version(void) { return "fuelgpu 0.1 (sm_90a)"; }

const char* fuelgpu_last_error(const FuelMap* map) { return map ? map->err : g_fuelgpu_err; }

int fuelgpu_device_info(int device_id, char* name, int name_len, int* cc_major, int* cc_minor) {
  int count = 0;
  if (cudaGetDeviceCount(&count) != cudaSuccess || count <= 0 || device_id >= count)
    return fuel_fail(nullptr, FUELGPU_ENODEVICE, "no CUDA device %s(id %lld)", "", device_id);
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, device_id) != cudaSuccess)
    return fuel_fail(nullptr, FUELGPU_ECUDA, "cudaGetDeviceProperties failed");
  if (name && name_len > 0) {
    strncpy(name, prop.name, name_len - 1);
    name[name_len - 1] = 0;
  }
  if (cc_major) *cc_major = prop.major;
  if (cc_minor) *cc_minor = prop.minor;
  return prop.multiProcessorCount;
}

int fuelgpu_map_create(const FuelGridDesc* grid, int device_id, FuelMap** out) {
  if (!grid || !out) return fuel_fail(nullptr, FUELGPU_EINVAL, "null argument");
  *out = nullptr;
  int count = 0;
  if (cudaGetDeviceCount(&count) != cudaSuccess || count <= 0)
    return fuel_fail(nullptr, FUELGPU_ENODEVICE,
                     "no CUDA device: libfuelgpu has no CPU fallback (the reference CPU path is the "
                     "oracle, not the product)");
  if (device_id < 0 || device_id >= count)
    return fuel_fail(nullptr, FUELGPU_ENODEVICE, "device id %s%lld out of range", "", device_id);
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, device_id) != cudaSuccess)
    return fuel_fail(nullptr, FUELGPU_ECUDA, "cudaGetDeviceProperties failed");
  if (prop.major != 9 || prop.minor != 0)
    return fuel_fail(nullptr, FUELGPU_ENODEVICE, "device is not sm_90 (Hopper H100): %s", prop.name);
  for (int i = 0; i < 3; ++i)
    if (grid->n[i] < 1 || grid->n[i] > 1024)
      return fuel_fail(nullptr, FUELGPU_EINVAL, "grid extent must be in 1..1024 per axis");
  if (!(grid->resolution > 0)) return fuel_fail(nullptr, FUELGPU_EINVAL, "resolution must be > 0");
  const int64_t nvox = (int64_t)grid->n[0] * grid->n[1] * grid->n[2];
  if (nvox >= (1ll << 31)) return fuel_fail(nullptr, FUELGPU_EINVAL, "more than 2^31 voxels");

  FuelMap* m = new (std::nothrow) FuelMap();
  if (!m) return fuel_fail(nullptr, FUELGPU_ENOMEM, "host allocation failed");
  memset(m, 0, sizeof(*m));
  m->desc = *grid;
  m->dev = device_id;
  m->sm_count = prop.multiProcessorCount;
  m->nvox = nvox;
  Geom& g = m->g;
  g.nx = grid->n[0];
  g.ny = grid->n[1];
  g.nz = grid->n[2];
  g.res = grid->resolution;
  g.res_inv = 1 / grid->resolution;  // sdf_map.cpp:33
  for (int i = 0; i < 3; ++i) {
    g.origin[i] = grid->origin[i];
    // map_max_boundary_ = map_origin_ + map_size_ (sdf_map.cpp:34-39)
    g.map_max[i] = grid->origin[i] + (grid->map_size[i] > 0.0 ? grid->map_size[i] : grid->n[i] * grid->resolution);
    g.box_mind[i] = grid->box_mind[i];
    g.box_maxd[i] = grid->box_maxd[i];
    // posToIndex(box_mind_/box_maxd_), sdf_map.cpp:83-84
    g.box_min[i] = (int)floor((grid->box_mind[i] - grid->origin[i]) * g.res_inv);
    g.box_max[i] = (int)floor((grid->box_maxd[i] - grid->origin[i]) * g.res_inv);
  }

#define CR(expr)                                                                        \
  do {                                                                                  \
    cudaError_t _e = (expr);                                                            \
    if (_e != cudaSuccess) {                                                            \
      snprintf(g_fuelgpu_err, 512, "map_create: %s: %s", #expr, cudaGetErrorString(_e)); \
      fuelgpu_map_destroy(m);                                                           \
      return _e == cudaErrorMemoryAllocation ? FUELGPU_ENOMEM : FUELGPU_ECUDA;          \
    }                                                                                   \
  } while (0)
  CR(cudaSetDevice(device_id));
  CR(cudaStreamCreateWithFlags(&m->own_stream, cudaStreamNonBlocking));
  m->stream = m->own_stream;
  CR(cudaStreamCreateWithFlags(&m->copy_stream, cudaStreamNonBlocking));
  CR(cudaEventCreateWithFlags(&m->copy_ev, cudaEventDisableTiming));
  CR(cudaStreamCreateWithFlags(&m->in_stream, cudaStreamNonBlocking));
  CR(cudaEventCreateWithFlags(&m->in_ev, cudaEventDisableTiming));
  for (int t = 0; t < T_COUNT; ++t) {
    CR(cudaEventCreate(&m->ev0[t]));
    CR(cudaEventCreate(&m->ev1[t]));
  }
  CR(cudaMalloc(&m->occ, nvox));
  CR(cudaMalloc(&m->dist, sizeof(float) * nvox));
  CR(cudaMalloc(&m->flag, nvox));
  {
    size_t rec_bytes = 0;
    int wc = 0;
    esdf_tile_scratch_sizes(g.nx, g.ny, g.nz, &rec_bytes, &m->esdf_p_bytes, &wc);
    CR(cudaMalloc(&m->esdf_rec, rec_bytes));
    CR(cudaMalloc(&m->esdf_p[0], m->esdf_p_bytes));
    CR(cudaMalloc(&m->esdf_p[1], m->esdf_p_bytes));
    CR(cudaStreamCreateWithFlags(&m->esdf_aux, cudaStreamNonBlocking));
    CR(cudaEventCreateWithFlags(&m->esdf_ev[0], cudaEventDisableTiming));
    CR(cudaEventCreateWithFlags(&m->esdf_ev[1], cudaEventDisableTiming));
  }
  // initMap: occupancy unknown, inflate 0, distance default_dist (0.0, algorithm.xml:41), flags 0
  CR(cudaMemsetAsync(m->occ, 0, nvox, m->stream));
  CR(cudaMemsetAsync(m->dist, 0, sizeof(float) * nvox, m->stream));
  CR(cudaMemsetAsync(m->flag, 0, nvox, m->stream));
#undef CR
  int rc = frontier_state_create(m);
  if (rc) {
    strncpy(g_fuelgpu_err, m->err, 511);
    fuelgpu_map_destroy(m);
    return rc;
  }
  if (cudaStreamSynchronize(m->stream) != cudaSuccess) {
    snprintf(g_fuelgpu_err, 512, "map_create: stream sync failed");
    fuelgpu_map_destroy(m);
    return FUELGPU_ECUDA;
  }
  m->err[0] = 0;
  *out = m;
  return 0;
}

int fuelgpu_map_destroy(FuelMap* m) {
  if (!m) return 0;
  cudaSetDevice(m->dev);
  if (m->own_stream) cudaStreamSynchronize(m->own_stream);
  frontier_state_destroy(m);
  fusion_state_destroy(m);
  if (m->bs_pin) cudaFreeHost(m->bs_pin);
  if (m->esdf_aux) {
    cudaStreamSynchronize(m->esdf_aux);
    cudaStreamDestroy(m->esdf_aux);
  }
  for (int i = 0; i < 2; ++i)
    if (m->esdf_ev[i]) cudaEventDestroy(m->esdf_ev[i]);
  void* ptrs[] = { m->occ,       m->dist,      m->dist_neg, m->flag,   m->esdf_rec,
                   m->esdf_p[0], m->esdf_p[1], m->stage,    m->bs_buf, m->fr_scr, m->bs_grad };
  for (void* p : ptrs)
    if (p) cudaFree(p);
  for (int t = 0; t < T_COUNT; ++t) {
    if (m->ev0[t]) cudaEventDestroy(m->ev0[t]);
    if (m->ev1[t]) cudaEventDestroy(m->ev1[t]);
  }
  if (m->copy_stream) {
    cudaStreamSynchronize(m->copy_stream);
    cudaStreamDestroy(m->copy_stream);
  }
  if (m->copy_ev) cudaEventDestroy(m->copy_ev);
  if (m->in_stream) {
    cudaStreamSynchronize(m->in_stream);
    cudaStreamDestroy(m->in_stream);
  }
  if (m->in_ev) cudaEventDestroy(m->in_ev);
  if (m->own_stream) cudaStreamDestroy(m->own_stream);
  delete m;
  return 0;
}

int fuelgpu_map_set_stream(FuelMap* m, void* cuda_stream) {
  if (!m) return fuel_fail(nullptr, FUELGPU_EINVAL, "null map");
  m->stream = cuda_stream ? (cudaStream_t)cuda_stream : m->own_stream;
  return 0;
}

int fuelgpu_map_synchronize(FuelMap* m) {
  if (!m) return fuel_fail(nullptr, FUELGPU_EINVAL, "null map");
  FUEL_CUDA(m, cudaStreamSynchronize(m->stream));
  FUEL_CUDA(m, cudaStreamSynchronize(m->copy_stream));
  FUEL_CUDA(m, cudaStreamSynchronize(frontier_stream_raw(m)));
  return 0;
}

int fuelgpu_map_device_ptrs(FuelMap* m, void** occ, void** dist, void** flag) {
  if (!m) return fuel_fail(nullptr, FUELGPU_EINVAL, "null map");
  if (occ) *occ = m->occ;
  if (dist) *dist = m->dist;
  if (flag) *flag = m->flag;
  return 0;
}

int fuelgpu_map_last_timing(FuelMap* m, float ms[8]) {
  if (!m || !ms) return fuel_fail(m, FUELGPU_EINVAL, "null argument");
  for (int t = 0; t < T_COUNT; ++t) {
    ms[t] = -1.f;
    if (m->ev_valid[t]) {
      if (cudaEventSynchronize(m->ev1[t]) == cudaSuccess) cudaEventElapsedTime(&ms[t], m->ev0[t], m->ev1[t]);
    }
  }
  return 0;
}

int fuelgpu_map_last_timeline(FuelMap* m, float start_ms[8], float end_ms[8]) {
  if (!m || !start_ms || !end_ms) return fuel_fail(m, FUELGPU_EINVAL, "null argument");
  for (int t = 0; t < T_COUNT; ++t) {
    start_ms[t] = end_ms[t] = -1.f;
    if (!m->ev_valid[t] || !m->ev_valid[T_UPLOAD]) continue;
    if (cudaEventSynchronize(m->ev1[t]) != cudaSuccess) continue;
    if (cudaEventElapsedTime(&start_ms[t], m->ev0[T_UPLOAD], m->ev0[t]) != cudaSuccess ||
        cudaEventElapsedTime(&end_ms[t], m->ev0[T_UPLOAD], m->ev1[t]) != cudaSuccess) {
      cudaGetLastError();  // (a stage older than the last upload: not on this timeline)
      start_ms[t] = end_ms[t] = -1.f;
    }
  }
  return 0;
}

int fuelgpu_host_register(void* ptr, uint64_t bytes) {
  if (!ptr || !bytes) return fuel_fail(nullptr, FUELGPU_EINVAL, "null argument");
  cudaError_t e = cudaHostRegister(ptr, bytes, cudaHostRegisterDefault);
  if (e == cudaErrorHostMemoryAlreadyRegistered) {
    cudaGetLastError();
    return 0;
  }
  FUEL_CUDA(nullptr, e);
  return 0;
}

int fuelgpu_host_unregister(void* ptr) {
  if (!ptr) return fuel_fail(nullptr, FUELGPU_EINVAL, "null argument");
  cudaError_t e = cudaHostUnregister(ptr);
  if (e == cudaErrorHostMemoryNotRegistered) {
    cudaGetLastError();
    return 0;
  }
  FUEL_CUDA(nullptr, e);
  return 0;
}

static int upload_occupancy_impl(FuelMap* m, const int8_t* inflate, const double* logodds, const uint8_t* tristate,
                                 double clamp_min_log, double min_occupancy_log, const int32_t bmin[3],
                                 const int32_t bmax[3], bool wait) {
  if (!m || !inflate) return fuel_fail(m, FUELGPU_EINVAL, "null argument");
  if ((logodds == nullptr) == (tristate == nullptr))
    return fuel_fail(m, FUELGPU_EINVAL, "give exactly one of logodds / tristate");
  int lo[3], hi[3];
  int rc = check_box(m, bmin, bmax, lo, hi);
  if (rc) return rc;
  FUEL_CUDA(m, cudaSetDevice(m->dev));
  const int64_t plane = (int64_t)m->g.ny * m->g.nz;
  const int64_t off = (int64_t)lo[0] * plane;
  const int64_t cnt = (int64_t)(hi[0] - lo[0] + 1) * plane;
  const size_t inf_bytes = ((size_t)cnt + 7) & ~(size_t)7;  // keeps the fp64 region 8-byte aligned
  rc = ensure_stage(m, inf_bytes + (size_t)cnt * (logodds ? 8 : 1));
  if (rc) return rc;
  frontier_order_writer(m);
  tbegin(m, T_UPLOAD);
  int8_t* d_inf = (int8_t*)m->stage;
  FUEL_CUDA(m, cudaMemcpyAsync(d_inf, inflate + off, cnt, cudaMemcpyHostToDevice, m->stream));
  const unsigned nb = (unsigned)((cnt + 255) / 256);
  if (logodds) {
    double* d_lo = (double*)((uint8_t*)m->stage + inf_bytes);
    FUEL_CUDA(m, cudaMemcpyAsync(d_lo, logodds + off, cnt * 8, cudaMemcpyHostToDevice, m->stream));
    ingest_logodds_kernel<<<nb, 256, 0, m->stream>>>(d_inf, d_lo, m->occ + off, cnt, clamp_min_log - 1e-3,
                                                     min_occupancy_log);
  } else {
    uint8_t* d_tri = (uint8_t*)m->stage + inf_bytes;
    FUEL_CUDA(m, cudaMemcpyAsync(d_tri, tristate + off, cnt, cudaMemcpyHostToDevice, m->stream));
    ingest_tri_kernel<<<nb, 256, 0, m->stream>>>(d_inf, d_tri, m->occ + off, cnt);
  }
  FUEL_LAUNCHES(m, 1);
  FUEL_CUDA(m, cudaGetLastError());
  tend(m, T_UPLOAD);
  if (wait) FUEL_CUDA(m, cudaStreamSynchronize(m->stream));  // host buffers may be reused by the caller
  return 0;
}

int fuelgpu_map_upload_occupancy(FuelMap* m, const int8_t* inflate, const double* logodds, const uint8_t* tristate,
                                 double clamp_min_log, double min_occupancy_log, const int32_t bmin[3],
                                 const int32_t bmax[3]) {
  return upload_occupancy_impl(m, inflate, logodds, tristate, clamp_min_log, min_occupancy_log, bmin, bmax, true);
}

int fuelgpu_map_upload_occupancy_async(FuelMap* m, const int8_t* inflate, const double* logodds, const uint8_t* tristate,
                                       double clamp_min_log, double min_occupancy_log, const int32_t bmin[3],
                                       const int32_t bmax[3]) {
  return upload_occupancy_impl(m, inflate, logodds, tristate, clamp_min_log, min_occupancy_log, bmin, bmax, false);
}

__global__ void split_occ_kernel(const uint8_t* __restrict__ occ, int8_t* __restrict__ inf, uint8_t* __restrict__ tri,
                                 int64_t n) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint8_t o = occ[i];
  if (inf) inf[i] = (o >> 2) & 1;
  if (tri) tri[i] = o & 3;
}

int fuelgpu_map_inflate(FuelMap* m, const int32_t bmin[3], const int32_t bmax[3], int32_t inf_step,
                        int32_t virtual_ceil_idx) {
  if (!m) return fuel_fail(nullptr, FUELGPU_EINVAL, "null map");
  if (inf_step < 0 || inf_step > 16) return fuel_fail(m, FUELGPU_EINVAL, "inf_step out of range");
  int lo[3], hi[3];
  int rc = check_box(m, bmin, bmax, lo, hi);
  if (rc) return rc;
  FUEL_CUDA(m, cudaSetDevice(m->dev));
  frontier_order_writer(m);
  return map_inflate_impl(m, lo, hi, inf_step, virtual_ceil_idx);
}

int fuelgpu_map_input_point_cloud(FuelMap* m, const float* points, int32_t point_num, int32_t point_stride,
                                  const double camera_pos[3],
                                  const FuelFusionParams* p, int32_t local_bound_min[3], int32_t local_bound_max[3]) {
  if (!m || !camera_pos || !p || !local_bound_min || !local_bound_max || (point_num > 0 && !points))
    return fuel_fail(m, FUELGPU_EINVAL, "null argument");
  if (point_num < 0) return fuel_fail(m, FUELGPU_EINVAL, "negative point count");
  if (point_stride != 3 && point_stride != 4) return fuel_fail(m, FUELGPU_EINVAL, "point_stride must be 3 (packed xyz) or 4 (pcl::PointXYZ)");
  const double pr[5] = { p->p_hit, p->p_miss, p->p_min, p->p_max, p->p_occ };
  for (double v : pr)
    if (!(v > 0.0 && v < 1.0)) return fuel_fail(m, FUELGPU_EINVAL, "fusion probabilities must lie in (0,1)");
  if (!(p->max_ray_length > 0.0)) return fuel_fail(m, FUELGPU_EINVAL, "max_ray_length must be positive");
  FUEL_CUDA(m, cudaSetDevice(m->dev));
  frontier_order_writer(m);
  return fusion_input_impl(m, points, point_stride, point_num, camera_pos, p, local_bound_min, local_bound_max);
}

int fuelgpu_map_input_depth_image(FuelMap* m, const uint16_t* depth, int32_t rows, int32_t cols, const FuelCameraParams* c,
                                  const double camera_R[9], const double camera_pos[3], const FuelFusionParams* p,
                                  int32_t local_bound_min[3], int32_t local_bound_max[3], int32_t* proj_points_cnt) {
  if (!m || !depth || !c || !camera_R || !camera_pos || !p || !local_bound_min || !local_bound_max)
    return fuel_fail(m, FUELGPU_EINVAL, "null argument");
  if (rows <= 0 || cols <= 0 || rows > 8192 || cols > 8192) return fuel_fail(m, FUELGPU_EINVAL, "image size out of range");
  if (c->skip_pixel < 1 || c->depth_filter_margin < 0 || !(c->fx != 0.0) || !(c->fy != 0.0) || !(c->k_depth_scaling_factor > 0.0))
    return fuel_fail(m, FUELGPU_EINVAL, "bad camera parameters");
  const double pr[5] = { p->p_hit, p->p_miss, p->p_min, p->p_max, p->p_occ };
  for (double v : pr)
    if (!(v > 0.0 && v < 1.0)) return fuel_fail(m, FUELGPU_EINVAL, "fusion probabilities must lie in (0,1)");
  if (!(p->max_ray_length > 0.0)) return fuel_fail(m, FUELGPU_EINVAL, "max_ray_length must be positive");
  FUEL_CUDA(m, cudaSetDevice(m->dev));
  frontier_order_writer(m);
  return fusion_input_depth_impl(m, depth, rows, cols, c, camera_R, camera_pos, p, local_bound_min, local_bound_max,
                                 proj_points_cnt);
}

int fuelgpu_map_get_updated_box(FuelMap* m, double bmin[3], double bmax[3], int32_t reset) {
  if (!m || !bmin || !bmax) return fuel_fail(m, FUELGPU_EINVAL, "null argument");
  fusion_get_updated_box(m, bmin, bmax, reset);
  return FUELGPU_OK;
}

int fuelgpu_map_set_logodds(FuelMap* m, const double* logodds, double p_min, double p_occ) {
  if (!m || !logodds) return fuel_fail(m, FUELGPU_EINVAL, "null argument");
  if (!(p_min > 0.0 && p_min < 1.0 && p_occ > 0.0 && p_occ < 1.0)) return fuel_fail(m, FUELGPU_EINVAL, "probability out of (0,1)");
  FUEL_CUDA(m, cudaSetDevice(m->dev));
  frontier_order_writer(m);
  return fusion_set_logodds(m, logodds, p_min, p_occ);
}

int fuelgpu_map_get_logodds(FuelMap* m, double* logodds) {
  if (!m || !logodds) return fuel_fail(m, FUELGPU_EINVAL, "null argument");
  FUEL_CUDA(m, cudaSetDevice(m->dev));
  return fusion_get_logodds(m, logodds);
}

int fuelgpu_map_download_occupancy(FuelMap* m, int8_t* inflate, uint8_t* tristate) {
  if (!m || (!inflate && !tristate)) return fuel_fail(m, FUELGPU_EINVAL, "null argument");
  FUEL_CUDA(m, cudaSetDevice(m->dev));
  int rc = ensure_stage(m, (size_t)m->nvox * 2);
  if (rc) return rc;
  int8_t* d_inf = (int8_t*)m->stage;
  uint8_t* d_tri = (uint8_t*)m->stage + m->nvox;
  split_occ_kernel<<<(unsigned)((m->nvox + 255) / 256), 256, 0, m->stream>>>(m->occ, d_inf, d_tri, m->nvox);
  FUEL_LAUNCHES(m, 1);
  FUEL_CUDA(m, cudaGetLastError());
  if (inflate) FUEL_CUDA(m, cudaMemcpyAsync(inflate, d_inf, m->nvox, cudaMemcpyDeviceToHost, m->stream));
  if (tristate) FUEL_CUDA(m, cudaMemcpyAsync(tristate, d_tri, m->nvox, cudaMemcpyDeviceToHost, m->stream));
  FUEL_CUDA(m, cudaStreamSynchronize(m->stream));
  return 0;
}

int fuelgpu_esdf_update(FuelMap* m, const int32_t bmin[3], const int32_t bmax[3], int flags) {
  if (!m) return fuel_fail(nullptr, FUELGPU_EINVAL, "null map");
  int lo[3], hi[3];
  int rc = check_box(m, bmin, bmax, lo, hi);
  if (rc) return rc;
  FUEL_CUDA(m, cudaSetDevice(m->dev));
  tbegin(m, T_ESDF);
  rc = esdf_update_impl(m, lo, hi, flags);
  tend(m, T_ESDF);
  m->dist_ev_ok = rc == 0;
  return rc;
}

int fuelgpu_esdf_download(FuelMap* m, const int32_t bmin[3], const int32_t bmax[3], float* out_f32,
                          double* out_f64) {
  if (!m) return fuel_fail(nullptr, FUELGPU_EINVAL, "null map");
  if ((out_f32 == nullptr) == (out_f64 == nullptr))
    return fuel_fail(m, FUELGPU_EINVAL, "give exactly one of out_f32 / out_f64");
  int lo[3], hi[3];
  int rc = check_box(m, bmin, bmax, lo, hi);
  if (rc) return rc;
  FUEL_CUDA(m, cudaSetDevice(m->dev));
  const int64_t plane = (int64_t)m->g.ny * m->g.nz;
  const int64_t off = (int64_t)lo[0] * plane;
  const int64_t cnt = (int64_t)(hi[0] - lo[0] + 1) * plane;
  tbegin(m, T_DOWNLOAD);
  if (out_f32) {
    FUEL_CUDA(m, cudaMemcpyAsync(out_f32 + off, m->dist + off, cnt * 4, cudaMemcpyDeviceToHost, m->stream));
  } else {
    rc = ensure_stage(m, (size_t)cnt * 8);
    if (rc) return rc;
    f32_to_f64_kernel<<<(unsigned)((cnt + 255) / 256), 256, 0, m->stream>>>(
        m->dist + off, (double*)m->stage, cnt, m->g.res * sqrt(1.7976931348623157e308));
    FUEL_LAUNCHES(m, 1);
    FUEL_CUDA(m, cudaGetLastError());
    FUEL_CUDA(m, cudaMemcpyAsync(out_f64 + off, m->stage, cnt * 8, cudaMemcpyDeviceToHost, m->stream));
  }
  tend(m, T_DOWNLOAD);
  FUEL_CUDA(m, cudaStreamSynchronize(m->stream));
  return 0;
}

int fuelgpu_esdf_set_from_slabs_dev(FuelMap* m, const void* slabs_dev, int32_t n_slabs) {
  if (!m || !slabs_dev) return fuel_fail(m, FUELGPU_EINVAL, "null argument");
  if (n_slabs < 1 || m->g.nz % n_slabs) return fuel_fail(m, FUELGPU_EINVAL, "nz is not a multiple of the slab count");
  FUEL_CUDA(m, cudaSetDevice(m->dev));
  if (n_slabs == 1) {
    FUEL_CUDA(m, cudaMemcpyAsync(m->dist, slabs_dev, sizeof(float) * m->nvox, cudaMemcpyDeviceToDevice, m->stream));
  } else {
    slabs_to_volume_kernel<<<(unsigned)((m->nvox + 255) / 256), 256, 0, m->stream>>>(
        (const float*)slabs_dev, m->dist, (int64_t)m->g.nx * m->g.ny, m->g.nz / n_slabs, n_slabs);
    FUEL_LAUNCHES(m, 1);
    FUEL_CUDA(m, cudaGetLastError());
  }
  m->dist_ev_ok = false;  // (the field no longer comes from the last fuelgpu_esdf_update)
  return 0;
}

int fuelgpu_esdf_download_async(FuelMap* m, const int32_t bmin[3], const int32_t bmax[3], float* out_f32) {
  if (!m || !out_f32) return fuel_fail(m, FUELGPU_EINVAL, "null argument");
  int lo[3], hi[3];
  int rc = check_box(m, bmin, bmax, lo, hi);
  if (rc) return rc;
  FUEL_CUDA(m, cudaSetDevice(m->dev));
  const int64_t plane = (int64_t)m->g.ny * m->g.nz;
  const int64_t off = (int64_t)lo[0] * plane;
  const int64_t cnt = (int64_t)(hi[0] - lo[0] + 1) * plane;
  if (m->dist_ev_ok) {  // after the ESDF update that wrote the field -- not after whatever the main stream got since (a solve)
    FUEL_CUDA(m, cudaStreamWaitEvent(m->copy_stream, m->ev1[T_ESDF], 0));
  } else {
    FUEL_CUDA(m, cudaEventRecord(m->copy_ev, m->stream));
    FUEL_CUDA(m, cudaStreamWaitEvent(m->copy_stream, m->copy_ev, 0));
  }
  tbegin(m, T_DOWNLOAD, m->copy_stream);
  FUEL_CUDA(m, cudaMemcpyAsync(out_f32 + off, m->dist + off, cnt * 4, cudaMemcpyDeviceToHost, m->copy_stream));
  tend(m, T_DOWNLOAD, m->copy_stream);
  return 0;
}

int fuelgpu_esdf_sample(FuelMap* m, int64_t n, const double* pos, double* dist, double* grad) {
  if (!m || (n > 0 && (!pos || !dist || !grad))) return fuel_fail(m, FUELGPU_EINVAL, "null argument");
  if (n <= 0) return 0;
  FUEL_CUDA(m, cudaSetDevice(m->dev));
  int rc = ensure_bs(m, (size_t)n * 7 * sizeof(double));
  if (rc) return rc;
  double* d_pos = (double*)m->bs_buf;
  double* d_d = d_pos + 3 * n;
  double* d_g = d_d + n;
  FUEL_CUDA(m, cudaMemcpyAsync(d_pos, pos, sizeof(double) * 3 * n, cudaMemcpyHostToDevice, m->stream));
  rc = esdf_sample_impl(m, n, d_pos, d_d, d_g);
  if (rc) return rc;
  FUEL_CUDA(m, cudaMemcpyAsync(dist, d_d, sizeof(double) * n, cudaMemcpyDeviceToHost, m->stream));
  FUEL_CUDA(m, cudaMemcpyAsync(grad, d_g, sizeof(double) * 3 * n, cudaMemcpyDeviceToHost, m->stream));
  FUEL_CUDA(m, cudaStreamSynchronize(m->stream));
  return 0;
}

int fuelgpu_frontier_search(FuelMap* m, const double upd_min[3], const double upd_max[3],
                            const FuelFrontierParams* params, int32_t* n_clusters, int32_t* n_cells,
                            int32_t* n_filtered) {
  if (!m || !upd_min || !upd_max || !params || !n_clusters || !n_cells || !n_filtered)
    return fuel_fail(m, FUELGPU_EINVAL, "null argument");
  if (params->down_sample < 1) return fuel_fail(m, FUELGPU_EINVAL, "down_sample must be >= 1");
  FUEL_CUDA(m, cudaSetDevice(m->dev));
  cudaStream_t fs = frontier_stream(m);
  tbegin(m, T_FRONTIER, fs);
  int rc = frontier_search_impl(m, upd_min, upd_max, params, n_clusters, n_cells, n_filtered);
  tend(m, T_FRONTIER, fs);
  return rc;
}

int fuelgpu_frontier_search_begin(FuelMap* m, const double upd_min[3], const double upd_max[3],
                                  const FuelFrontierParams* params) {
  if (!m || !upd_min || !upd_max || !params) return fuel_fail(m, FUELGPU_EINVAL, "null argument");
  if (params->down_sample < 1) return fuel_fail(m, FUELGPU_EINVAL, "down_sample must be >= 1");
  FUEL_CUDA(m, cudaSetDevice(m->dev));
  cudaStream_t fs = frontier_stream(m);
  tbegin(m, T_FRONTIER, fs);
  return frontier_search_begin_impl(m, upd_min, upd_max, params);
}

int fuelgpu_frontier_search_end(FuelMap* m, int32_t* n_clusters, int32_t* n_cells, int32_t* n_filtered) {
  if (!m || !n_clusters || !n_cells || !n_filtered) return fuel_fail(m, FUELGPU_EINVAL, "null argument");
  FUEL_CUDA(m, cudaSetDevice(m->dev));
  int rc = frontier_search_end_impl(m, n_clusters, n_cells, n_filtered);
  tend(m, T_FRONTIER, frontier_stream_raw(m));
  return rc;
}

int fuelgpu_frontier_fetch(FuelMap* m, int32_t* cell_offsets, int32_t* cell_addr, int32_t* filt_offsets,
                           double* filtered, double* average, double* box_min, double* box_max) {
  if (!m) return fuel_fail(nullptr, FUELGPU_EINVAL, "null map");
  return frontier_fetch_impl(m, cell_offsets, cell_addr, filt_offsets, filtered, average, box_min, box_max);
}

int fuelgpu_frontier_candidates(FuelMap* m, const double upd_min[3], const double upd_max[3], const FuelFrontierParams* p,
                                int32_t z_lo, int32_t z_hi, int32_t* n_candidates) {
  if (!m || !upd_min || !upd_max || !p || !n_candidates) return fuel_fail(m, FUELGPU_EINVAL, "null argument");
  if (z_lo < 0 || z_hi >= m->g.nz || z_lo > z_hi) return fuel_fail(m, FUELGPU_EINVAL, "bad z range");
  FUEL_CUDA(m, cudaSetDevice(m->dev));
  tbegin(m, T_FRONTIER, frontier_stream(m));  // (the sweep alone: fuelgpu_map_last_timing reports it as the frontier stage)
  const int rc = frontier_candidates_impl(m, upd_min, upd_max, p, z_lo, z_hi, n_candidates);
  tend(m, T_FRONTIER, frontier_stream_raw(m));
  return rc;
}

int fuelgpu_frontier_candidates_fetch(FuelMap* m, int32_t n, int32_t* addr, uint8_t* cls) {
  if (!m || (n > 0 && (!addr || !cls))) return fuel_fail(m, FUELGPU_EINVAL, "null argument");
  FUEL_CUDA(m, cudaSetDevice(m->dev));
  return frontier_candidates_fetch_impl(m, n, addr, cls);
}

int fuelgpu_frontier_search_from_candidates(FuelMap* m, const double upd_min[3], const double upd_max[3],
                                            const FuelFrontierParams* p, int32_t n, const int32_t* addr, const uint8_t* cls,
                                            int32_t* n_clusters, int32_t* n_cells, int32_t* n_filtered) {
  if (!m || !upd_min || !upd_max || !p || !n_clusters || !n_cells || !n_filtered || (n > 0 && (!addr || !cls)))
    return fuel_fail(m, FUELGPU_EINVAL, "null argument");
  FUEL_CUDA(m, cudaSetDevice(m->dev));
  return frontier_search_from_candidates_impl(m, upd_min, upd_max, p, n, addr, cls, n_clusters, n_cells, n_filtered);
}

// one z plane of the occupancy byte <-> a contiguous [nx][ny] device buffer (the halo planes of a z-sharded map)
namespace {
__global__ void occ_plane_kernel(uint8_t* occ, uint8_t* plane, int64_t nxy, int nz, int z, int set) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nxy) return;
  if (set)
    occ[i * nz + z] = plane[i];
  else
    plane[i] = occ[i * nz + z];
}
}  // namespace

int fuelgpu_map_occupancy_plane_dev(FuelMap* m, int32_t z, void* plane_dev, int32_t set) {
  if (!m || !plane_dev) return fuel_fail(m, FUELGPU_EINVAL, "null argument");
  if (z < 0 || z >= m->g.nz) return fuel_fail(m, FUELGPU_EINVAL, "z outside the map");
  FUEL_CUDA(m, cudaSetDevice(m->dev));
  if (set) frontier_order_writer(m);
  const int64_t nxy = (int64_t)m->g.nx * m->g.ny;
  occ_plane_kernel<<<(unsigned)((nxy + 255) / 256), 256, 0, m->stream>>>(m->occ, (uint8_t*)plane_dev, nxy, m->g.nz, z, set);
  FUEL_LAUNCHES(m, 1);
  FUEL_CUDA(m, cudaGetLastError());
  return 0;
}

int fuelgpu_frontier_set_cell_order(FuelMap* m, int32_t order) {
  if (!m) return fuel_fail(nullptr, FUELGPU_EINVAL, "null map");
  return frontier_set_cell_order(m, order);
}

int fuelgpu_frontier_clear_flags(FuelMap* m, int32_t n, const int32_t* addr) {
  if (!m || (n > 0 && !addr)) return fuel_fail(m, FUELGPU_EINVAL, "null argument");
  if (n <= 0) return 0;
  FUEL_CUDA(m, cudaSetDevice(m->dev));
  for (int i = 0; i < n; ++i)
    if (addr[i] < 0 || addr[i] >= m->nvox) return fuel_fail(m, FUELGPU_EINVAL, "address out of range");
  // own small allocation: m->stage belongs to the main-stream ingest path
  int* d_addr = nullptr;
  FUEL_CUDA(m, cudaMalloc(&d_addr, sizeof(int) * (size_t)n));
  cudaStream_t fs = frontier_stream(m);
  FUEL_CUDA(m, cudaMemcpyAsync(d_addr, addr, sizeof(int) * n, cudaMemcpyHostToDevice, fs));
  clear_flags_kernel<<<(n + 255) / 256, 256, 0, fs>>>(m->flag, d_addr, n);
  FUEL_LAUNCHES(m, 1);
  FUEL_CUDA(m, cudaGetLastError());
  FUEL_CUDA(m, cudaStreamSynchronize(fs));
  cudaFree(d_addr);
  return 0;
}

int fuelgpu_frontier_is_changed(FuelMap* m, int32_t mcl, const int32_t* cell_offsets,
                                const int32_t* cell_addr, uint8_t* changed) {
  if (!m || (mcl > 0 && (!cell_offsets || !cell_addr || !changed)))
    return fuel_fail(m, FUELGPU_EINVAL, "null argument");
  FUEL_CUDA(m, cudaSetDevice(m->dev));
  frontier_stream(m);
  return frontier_is_changed_impl(m, mcl, cell_offsets, cell_addr, changed);
}

int fuelgpu_frontier_changed_counts(FuelMap* m, int32_t mcl, const int32_t* cell_offsets, const int32_t* cell_addr,
                                    int32_t* counts) {
  if (!m || (mcl > 0 && (!cell_offsets || !cell_addr || !counts))) return fuel_fail(m, FUELGPU_EINVAL, "null argument");
  FUEL_CUDA(m, cudaSetDevice(m->dev));
  frontier_stream(m);
  return frontier_is_changed_impl(m, mcl, cell_offsets, cell_addr, nullptr, counts);
}

int32_t fuelgpu_viewpoint_candidate_count(const FuelViewParams* p) {
  if (!p || p->candidate_rnum <= 0 || !(p->candidate_dphi > 0.0) || !(p->candidate_rmax >= p->candidate_rmin)) return -1;
  return viewpoint_candidates_host(p, nullptr);
}

int fuelgpu_frontier_sample_viewpoints(FuelMap* m, int32_t n_clusters, const int32_t* filt_offsets, const double* filtered,
                                       const double* average, const FuelViewParams* p, int32_t n_cand, double* cand_pos,
                                       double* cand_yaw, int32_t* cand_visib) {
  if (!m || !p) return fuel_fail(m, FUELGPU_EINVAL, "null argument");
  if (n_clusters < 0) return fuel_fail(m, FUELGPU_EINVAL, "negative cluster count");
  if (n_clusters > 0 && (!filt_offsets || !average || !cand_pos || !cand_yaw || !cand_visib || (filt_offsets[n_clusters] > 0 && !filtered)))
    return fuel_fail(m, FUELGPU_EINVAL, "null argument");
  if (fuelgpu_viewpoint_candidate_count(p) <= 0) return fuel_fail(m, FUELGPU_EINVAL, "degenerate candidate parameters");
  for (int i = 0; i < n_clusters; ++i)
    if (filt_offsets[i + 1] < filt_offsets[i]) return fuel_fail(m, FUELGPU_EINVAL, "filt_offsets not monotone");
  FUEL_CUDA(m, cudaSetDevice(m->dev));
  return sample_viewpoints_impl(m, n_clusters, filt_offsets, filtered, average, p, n_cand, cand_pos, cand_yaw, cand_visib);
}

int fuelgpu_frontier_reset_flags(FuelMap* m) {
  if (!m) return fuel_fail(nullptr, FUELGPU_EINVAL, "null map");
  FUEL_CUDA(m, cudaSetDevice(m->dev));
  FUEL_CUDA(m, cudaMemsetAsync(m->flag, 0, m->nvox, frontier_stream(m)));
  return 0;
}

int fuelgpu_map_launch_count(FuelMap* m, int64_t* count) {
  if (!m || !count) return fuel_fail(m, FUELGPU_EINVAL, "null argument");
  *count = m->launches;
  return 0;
}

int fuelgpu_frontier_download_flags(FuelMap* m, int8_t* out) {
  if (!m || !out) return fuel_fail(m, FUELGPU_EINVAL, "null argument");
  FUEL_CUDA(m, cudaSetDevice(m->dev));
  cudaStream_t fs = frontier_stream(m);
  FUEL_CUDA(m, cudaMemcpyAsync(out, m->flag, m->nvox, cudaMemcpyDeviceToHost, fs));
  FUEL_CUDA(m, cudaStreamSynchronize(fs));
  return 0;
}

int fuelgpu_frontier_upload_flags(FuelMap* m, const int8_t* in) {
  if (!m || !in) return fuel_fail(m, FUELGPU_EINVAL, "null argument");
  FUEL_CUDA(m, cudaSetDevice(m->dev));
  cudaStream_t fs = frontier_stream(m);
  FUEL_CUDA(m, cudaMemcpyAsync(m->flag, in, m->nvox, cudaMemcpyHostToDevice, fs));
  FUEL_CUDA(m, cudaStreamSynchronize(fs));
  return 0;
}

// H2D of the per-trajectory constants.  The guide / waypoint arrays are 3 KB of the 3.3 KB record; when no
// trajectory uses them (the exploration objective) only the leading part (+ n_waypt) is sent: packed into the
// page-locked bounce buffer, one contiguous DMA, then two strided device-side copies into the records.
// `pin` = host bounce area of >= B*(head+4) bytes, `d_pack` = device scratch of the same size.
static cudaError_t upload_traj(FuelMap* m, FuelTrajConst* d_tc, const FuelTrajConst* traj, int B, uint8_t* pin,
                               uint8_t* d_pack, int mask = 0, cudaStream_t st = nullptr) {
  if (!st) st = m->stream;
  bool lean = !(mask & FUELGPU_VIEWCONS);  // the view constraint sits at the end of the record
  for (int b = 0; b < B && lean; ++b) lean = traj[b].n_guide == 0 && traj[b].n_waypt == 0;
  if (!lean) return cudaMemcpyAsync(d_tc, traj, sizeof(FuelTrajConst) * (size_t)B, cudaMemcpyHostToDevice, st);
  const size_t head = offsetof(FuelTrajConst, guide), rec = head + sizeof(int32_t);
  for (int b = 0; b < B; ++b) {
    memcpy(pin + rec * b, &traj[b], head);
    memcpy(pin + rec * b + head, &traj[b].n_waypt, sizeof(int32_t));
  }
  cudaError_t e = cudaMemcpyAsync(d_pack, pin, rec * B, cudaMemcpyHostToDevice, st);
  if (e != cudaSuccess) return e;
  e = cudaMemcpy2DAsync(d_tc, sizeof(FuelTrajConst), d_pack, rec, head, B, cudaMemcpyDeviceToDevice, st);
  if (e != cudaSuccess) return e;
  return cudaMemcpy2DAsync((char*)d_tc + offsetof(FuelTrajConst, n_waypt), sizeof(FuelTrajConst), d_pack + head, rec,
                           sizeof(int32_t), B, cudaMemcpyDeviceToDevice, st);
}

// page-locked (cudaHostRegister / cudaMallocHost) host memory can be DMA'd without the bounce copy
static bool is_pinned_host(const void* p) {
  cudaPointerAttributes a;
  if (cudaPointerGetAttributes(&a, p) != cudaSuccess) {
    cudaGetLastError();
    return false;
  }
  return a.type == cudaMemoryTypeHost;
}

static int check_bspline_args(FuelMap* m, int32_t B, int32_t n_pts, int32_t mask,
                              const FuelOptParams* p) {
  if (!m || !p) return fuel_fail(m, FUELGPU_EINVAL, "null argument");
  if (B < 0) return fuel_fail(m, FUELGPU_EINVAL, "negative batch");
  if (n_pts < 4 || n_pts > FUELGPU_MAX_PTS)
    return fuel_fail(m, FUELGPU_EINVAL, "n_pts must be in 4..64");
  if (p->order < 1 || 2 * p->order >= n_pts) return fuel_fail(m, FUELGPU_EINVAL, "bad spline order");
  return 0;
}

int fuelgpu_bspline_cost_batch_dev(FuelMap* m, int32_t B, int32_t n_pts, int32_t mask,
                                   const FuelOptParams* p, const void* traj_dev, const void* x_dev,
                                   void* f_dev, void* grad_dev) {
  int rc = check_bspline_args(m, B, n_pts, mask, p);
  if (rc) return rc;
  if (B == 0) return 0;
  if (!traj_dev || !x_dev || !f_dev || !grad_dev) return fuel_fail(m, FUELGPU_EINVAL, "null argument");
  FUEL_CUDA(m, cudaSetDevice(m->dev));
  tbegin(m, T_BSPLINE);
  rc = bspline_cost_batch_dev_impl(m, B, n_pts, mask, p, (const FuelTrajConst*)traj_dev,
                                   (const double*)x_dev, (double*)f_dev, (double*)grad_dev);
  tend(m, T_BSPLINE);
  return rc;
}

int fuelgpu_bspline_cost_batch(FuelMap* m, int32_t B, int32_t n_pts, int32_t mask,
                               const FuelOptParams* p, const FuelTrajConst* traj, const double* x,
                               double* f, double* grad) {
  int rc = check_bspline_args(m, B, n_pts, mask, p);
  if (rc) return rc;
  if (B == 0) return 0;
  if (!traj || !x || !f || !grad) return fuel_fail(m, FUELGPU_EINVAL, "null argument");
  if (m->bs_pend_B)  // the pending solve owns the device scratch and the pinned result block
    return fuel_fail(m, FUELGPU_EINVAL, "fuelgpu_bspline_optimize_batch_begin is outstanding: call _end first");
  FUEL_CUDA(m, cudaSetDevice(m->dev));
  const int nvar = (mask & FUELGPU_MINTIME) ? 3 * n_pts + 1 : 3 * n_pts;
  const size_t tcb = sizeof(FuelTrajConst) * (size_t)B;
  const size_t xb = sizeof(double) * (size_t)B * nvar;
  const size_t packb = ((offsetof(FuelTrajConst, guide) + sizeof(int32_t)) * (size_t)B + 63) & ~(size_t)63;
  const size_t fb = sizeof(double) * (size_t)B;
  rc = ensure_bs(m, tcb + 2 * xb + fb + packb + 64);
  if (rc) return rc;
  rc = ensure_bs_pin(m, packb + 2 * xb + fb);
  if (rc) return rc;
  uint8_t* base = (uint8_t*)m->bs_buf;
  FuelTrajConst* d_tc = (FuelTrajConst*)base;
  double* d_x = (double*)(base + tcb);
  double* d_g = d_x + (size_t)B * nvar;
  double* d_f = d_g + (size_t)B * nvar;
  uint8_t* d_pack = (uint8_t*)(d_f + B);
  // host buffers of unknown provenance (pageable or pinned) bounce through the page-locked area
  uint8_t* pin = (uint8_t*)m->bs_pin;
  double* h_x = (double*)(pin + packb);
  double* h_g = h_x + (size_t)B * nvar;
  double* h_f = h_g + (size_t)B * nvar;
  if (mask & FUELGPU_VIEWCONS)
    for (int b = 0; b < B; ++b)
      if (traj[b].view_idx < 0 || traj[b].view_idx >= n_pts)
        return fuel_fail(m, FUELGPU_EINVAL, "VIEWCONS needs FuelTrajConst.view_idx in [0, n_pts) (setViewConstraint)");
  FUEL_CUDA(m, upload_traj(m, d_tc, traj, B, pin, d_pack, mask));
  memcpy(h_x, x, xb);
  FUEL_CUDA(m, cudaMemcpyAsync(d_x, h_x, xb, cudaMemcpyHostToDevice, m->stream));
  tbegin(m, T_BSPLINE);
  rc = bspline_cost_batch_dev_impl(m, B, n_pts, mask, p, d_tc, d_x, d_f, d_g);
  tend(m, T_BSPLINE);
  if (rc) return rc;
  FUEL_CUDA(m, cudaMemcpyAsync(h_g, d_g, xb + fb, cudaMemcpyDeviceToHost, m->stream));  // grad and f are adjacent
  FUEL_CUDA(m, cudaStreamSynchronize(m->stream));
  memcpy(grad, h_g, xb);
  memcpy(f, h_f, fb);
  return 0;
}

int fuelgpu_bspline_optimize_batch_dev(FuelMap* m, int32_t B, int32_t n_pts, int32_t mask,
                                       const FuelOptParams* p, const void* traj_dev,
                                       const FuelSolveParams* solve, void* x_dev, void* f_best_dev,
                                       void* n_eval_dev) {
  int rc = check_bspline_args(m, B, n_pts, mask, p);
  if (rc) return rc;
  if (B == 0) return 0;
  if (!traj_dev || !x_dev || !f_best_dev || !n_eval_dev || !solve)
    return fuel_fail(m, FUELGPU_EINVAL, "null argument");
  if (solve->lbfgs_m < 1 || solve->lbfgs_m > 8 || solve->max_eval < 1)
    return fuel_fail(m, FUELGPU_EINVAL, "bad solver parameters");
  FUEL_CUDA(m, cudaSetDevice(m->dev));
  tbegin(m, T_BSPLINE);
  rc = bspline_optimize_batch_dev_impl(m, B, n_pts, mask, p, (const FuelTrajConst*)traj_dev, solve,
                                       (double*)x_dev, (double*)f_best_dev, (int32_t*)n_eval_dev);
  tend(m, T_BSPLINE);
  return rc;
}

int fuelgpu_bspline_optimize_batch_begin(FuelMap* m, int32_t B, int32_t n_pts, int32_t mask, const FuelOptParams* p,
                                         const FuelTrajConst* traj, const FuelSolveParams* solve, const double* x) {
  int rc = check_bspline_args(m, B, n_pts, mask, p);
  if (rc) return rc;
  if (m->bs_pend_B) return fuel_fail(m, FUELGPU_EINVAL, "an optimize_batch_begin is already outstanding");
  if (B == 0) return 0;
  if (!traj || !x || !solve) return fuel_fail(m, FUELGPU_EINVAL, "null argument");
  if (solve->lbfgs_m < 1 || solve->lbfgs_m > 8 || solve->max_eval < 1)
    return fuel_fail(m, FUELGPU_EINVAL, "bad solver parameters");
  FUEL_CUDA(m, cudaSetDevice(m->dev));
  const int nvar = (mask & FUELGPU_MINTIME) ? 3 * n_pts + 1 : 3 * n_pts;
  const size_t tcb = sizeof(FuelTrajConst) * (size_t)B;
  const size_t xb = sizeof(double) * (size_t)B * nvar;
  const size_t packb = ((offsetof(FuelTrajConst, guide) + sizeof(int32_t)) * (size_t)B + 63) & ~(size_t)63;
  const size_t fb = sizeof(double) * (size_t)B, nb = sizeof(int32_t) * (size_t)B;
  rc = ensure_bs(m, tcb + xb + fb + nb + packb + 64);
  if (rc) return rc;
  rc = ensure_bs_pin(m, packb + xb + fb + nb);
  if (rc) return rc;
  uint8_t* base = (uint8_t*)m->bs_buf;
  FuelTrajConst* d_tc = (FuelTrajConst*)base;
  double* d_x = (double*)(base + tcb);
  double* d_f = d_x + (size_t)B * nvar;
  int32_t* d_n = (int32_t*)(d_f + B);
  uint8_t* d_pack = (uint8_t*)(((uintptr_t)(d_n + B) + 63) & ~(uintptr_t)63);
  // host buffers of unknown provenance (pageable or pinned) bounce through the page-locked area
  uint8_t* pin = (uint8_t*)m->bs_pin;
  double* h_x = (double*)(pin + packb);  // x, f_best, n_eval adjacent on both sides: one DMA back
  if (mask & FUELGPU_VIEWCONS)
    for (int b = 0; b < B; ++b)
      if (traj[b].view_idx < 0 || traj[b].view_idx >= n_pts)
        return fuel_fail(m, FUELGPU_EINVAL, "VIEWCONS needs FuelTrajConst.view_idx in [0, n_pts) (setViewConstraint)");
  // The inputs go out on their own stream -- at once, beside whatever the main stream is still running (the ESDF
  // update, typically) -- and the solver waits for them.  (The scratch is free: every user of it synchronises.)
  FUEL_CUDA(m, upload_traj(m, d_tc, traj, B, pin, d_pack, mask, m->in_stream));
  if (is_pinned_host(x)) {  // caller's buffer is page-locked (fuelgpu_host_register): DMA straight from it
    FUEL_CUDA(m, cudaMemcpyAsync(d_x, x, xb, cudaMemcpyHostToDevice, m->in_stream));
  } else {
    memcpy(h_x, x, xb);
    FUEL_CUDA(m, cudaMemcpyAsync(d_x, h_x, xb, cudaMemcpyHostToDevice, m->in_stream));
  }
  FUEL_CUDA(m, cudaEventRecord(m->in_ev, m->in_stream));
  FUEL_CUDA(m, cudaStreamWaitEvent(m->stream, m->in_ev, 0));
  tbegin(m, T_BSPLINE);
  rc = bspline_optimize_batch_dev_impl(m, B, n_pts, mask, p, d_tc, solve, d_x, d_f, d_n);
  tend(m, T_BSPLINE);
  if (rc) return rc;
  FUEL_CUDA(m, cudaMemcpyAsync(h_x, d_x, xb + fb + nb, cudaMemcpyDeviceToHost, m->stream));
  m->bs_pend_B = B;
  m->bs_pend_nvar = nvar;
  m->bs_pend_off = packb;
  return 0;
}

int fuelgpu_bspline_optimize_batch_end(FuelMap* m, double* x, double* f_best, int32_t* n_eval) {
  if (!m) return fuel_fail(nullptr, FUELGPU_EINVAL, "null map");
  if (!m->bs_pend_B) return 0;
  if (!x || !f_best || !n_eval) return fuel_fail(m, FUELGPU_EINVAL, "null argument");
  const int B = m->bs_pend_B;
  const size_t xb = sizeof(double) * (size_t)B * m->bs_pend_nvar, fb = sizeof(double) * (size_t)B, nb = sizeof(int32_t) * (size_t)B;
  m->bs_pend_B = 0;
  FUEL_CUDA(m, cudaSetDevice(m->dev));
  FUEL_CUDA(m, cudaStreamSynchronize(m->stream));
  const uint8_t* h = (const uint8_t*)m->bs_pin + m->bs_pend_off;
  memcpy(x, h, xb);
  memcpy(f_best, h + xb, fb);
  memcpy(n_eval, h + xb + fb, nb);
  return 0;
}

int fuelgpu_bspline_optimize_batch(FuelMap* m, int32_t B, int32_t n_pts, int32_t mask,
                                   const FuelOptParams* p, const FuelTrajConst* traj,
                                   const FuelSolveParams* solve, double* x, double* f_best,
                                   int32_t* n_eval) {
  if (B > 0 && (!x || !f_best || !n_eval)) return fuel_fail(m, FUELGPU_EINVAL, "null argument");
  int rc = fuelgpu_bspline_optimize_batch_begin(m, B, n_pts, mask, p, traj, solve, x);
  if (rc) return rc;
  return fuelgpu_bspline_optimize_batch_end(m, x, f_best, n_eval);
}



}  // extern "C"
