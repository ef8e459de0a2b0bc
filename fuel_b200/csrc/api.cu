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

size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }

// The host arrays of one host-facing batch call, staged in tc_buf in 256-byte aligned pieces.  in() and out() name
// a device pointer and the host array it stands for; a null host array gives a null device pointer.  upload() lays
// the arrays out and enqueues the copies of the inputs on m->stream; download() enqueues the copies of the outputs
// and waits for them.
class HostStaging {
 public:
  explicit HostStaging(FuelMap* m) : m_(m) {}
  template <typename T>
  HostStaging& in(T** dev, const T* host, size_t n) {
    arrays_.push_back({ dev, nullptr, host, nullptr, sizeof(T) * n });
    return *this;
  }
  template <typename T>
  HostStaging& out(T** dev, T* host, size_t n) {
    arrays_.push_back({ dev, nullptr, host, host, sizeof(T) * n });
    return *this;
  }
  int upload() {
    FuelMap* m = m_;
    size_t total = 0;
    for (const Array& a : arrays_)
      if (a.host) total += align256(a.bytes);
    int rc = m->tc_buf.ensure(m, total);
    if (rc) return rc;
    uint8_t* q = m->tc_buf.p;
    for (Array& a : arrays_) {
      if (a.host) {
        a.dev = q;
        q += align256(a.bytes);
      }
      memcpy(a.slot, &a.dev, sizeof(a.dev));  // *(T**)slot = dev, without type punning
      if (a.host && !a.out && a.bytes)
        FUEL_CUDA(m, cudaMemcpyAsync(a.dev, a.host, a.bytes, cudaMemcpyHostToDevice, m->stream));
    }
    return 0;
  }
  int download() {
    FuelMap* m = m_;
    for (const Array& a : arrays_)
      if (a.out && a.bytes) FUEL_CUDA(m, cudaMemcpyAsync(a.out, a.dev, a.bytes, cudaMemcpyDeviceToHost, m->stream));
    FUEL_CUDA(m, cudaStreamSynchronize(m->stream));
    return 0;
  }

 private:
  struct Array {
    void* slot;       // the caller's T* that receives dev
    void* dev;        // place in tc_buf, null for a null host array
    const void* host;
    void* out;        // the host array again for an output, null for an input
    size_t bytes;
  };
  FuelMap* m_;
  std::vector<Array> arrays_;
};

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
  CR(cudaEventCreateWithFlags(&m->mirror_ev, cudaEventDisableTiming));
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
  if (m->esdf_aux) {
    cudaStreamSynchronize(m->esdf_aux);
    cudaStreamDestroy(m->esdf_aux);
  }
  for (int i = 0; i < 2; ++i)
    if (m->esdf_ev[i]) cudaEventDestroy(m->esdf_ev[i]);
  void* ptrs[] = { m->occ, m->dist, m->dist_neg, m->flag, m->esdf_rec, m->esdf_p[0], m->esdf_p[1] };
  for (void* p : ptrs)
    if (p) cudaFree(p);
  m->stage.release();
  m->bs_buf.release();
  m->bs_pin.release();
  m->bs_grad.release();
  m->fr_scr.release();
  m->tc_buf.release();
  m->as_buf.release();
  m->ks_buf.release();
  m->vc_buf.release();
  m->lt_buf.release();
  m->gt_buf.release();
  for (int t = 0; t < T_COUNT; ++t) {
    if (m->ev0[t]) cudaEventDestroy(m->ev0[t]);
    if (m->ev1[t]) cudaEventDestroy(m->ev1[t]);
  }
  if (m->copy_stream) {
    cudaStreamSynchronize(m->copy_stream);
    cudaStreamDestroy(m->copy_stream);
  }
  if (m->copy_ev) cudaEventDestroy(m->copy_ev);
  if (m->mirror_ev) cudaEventDestroy(m->mirror_ev);
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
  rc = m->stage.ensure(m, inf_bytes + (size_t)cnt * (logodds ? 8 : 1));
  if (rc) return rc;
  frontier_order_writer(m);
  tbegin(m, T_UPLOAD);
  int8_t* d_inf = (int8_t*)m->stage.p;
  FUEL_CUDA(m, cudaMemcpyAsync(d_inf, inflate + off, cnt, cudaMemcpyHostToDevice, m->stream));
  const unsigned nb = (unsigned)((cnt + 255) / 256);
  if (logodds) {
    double* d_lo = (double*)(m->stage.p + inf_bytes);
    FUEL_CUDA(m, cudaMemcpyAsync(d_lo, logodds + off, cnt * 8, cudaMemcpyHostToDevice, m->stream));
    ingest_logodds_kernel<<<nb, 256, 0, m->stream>>>(d_inf, d_lo, m->occ + off, cnt, clamp_min_log - 1e-3,
                                                     min_occupancy_log);
  } else {
    uint8_t* d_tri = m->stage.p + inf_bytes;
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
  int rc = m->stage.ensure(m, (size_t)m->nvox * 2);
  if (rc) return rc;
  int8_t* d_inf = (int8_t*)m->stage.p;
  uint8_t* d_tri = m->stage.p + m->nvox;
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
  esdf_order_writer(m);
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
    rc = m->stage.ensure(m, (size_t)cnt * 8);
    if (rc) return rc;
    f32_to_f64_kernel<<<(unsigned)((cnt + 255) / 256), 256, 0, m->stream>>>(
        m->dist + off, (double*)m->stage.p, cnt, m->g.res * sqrt(1.7976931348623157e308));
    FUEL_LAUNCHES(m, 1);
    FUEL_CUDA(m, cudaGetLastError());
    FUEL_CUDA(m, cudaMemcpyAsync(out_f64 + off, m->stage.p, cnt * 8, cudaMemcpyDeviceToHost, m->stream));
  }
  tend(m, T_DOWNLOAD);
  FUEL_CUDA(m, cudaStreamSynchronize(m->stream));
  return 0;
}

int fuelgpu_esdf_set_from_slabs_dev(FuelMap* m, const void* slabs_dev, int32_t n_slabs) {
  if (!m || !slabs_dev) return fuel_fail(m, FUELGPU_EINVAL, "null argument");
  if (n_slabs < 1 || m->g.nz % n_slabs) return fuel_fail(m, FUELGPU_EINVAL, "nz is not a multiple of the slab count");
  FUEL_CUDA(m, cudaSetDevice(m->dev));
  esdf_order_writer(m);
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
  FUEL_CUDA(m, cudaEventRecord(m->mirror_ev, m->copy_stream));
  m->mirror_pending = true;
  return 0;
}

int fuelgpu_esdf_sample(FuelMap* m, int64_t n, const double* pos, double* dist, double* grad) {
  if (!m || (n > 0 && (!pos || !dist || !grad))) return fuel_fail(m, FUELGPU_EINVAL, "null argument");
  if (n <= 0) return 0;
  FUEL_CUDA(m, cudaSetDevice(m->dev));
  double *d_pos, *d_d, *d_g;
  HostStaging st(m);
  st.in(&d_pos, pos, 3 * (size_t)n).out(&d_d, dist, (size_t)n).out(&d_g, grad, 3 * (size_t)n);
  int rc = st.upload();
  if (rc) return rc;
  rc = esdf_sample_impl(m, n, d_pos, d_d, d_g);
  if (rc) return rc;
  return st.download();
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
#ifdef FUEL_PROF
  const double t0 = prof_now_us();
#endif
  int rc = frontier_search_end_impl(m, n_clusters, n_cells, n_filtered);
#ifdef FUEL_PROF
  const double t1 = prof_now_us();
  m->end_prof_us[1] = t1 - t0 - m->end_prof_us[0];  // everything of _end but the stream wait
#endif
  tend(m, T_FRONTIER, frontier_stream_raw(m));
#ifdef FUEL_PROF
  m->end_prof_us[2] = prof_now_us() - t1;
#endif
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
  // the frontier stream's scratch: m->stage belongs to the main-stream ingest path
  int rc = m->fr_scr.ensure(m, sizeof(int) * (size_t)n);
  if (rc) return rc;
  int* d_addr = (int*)m->fr_scr.p;
  cudaStream_t fs = frontier_stream(m);
  FUEL_CUDA(m, cudaMemcpyAsync(d_addr, addr, sizeof(int) * n, cudaMemcpyHostToDevice, fs));
  clear_flags_kernel<<<(n + 255) / 256, 256, 0, fs>>>(m->flag, d_addr, n);
  FUEL_LAUNCHES(m, 1);
  FUEL_CUDA(m, cudaGetLastError());
  FUEL_CUDA(m, cudaStreamSynchronize(fs));
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
  rc = m->bs_buf.ensure(m, tcb + 2 * xb + fb + packb + 64);
  if (rc) return rc;
  rc = m->bs_pin.ensure(m, packb + 2 * xb + fb);
  if (rc) return rc;
  uint8_t* base = m->bs_buf.p;
  FuelTrajConst* d_tc = (FuelTrajConst*)base;
  double* d_x = (double*)(base + tcb);
  double* d_g = d_x + (size_t)B * nvar;
  double* d_f = d_g + (size_t)B * nvar;
  uint8_t* d_pack = (uint8_t*)(d_f + B);
  // host buffers of unknown provenance (pageable or pinned) bounce through the page-locked area
  uint8_t* pin = m->bs_pin.p;
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
  rc = m->bs_buf.ensure(m, tcb + xb + fb + nb + packb + 64);
  if (rc) return rc;
  rc = m->bs_pin.ensure(m, packb + xb + fb + nb);
  if (rc) return rc;
  uint8_t* base = m->bs_buf.p;
  FuelTrajConst* d_tc = (FuelTrajConst*)base;
  double* d_x = (double*)(base + tcb);
  double* d_f = d_x + (size_t)B * nvar;
  int32_t* d_n = (int32_t*)(d_f + B);
  uint8_t* d_pack = (uint8_t*)(((uintptr_t)(d_n + B) + 63) & ~(uintptr_t)63);
  // host buffers of unknown provenance (pageable or pinned) bounce through the page-locked area
  uint8_t* pin = m->bs_pin.p;
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
  const uint8_t* h = m->bs_pin.p + m->bs_pend_off;
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

static int check_traj_args(FuelMap* m, int32_t B, int32_t n_pts, int32_t nvar, bool has_x, bool has_dt) {
  if (!m) return fuel_fail(nullptr, FUELGPU_EINVAL, "null map");
  if (B < 0) return fuel_fail(m, FUELGPU_EINVAL, "negative batch");
  if (n_pts < 4 || n_pts > FUELGPU_MAX_PTS) return fuel_fail(m, FUELGPU_EINVAL, "n_pts must be in 4..64");
  if (nvar == 3 * n_pts + 1) {
    if (has_dt) return fuel_fail(m, FUELGPU_EINVAL, "nvar == 3*n_pts + 1 carries dt in x: pass dt = NULL");
  } else if (nvar == 3 * n_pts) {
    if (B > 0 && !has_dt) return fuel_fail(m, FUELGPU_EINVAL, "nvar == 3*n_pts needs dt[B]");
  } else {
    return fuel_fail(m, FUELGPU_EINVAL, "nvar must be 3*n_pts or 3*n_pts + 1");
  }
  if (B > 0 && !has_x) return fuel_fail(m, FUELGPU_EINVAL, "null argument");
  return 0;
}

int fuelgpu_bspline_check_batch_dev(FuelMap* m, int32_t B, int32_t n_pts, int32_t nvar, const void* x_dev,
                                    const void* dt_dev, const FuelTrajCheckParams* p, void* report_dev, void* best_dev) {
  int rc = check_traj_args(m, B, n_pts, nvar, x_dev != nullptr, dt_dev != nullptr);
  if (rc) return rc;
  if (!p || !best_dev || (B > 0 && !report_dev)) return fuel_fail(m, FUELGPU_EINVAL, "null argument");
  FUEL_CUDA(m, cudaSetDevice(m->dev));
  tbegin(m, T_CHECK);
  rc = traj_check_impl(m, B, n_pts, nvar, (const double*)x_dev, (const double*)dt_dev, p, (FuelTrajReport*)report_dev,
                       (int32_t*)best_dev);
  tend(m, T_CHECK);
  return rc;
}

int fuelgpu_bspline_check_batch(FuelMap* m, int32_t B, int32_t n_pts, int32_t nvar, const double* x, const double* dt,
                                const FuelTrajCheckParams* p, FuelTrajReport* report, int32_t best[2]) {
  int rc = check_traj_args(m, B, n_pts, nvar, x != nullptr, dt != nullptr);
  if (rc) return rc;
  if (!p || !best || (B > 0 && !report)) return fuel_fail(m, FUELGPU_EINVAL, "null argument");
  FUEL_CUDA(m, cudaSetDevice(m->dev));
  double *d_x, *d_dt;
  FuelTrajReport* d_rep;
  int32_t* d_best;
  HostStaging st(m);
  st.in(&d_x, x, (size_t)B * nvar).in(&d_dt, dt, (size_t)B).out(&d_rep, report, (size_t)B).out(&d_best, best, 2);
  rc = st.upload();
  if (rc) return rc;
  tbegin(m, T_CHECK);
  rc = traj_check_impl(m, B, n_pts, nvar, d_x, d_dt, p, d_rep, d_best);
  tend(m, T_CHECK);
  if (rc) return rc;
  return st.download();
}

int fuelgpu_bspline_evaluate_batch(FuelMap* m, int32_t B, int32_t n_pts, int32_t nvar, const double* x, const double* dt,
                                   int32_t n_t, const double* t, int32_t deriv, double* out) {
  int rc = check_traj_args(m, B, n_pts, nvar, x != nullptr, dt != nullptr);
  if (rc) return rc;
  if (n_t < 0 || deriv < 0 || deriv > 2) return fuel_fail(m, FUELGPU_EINVAL, "n_t must be >= 0 and deriv 0, 1 or 2");
  if (B == 0 || n_t == 0) return 0;
  if (!t || !out) return fuel_fail(m, FUELGPU_EINVAL, "null argument");
  FUEL_CUDA(m, cudaSetDevice(m->dev));
  const size_t nt = (size_t)B * n_t;
  double *d_x, *d_dt, *d_t, *d_out;
  HostStaging st(m);
  st.in(&d_x, x, (size_t)B * nvar).in(&d_dt, dt, (size_t)B).in(&d_t, t, nt).out(&d_out, out, 3 * nt);
  rc = st.upload();
  if (rc) return rc;
  rc = traj_evaluate_impl(m, B, n_pts, nvar, d_x, d_dt, n_t, d_t, deriv, d_out);
  if (rc) return rc;
  return st.download();
}

static int check_param_args(FuelMap* m, int32_t B, int32_t n_pts, int32_t nvar, const void* points, const void* derivs,
                            const void* dt, const void* x, const void* traj) {
  if (!m) return fuel_fail(nullptr, FUELGPU_EINVAL, "null map");
  if (B < 0) return fuel_fail(m, FUELGPU_EINVAL, "negative batch");
  if (n_pts < 4 || n_pts > FUELGPU_MAX_PTS) return fuel_fail(m, FUELGPU_EINVAL, "n_pts must be in 4..64");
  if (nvar != 3 * n_pts && nvar != 3 * n_pts + 1) return fuel_fail(m, FUELGPU_EINVAL, "nvar must be 3*n_pts or 3*n_pts + 1");
  if (B > 0 && (!points || !derivs || !dt || !x || !traj)) return fuel_fail(m, FUELGPU_EINVAL, "null argument");
  return 0;
}

int fuelgpu_bspline_parameterize_batch_dev(FuelMap* m, int32_t B, int32_t n_pts, int32_t nvar, const void* points_dev,
                                           const void* derivs_dev, const void* dt_dev, const void* time_lb_dev, void* x_dev,
                                           void* traj_dev) {
  int rc = check_param_args(m, B, n_pts, nvar, points_dev, derivs_dev, dt_dev, x_dev, traj_dev);
  if (rc) return rc;
  FUEL_CUDA(m, cudaSetDevice(m->dev));
  tbegin(m, T_PARAM);
  rc = traj_param_impl(m, B, n_pts, nvar, (const double*)points_dev, (const double*)derivs_dev, (const double*)dt_dev,
                       (const double*)time_lb_dev, (double*)x_dev, (FuelTrajConst*)traj_dev);
  tend(m, T_PARAM);
  return rc;
}

int fuelgpu_bspline_parameterize_batch(FuelMap* m, int32_t B, int32_t n_pts, int32_t nvar, const double* points,
                                       const double* derivs, const double* dt, const double* time_lb, double* x,
                                       FuelTrajConst* traj) {
  int rc = check_param_args(m, B, n_pts, nvar, points, derivs, dt, x, traj);
  if (rc) return rc;
  for (int32_t b = 0; b < B; ++b)  // parameterizeToBspline prints and returns on ts <= 0 (:181-184)
    if (!(dt[b] > 0.0 && dt[b] <= 1.7976931348623157e308))
      return fuel_fail(m, FUELGPU_EINVAL, "dt[%s%lld] must be finite and positive", "", (long long)b);
  if (B == 0) return 0;
  FUEL_CUDA(m, cudaSetDevice(m->dev));
  const size_t nb = (size_t)B, K = (size_t)n_pts - 2;
  double *d_pts, *d_der, *d_dt, *d_tlb, *d_x;
  FuelTrajConst* d_tc;
  HostStaging st(m);
  st.in(&d_pts, points, nb * K * 3).in(&d_der, derivs, nb * 12).in(&d_dt, dt, nb).in(&d_tlb, time_lb, nb);
  st.out(&d_x, x, nb * nvar).out(&d_tc, traj, nb);
  rc = st.upload();
  if (rc) return rc;
  tbegin(m, T_PARAM);
  rc = traj_param_impl(m, B, n_pts, nvar, d_pts, d_der, d_dt, d_tlb, d_x, d_tc);
  tend(m, T_PARAM);
  if (rc) return rc;
  return st.download();
}


static bool finite_pos(double v) { return v > 0.0 && v <= 1.7976931348623157e308; }

static int check_poly_args(FuelMap* m, int32_t B, int32_t w_max, const void* n_wp, const void* waypts,
                           const void* start_vel, const void* start_acc, const FuelPolyParams* p, const void* info,
                           const void* points, const void* derivs) {
  if (!m) return fuel_fail(nullptr, FUELGPU_EINVAL, "null map");
  if (B < 0) return fuel_fail(m, FUELGPU_EINVAL, "negative batch");
  if (w_max < 3) return fuel_fail(m, FUELGPU_EINVAL, "w_max must be at least 3");
  if (!p) return fuel_fail(m, FUELGPU_EINVAL, "null params");
  if (!finite_pos(p->max_vel)) return fuel_fail(m, FUELGPU_EINVAL, "max_vel must be finite and positive");
  if (!finite_pos(p->ctrl_pt_dist)) return fuel_fail(m, FUELGPU_EINVAL, "ctrl_pt_dist must be finite and positive");
  if (p->min_seg_num < 1) return fuel_fail(m, FUELGPU_EINVAL, "min_seg_num must be at least 1");
  if (B > 0 && (!n_wp || !waypts || !start_vel || !start_acc || !info || !points || !derivs))
    return fuel_fail(m, FUELGPU_EINVAL, "null argument");
  return 0;
}

int fuelgpu_poly_waypoints_batch_dev(FuelMap* m, int32_t B, int32_t w_max, const void* n_wp_dev, const void* waypts_dev,
                                     const void* start_vel_dev, const void* start_acc_dev, const void* end_vel_dev,
                                     const void* end_acc_dev, const void* times_dev, const FuelPolyParams* p,
                                     void* info_dev, void* coeffs_dev, void* points_dev, void* derivs_dev) {
  int rc = check_poly_args(m, B, w_max, n_wp_dev, waypts_dev, start_vel_dev, start_acc_dev, p, info_dev, points_dev,
                           derivs_dev);
  if (rc) return rc;
  FUEL_CUDA(m, cudaSetDevice(m->dev));
  tbegin(m, T_POLY);
  rc = poly_waypoints_impl(m, B, w_max, (const int32_t*)n_wp_dev, (const double*)waypts_dev,
                           (const double*)start_vel_dev, (const double*)start_acc_dev, (const double*)end_vel_dev,
                           (const double*)end_acc_dev, (const double*)times_dev, p, (FuelPolyInfo*)info_dev,
                           (double*)coeffs_dev, (double*)points_dev, (double*)derivs_dev);
  tend(m, T_POLY);
  return rc;
}

int fuelgpu_poly_waypoints_batch(FuelMap* m, int32_t B, int32_t w_max, const int32_t* n_wp, const double* waypts,
                                 const double* start_vel, const double* start_acc, const double* end_vel,
                                 const double* end_acc, const double* times, const FuelPolyParams* p,
                                 FuelPolyInfo* info, double* coeffs, double* points, double* derivs) {
  int rc = check_poly_args(m, B, w_max, n_wp, waypts, start_vel, start_acc, p, info, points, derivs);
  if (rc) return rc;
  for (int32_t b = 0; b < B; ++b) {
    const int32_t W = n_wp[b];
    if (W < 3 || W > FUELGPU_MAX_WAYPTS)  // W = 2: waypointsTraj writes Ct out of bounds (polynomial_traj.cpp:74-75)
      return fuel_fail(m, FUELGPU_EINVAL, "n_wp[%s%lld] must be in 3..32", "", (long long)b);
    if (W > w_max) return fuel_fail(m, FUELGPU_EINVAL, "n_wp[%s%lld] exceeds w_max", "", (long long)b);
    for (int32_t i = 0; i + 1 < W; ++i) {  // the segment times, given or as planner_manager.cpp:276-278 makes them
      double t;
      if (times) {
        t = times[(size_t)b * (w_max - 1) + i];
      } else {
        const double* q = waypts + ((size_t)b * w_max + i) * 3;
        const double dx = q[3] - q[0], dy = q[4] - q[1], dz = q[5] - q[2];
        t = sqrt((dx * dx + dy * dy) + dz * dz) / (p->max_vel * 0.5);
      }
      if (!finite_pos(t))
        return fuel_fail(m, FUELGPU_EINVAL, "tour %s%lld has a segment time that is not finite and positive", "",
                         (long long)b);
    }
  }
  if (B == 0) return 0;
  FUEL_CUDA(m, cudaSetDevice(m->dev));
  const size_t nb = (size_t)B, S1 = (size_t)w_max - 1, K = FUELGPU_MAX_PTS - 2;
  int32_t* d_n;
  double *d_wp, *d_sv, *d_sa, *d_ev, *d_ea, *d_t, *d_c, *d_p, *d_d;
  FuelPolyInfo* d_info;
  HostStaging st(m);
  st.in(&d_n, n_wp, nb).in(&d_wp, waypts, nb * w_max * 3).in(&d_sv, start_vel, nb * 3).in(&d_sa, start_acc, nb * 3);
  st.in(&d_ev, end_vel, nb * 3).in(&d_ea, end_acc, nb * 3).in(&d_t, times, nb * S1);
  st.out(&d_info, info, nb).out(&d_c, coeffs, nb * S1 * 18).out(&d_p, points, nb * K * 3).out(&d_d, derivs, nb * 12);
  rc = st.upload();
  if (rc) return rc;
  tbegin(m, T_POLY);
  rc = poly_waypoints_impl(m, B, w_max, d_n, d_wp, d_sv, d_sa, d_ev, d_ea, d_t, p, d_info, d_c, d_p, d_d);
  tend(m, T_POLY);
  if (rc) return rc;
  return st.download();
}

static int check_yaw_args(FuelMap* m, int32_t B, int32_t n_pts, int32_t nvar, const void* x, const void* dt,
                          const void* start_yaw, const void* end_yaw, const FuelOptParams* p, const FuelYawParams* yp,
                          const void* yaw, const void* info) {
  int rc = check_traj_args(m, B, n_pts, nvar, x != nullptr, dt != nullptr);
  if (rc) return rc;
  if (!p || !yp) return fuel_fail(m, FUELGPU_EINVAL, "null params");
  if (!finite_pos(p->ld_smooth) || !finite_pos(p->ld_start))
    return fuel_fail(m, FUELGPU_EINVAL, "ld_smooth and ld_start must be finite and positive");
  if (!(yp->relax_time >= 0.0 && yp->relax_time <= 1.7976931348623157e308))
    return fuel_fail(m, FUELGPU_EINVAL, "relax_time must be finite and >= 0");
  if (B > 0 && (!start_yaw || !end_yaw || !yaw || !info)) return fuel_fail(m, FUELGPU_EINVAL, "null argument");
  return 0;
}

int fuelgpu_yaw_explore_batch_dev(FuelMap* m, int32_t B, int32_t n_pts, int32_t nvar, const void* x_dev,
                                  const void* dt_dev, const void* start_yaw_dev, const void* end_yaw_dev,
                                  const FuelOptParams* p, const FuelYawParams* yp, void* yaw_dev, void* info_dev,
                                  void* waypt_dev) {
  int rc = check_yaw_args(m, B, n_pts, nvar, x_dev, dt_dev, start_yaw_dev, end_yaw_dev, p, yp, yaw_dev, info_dev);
  if (rc) return rc;
  FUEL_CUDA(m, cudaSetDevice(m->dev));
  return yaw_explore_impl(m, B, n_pts, nvar, (const double*)x_dev, (const double*)dt_dev, (const double*)start_yaw_dev,
                          (const double*)end_yaw_dev, p, yp, (double*)yaw_dev, (FuelYawInfo*)info_dev,
                          (double*)waypt_dev);
}

int fuelgpu_yaw_explore_batch(FuelMap* m, int32_t B, int32_t n_pts, int32_t nvar, const double* x, const double* dt,
                              const double* start_yaw, const double* end_yaw, const FuelOptParams* p,
                              const FuelYawParams* yp, double* yaw, FuelYawInfo* info, double* waypt) {
  int rc = check_yaw_args(m, B, n_pts, nvar, x, dt, start_yaw, end_yaw, p, yp, yaw, info);
  if (rc) return rc;
  for (int32_t b = 0; b < B; ++b) {
    const double d = dt ? dt[b] : x[(size_t)b * nvar + 3 * n_pts];
    if (!finite_pos(d)) return fuel_fail(m, FUELGPU_EINVAL, "dt of trajectory %s%lld must be finite and positive", "",
                                         (long long)b);
    const double* s = start_yaw + 3 * (size_t)b;
    // the reference's wrapping loops (planner_manager.cpp:782-783) never end on a non-finite start yaw
    if (!(fabs(s[0]) <= FUELGPU_YAW_MAX_START) || !isfinite(s[1]) || !isfinite(s[2]) || !isfinite(end_yaw[b]))
      return fuel_fail(m, FUELGPU_EINVAL, "trajectory %s%lld: start yaw must be finite with |yaw| <= 1000, end yaw finite",
                       "", (long long)b);
  }
  if (B == 0) return 0;
  FUEL_CUDA(m, cudaSetDevice(m->dev));
  const size_t nb = (size_t)B;
  double *d_x, *d_dt, *d_sy, *d_ey, *d_yaw, *d_wp;
  FuelYawInfo* d_info;
  HostStaging st(m);
  st.in(&d_x, x, nb * nvar).in(&d_dt, dt, nb).in(&d_sy, start_yaw, nb * 3).in(&d_ey, end_yaw, nb);
  st.out(&d_yaw, yaw, nb * FUELGPU_YAW_PTS).out(&d_info, info, nb).out(&d_wp, waypt, nb * FUELGPU_YAW_MAX_WAYPT);
  rc = st.upload();
  if (rc) return rc;
  rc = yaw_explore_impl(m, B, n_pts, nvar, d_x, d_dt, d_sy, d_ey, p, yp, d_yaw, d_info, d_wp);
  if (rc) return rc;
  return st.download();
}

static int check_plan_yaw_args(FuelMap* m, int32_t B, int32_t n_pts, int32_t nvar, const void* x, const void* dt,
                               const void* start_yaw, const FuelOptParams* p, const void* yaw, const void* info) {
  int rc = check_traj_args(m, B, n_pts, nvar, x != nullptr, dt != nullptr);
  if (rc) return rc;
  if (!p) return fuel_fail(m, FUELGPU_EINVAL, "null params");
  if (!finite_pos(p->ld_smooth) || !finite_pos(p->ld_start))
    return fuel_fail(m, FUELGPU_EINVAL, "ld_smooth and ld_start must be finite and positive");
  if (B > 0 && (!start_yaw || !yaw || !info)) return fuel_fail(m, FUELGPU_EINVAL, "null argument");
  return 0;
}

int fuelgpu_plan_yaw_batch_dev(FuelMap* m, int32_t B, int32_t n_pts, int32_t nvar, const void* x_dev,
                               const void* dt_dev, const void* start_yaw_dev, const FuelOptParams* p, void* yaw_dev,
                               void* info_dev, void* waypt_dev) {
  int rc = check_plan_yaw_args(m, B, n_pts, nvar, x_dev, dt_dev, start_yaw_dev, p, yaw_dev, info_dev);
  if (rc) return rc;
  FUEL_CUDA(m, cudaSetDevice(m->dev));
  return plan_yaw_impl(m, B, n_pts, nvar, (const double*)x_dev, (const double*)dt_dev, (const double*)start_yaw_dev, p,
                       (double*)yaw_dev, (FuelPlanYawInfo*)info_dev, (double*)waypt_dev);
}

int fuelgpu_plan_yaw_batch(FuelMap* m, int32_t B, int32_t n_pts, int32_t nvar, const double* x, const double* dt,
                           const double* start_yaw, const FuelOptParams* p, double* yaw, FuelPlanYawInfo* info,
                           double* waypt) {
  int rc = check_plan_yaw_args(m, B, n_pts, nvar, x, dt, start_yaw, p, yaw, info);
  if (rc) return rc;
  for (int32_t b = 0; b < B; ++b) {
    const double d = dt ? dt[b] : x[(size_t)b * nvar + 3 * n_pts];
    if (!finite_pos(d)) return fuel_fail(m, FUELGPU_EINVAL, "dt of trajectory %s%lld must be finite and positive", "",
                                         (long long)b);
    const double* s = start_yaw + 3 * (size_t)b;
    // bounds calcNextYaw's wrapping loops (planner_manager.cpp:869-870), which never end on a non-finite yaw
    if (!(fabs(s[0]) <= FUELGPU_YAW_MAX_START) || !isfinite(s[1]) || !isfinite(s[2]))
      return fuel_fail(m, FUELGPU_EINVAL, "trajectory %s%lld: start yaw must be finite with |yaw| <= 1000", "",
                       (long long)b);
  }
  if (B == 0) return 0;
  FUEL_CUDA(m, cudaSetDevice(m->dev));
  const size_t nb = (size_t)B;
  double *d_x, *d_dt, *d_sy, *d_yaw, *d_wp;
  FuelPlanYawInfo* d_info;
  HostStaging st(m);
  st.in(&d_x, x, nb * nvar).in(&d_dt, dt, nb).in(&d_sy, start_yaw, nb * 3);
  st.out(&d_yaw, yaw, nb * FUELGPU_PLANYAW_MAX_PTS).out(&d_info, info, nb).out(&d_wp, waypt, nb * FUELGPU_PLANYAW_MAX_SEG);
  rc = st.upload();
  if (rc) return rc;
  rc = plan_yaw_impl(m, B, n_pts, nvar, d_x, d_dt, d_sy, p, d_yaw, d_info, d_wp);
  if (rc) return rc;
  return st.download();
}

static int check_astar_params(FuelMap* m, const FuelAstarParams* p) {
  if (!p) return fuel_fail(m, FUELGPU_EINVAL, "null params");
  // above 1e-3 the reference's neighbour loop (astar2.cpp:90-94) makes exactly the 26 steps
  if (!(p->resolution > 1e-3 && p->resolution <= 1.7976931348623157e308))
    return fuel_fail(m, FUELGPU_EINVAL, "resolution must be finite and > 1e-3");
  if (!isfinite(p->lambda_heu)) return fuel_fail(m, FUELGPU_EINVAL, "lambda_heu must be finite");
  if (p->allocate_num < 2 || p->max_iter < 1)
    return fuel_fail(m, FUELGPU_EINVAL, "allocate_num must be at least 2 and max_iter at least 1");
  if (p->allocate_num > (1 << 28)) return fuel_fail(m, FUELGPU_EINVAL, "allocate_num above 2^28");
  return 0;
}

static int check_astar_args(FuelMap* m, int32_t B, const void* start, const void* goal, const FuelAstarParams* p,
                            const void* info, int32_t path_max, const void* path, int32_t w_max, const void* n_wp,
                            const void* waypts) {
  if (!m) return fuel_fail(nullptr, FUELGPU_EINVAL, "null map");
  if (B < 0) return fuel_fail(m, FUELGPU_EINVAL, "negative batch");
  const int rc = check_astar_params(m, p);
  if (rc) return rc;
  if (w_max < 3) return fuel_fail(m, FUELGPU_EINVAL, "w_max must be at least 3");
  if (path && path_max < 1) return fuel_fail(m, FUELGPU_EINVAL, "path_max must be at least 1 with a path buffer");
  if (B > 0 && (!start || !goal || !info || !n_wp || !waypts)) return fuel_fail(m, FUELGPU_EINVAL, "null argument");
  return 0;
}

int fuelgpu_astar_batch_dev(FuelMap* m, int32_t B, const void* start_dev, const void* goal_dev, const FuelAstarParams* p,
                            void* info_dev, int32_t path_max, void* path_dev, int32_t w_max, void* n_wp_dev,
                            void* waypts_dev) {
  int rc = check_astar_args(m, B, start_dev, goal_dev, p, info_dev, path_max, path_dev, w_max, n_wp_dev, waypts_dev);
  if (rc) return rc;
  FUEL_CUDA(m, cudaSetDevice(m->dev));
  return astar_impl(m, B, (const double*)start_dev, (const double*)goal_dev, p, (FuelPathInfo*)info_dev, path_max,
                    (double*)path_dev, w_max, (int32_t*)n_wp_dev, (double*)waypts_dev);
}

int fuelgpu_astar_batch(FuelMap* m, int32_t B, const double* start, const double* goal, const FuelAstarParams* p,
                        FuelPathInfo* info, int32_t path_max, double* path, int32_t w_max, int32_t* n_wp,
                        double* waypts) {
  int rc = check_astar_args(m, B, start, goal, p, info, path_max, path, w_max, n_wp, waypts);
  if (rc) return rc;
  for (int32_t b = 0; b < B; ++b)
    for (int k = 0; k < 3; ++k)
      if (!isfinite(start[3 * (size_t)b + k]) || !isfinite(goal[3 * (size_t)b + k]))
        return fuel_fail(m, FUELGPU_EINVAL, "query %s%lld: start and goal must be finite", "", (long long)b);
  if (B == 0) return 0;
  FUEL_CUDA(m, cudaSetDevice(m->dev));
  const size_t nb = (size_t)B;
  double *d_s, *d_g, *d_path, *d_wp;
  FuelPathInfo* d_info;
  int32_t* d_n;
  HostStaging st(m);
  st.in(&d_s, start, nb * 3).in(&d_g, goal, nb * 3).out(&d_info, info, nb);
  st.out(&d_path, path, nb * path_max * 3).out(&d_n, n_wp, nb).out(&d_wp, waypts, nb * w_max * 3);
  rc = st.upload();
  if (rc) return rc;
  rc = astar_impl(m, B, d_s, d_g, p, d_info, path_max, d_path, w_max, d_n, d_wp);
  if (rc) return rc;
  return st.download();
}

static int check_kino_args(FuelMap* m, int32_t B, const void* start, const void* vel, const void* acc, const void* goal,
                           const FuelKinoParams* p, const void* info, const void* points, const void* derivs,
                           const void* dt, int32_t node_max, const void* nodes) {
  if (!m) return fuel_fail(nullptr, FUELGPU_EINVAL, "null map");
  if (B < 0) return fuel_fail(m, FUELGPU_EINVAL, "negative batch");
  const int rc = kino_check_params(m, p);
  if (rc) return rc;
  if (nodes && node_max < 1) return fuel_fail(m, FUELGPU_EINVAL, "node_max must be at least 1 with a node buffer");
  if (B > 0 && (!start || !vel || !acc || !goal || !info || !points || !derivs || !dt))
    return fuel_fail(m, FUELGPU_EINVAL, "null argument");
  return 0;
}

int fuelgpu_kino_search_batch_dev(FuelMap* m, int32_t B, const void* start_dev, const void* vel_dev, const void* acc_dev,
                                  const void* goal_dev, const void* gate_dev, const FuelKinoParams* p, void* info_dev,
                                  void* points_dev, void* derivs_dev, void* dt_dev, int32_t node_max, void* nodes_dev,
                                  void* shot_dev) {
  int rc = check_kino_args(m, B, start_dev, vel_dev, acc_dev, goal_dev, p, info_dev, points_dev, derivs_dev, dt_dev,
                           node_max, nodes_dev);
  if (rc) return rc;
  FUEL_CUDA(m, cudaSetDevice(m->dev));
  return kino_search_impl(m, B, (const double*)start_dev, (const double*)vel_dev, (const double*)acc_dev,
                          (const double*)goal_dev, (const FuelPathInfo*)gate_dev, p, (FuelKinoInfo*)info_dev,
                          (double*)points_dev, (double*)derivs_dev, (double*)dt_dev, node_max, (double*)nodes_dev,
                          (double*)shot_dev);
}

int fuelgpu_kino_search_batch(FuelMap* m, int32_t B, const double* start, const double* vel, const double* acc,
                              const double* goal, const FuelKinoParams* p, FuelKinoInfo* info, double* points,
                              double* derivs, double* dt, int32_t node_max, double* nodes, double* shot) {
  int rc = check_kino_args(m, B, start, vel, acc, goal, p, info, points, derivs, dt, node_max, nodes);
  if (rc) return rc;
  for (int32_t b = 0; b < B; ++b)
    for (int k = 0; k < 3; ++k) {
      const size_t i = 3 * (size_t)b + k;
      if (!isfinite(start[i]) || !isfinite(vel[i]) || !isfinite(acc[i]) || !isfinite(goal[i]))
        return fuel_fail(m, FUELGPU_EINVAL, "query %s%lld: start, vel, acc and goal must be finite", "", (long long)b);
    }
  if (B == 0) return 0;
  FUEL_CUDA(m, cudaSetDevice(m->dev));
  const size_t nb = (size_t)B;
  double *d_s, *d_v, *d_a, *d_g, *d_pts, *d_der, *d_dt, *d_nodes, *d_shot;
  FuelKinoInfo* d_info;
  HostStaging st(m);
  st.in(&d_s, start, nb * 3).in(&d_v, vel, nb * 3).in(&d_a, acc, nb * 3).in(&d_g, goal, nb * 3).out(&d_info, info, nb);
  st.out(&d_pts, points, nb * (FUELGPU_MAX_PTS - 2) * 3).out(&d_der, derivs, nb * 12).out(&d_dt, dt, nb);
  st.out(&d_nodes, nodes, nodes ? nb * node_max * 12 : 0).out(&d_shot, shot, nb * 12);
  rc = st.upload();
  if (rc) return rc;
  rc = kino_search_impl(m, B, d_s, d_v, d_a, d_g, nullptr, p, d_info, d_pts, d_der, d_dt, node_max, d_nodes, d_shot);
  if (rc) return rc;
  return st.download();
}

static int check_view_cost_args(FuelMap* m, int32_t P, const void* p1, const void* p2, const void* y1, const void* y2,
                                const void* v1, const FuelViewCostParams* p, const void* info, int32_t path_max,
                                const void* path) {
  if (!m) return fuel_fail(nullptr, FUELGPU_EINVAL, "null map");
  if (P < 0) return fuel_fail(m, FUELGPU_EINVAL, "negative batch");
  if (!p) return fuel_fail(m, FUELGPU_EINVAL, "null params");
  if (!finite_pos(p->vm) || !finite_pos(p->yd)) return fuel_fail(m, FUELGPU_EINVAL, "vm and yd must be finite and positive");
  if (!isfinite(p->w_dir)) return fuel_fail(m, FUELGPU_EINVAL, "w_dir must be finite");
  const int rc = check_astar_params(m, &p->astar);
  if (rc) return rc;
  if (path && path_max < 1) return fuel_fail(m, FUELGPU_EINVAL, "path_max must be at least 1 with a path buffer");
  if (P > 0 && (!p1 || !p2 || !y1 || !y2 || !v1 || !info)) return fuel_fail(m, FUELGPU_EINVAL, "null argument");
  return 0;
}

int fuelgpu_view_cost_batch_dev(FuelMap* m, int32_t P, const void* p1_dev, const void* p2_dev, const void* y1_dev,
                                const void* y2_dev, const void* v1_dev, const FuelViewCostParams* p, void* info_dev,
                                int32_t path_max, void* path_dev) {
  int rc = check_view_cost_args(m, P, p1_dev, p2_dev, y1_dev, y2_dev, v1_dev, p, info_dev, path_max, path_dev);
  if (rc) return rc;
  FUEL_CUDA(m, cudaSetDevice(m->dev));
  return view_cost_impl(m, P, (const double*)p1_dev, (const double*)p2_dev, (const double*)y1_dev,
                        (const double*)y2_dev, (const double*)v1_dev, p, (FuelViewCostInfo*)info_dev, path_max,
                        (double*)path_dev);
}

int fuelgpu_view_cost_batch(FuelMap* m, int32_t P, const double* p1, const double* p2, const double* y1,
                            const double* y2, const double* v1, const FuelViewCostParams* p, FuelViewCostInfo* info,
                            int32_t path_max, double* path) {
  int rc = check_view_cost_args(m, P, p1, p2, y1, y2, v1, p, info, path_max, path);
  if (rc) return rc;
  if (P == 0) return 0;
  FUEL_CUDA(m, cudaSetDevice(m->dev));
  const size_t np = (size_t)P;
  double *d_p1, *d_p2, *d_y1, *d_y2, *d_v1, *d_path;
  FuelViewCostInfo* d_info;
  HostStaging st(m);
  st.in(&d_p1, p1, np * 3).in(&d_p2, p2, np * 3).in(&d_y1, y1, np).in(&d_y2, y2, np).in(&d_v1, v1, np * 3);
  st.out(&d_info, info, np).out(&d_path, path, np * path_max * 3);
  rc = st.upload();
  if (rc) return rc;
  rc = view_cost_impl(m, P, d_p1, d_p2, d_y1, d_y2, d_v1, p, d_info, path_max, d_path);
  if (rc) return rc;
  return st.download();
}

// The structure of a local-tour batch: returns 0 and the group, viewpoint and edge counts, or FUELGPU_EINVAL.
static int check_local_tour_args(FuelMap* m, int32_t B, const int32_t* prob_off, const int32_t* group_off,
                                 const FuelLocalTourParams* p, int32_t kmax, int32_t tour_max, const void* cur_pos,
                                 const void* cur_vel, const void* cur_yaw, const void* vp_pos, const void* vp_yaw,
                                 const void* info, const void* refined, const void* tour, int32_t* G_out,
                                 int32_t* N_out, int64_t* E_out) {
  if (!m) return fuel_fail(nullptr, FUELGPU_EINVAL, "null map");
  if (B < 0) return fuel_fail(m, FUELGPU_EINVAL, "negative batch");
  if (!p) return fuel_fail(m, FUELGPU_EINVAL, "null params");
  const int rc = check_view_cost_args(m, 0, nullptr, nullptr, nullptr, nullptr, nullptr, &p->view, nullptr, 0, nullptr);
  if (rc) return rc;
  if (!isfinite(p->tour_lambda_heu)) return fuel_fail(m, FUELGPU_EINVAL, "tour_lambda_heu must be finite");
  if (tour_max < 1) return fuel_fail(m, FUELGPU_EINVAL, "tour_max must be at least 1");
  if (kmax < 1) return fuel_fail(m, FUELGPU_EINVAL, "kmax must be at least 1");
  *G_out = 0, *N_out = 0, *E_out = 0;
  if (B == 0) return 0;
  if (!prob_off || !group_off || !cur_pos || !cur_vel || !cur_yaw || !info || !refined || !tour)
    return fuel_fail(m, FUELGPU_EINVAL, "null argument");
  if (prob_off[0] != 0) return fuel_fail(m, FUELGPU_EINVAL, "prob_off[0] must be 0");
  for (int32_t b = 0; b < B; ++b) {
    const int32_t ng = prob_off[b + 1] - prob_off[b];
    if (prob_off[b + 1] < prob_off[b] || ng < 1)
      return fuel_fail(m, FUELGPU_EINVAL, "problem %s%lld has no group", "", (long long)b);
    if (ng > kmax) return fuel_fail(m, FUELGPU_EINVAL, "problem %s%lld has more groups than kmax", "", (long long)b);
  }
  const int32_t G = prob_off[B];
  if (group_off[0] != 0) return fuel_fail(m, FUELGPU_EINVAL, "group_off[0] must be 0");
  for (int32_t g = 0; g < G; ++g)
    if (group_off[g + 1] < group_off[g]) return fuel_fail(m, FUELGPU_EINVAL, "group_off decreases at %s%lld", "", g);
  int64_t E = 0;
  for (int32_t b = 0; b < B; ++b) {
    const int32_t g0 = prob_off[b], ng = prob_off[b + 1] - g0;
    if (group_off[g0 + ng] == group_off[g0 + ng - 1])  // final_node would stay null (fast_exploration_manager.cpp:460)
      return fuel_fail(m, FUELGPU_EINVAL, "problem %s%lld: the last group is empty", "", (long long)b);
    int64_t nodes = 1, n_in = 1;
    for (int32_t i = 0; i < ng; ++i) {
      const int64_t sz = group_off[g0 + i + 1] - group_off[g0 + i], eff = i == ng - 1 ? 1 : sz;
      nodes += eff;
      E += eff * n_in;
      n_in = eff;
    }
    if (nodes > FUELGPU_TOUR_MAX_NODES)
      return fuel_fail(m, FUELGPU_EINVAL, "problem %s%lld has more than FUELGPU_TOUR_MAX_NODES nodes", "", (long long)b);
  }
  if (E > INT32_MAX / 2) return fuel_fail(m, FUELGPU_EINVAL, "too many edges in one batch");
  if (G > 0 && (int64_t)G * tour_max > INT32_MAX / 4) return fuel_fail(m, FUELGPU_EINVAL, "groups * tour_max too large");
  if (group_off[G] > 0 && (!vp_pos || !vp_yaw)) return fuel_fail(m, FUELGPU_EINVAL, "null argument");
  *G_out = G, *N_out = group_off[G], *E_out = E;
  return 0;
}

int fuelgpu_local_tour_batch_dev(FuelMap* m, int32_t B, const int32_t* prob_off, const int32_t* group_off,
                                 const void* cur_pos_dev, const void* cur_vel_dev, const void* cur_yaw_dev,
                                 const void* vp_pos_dev, const void* vp_yaw_dev, const FuelLocalTourParams* p,
                                 void* info_dev, int32_t kmax, void* refined_dev, int32_t tour_max, void* tour_dev,
                                 void* edge_cost_dev) {
  int32_t G, N;
  int64_t E;
  int rc = check_local_tour_args(m, B, prob_off, group_off, p, kmax, tour_max, cur_pos_dev, cur_vel_dev, cur_yaw_dev,
                                 vp_pos_dev, vp_yaw_dev, info_dev, refined_dev, tour_dev, &G, &N, &E);
  if (rc || B == 0) return rc;
  FUEL_CUDA(m, cudaSetDevice(m->dev));
  const LocalTourIO io{ (const double*)cur_pos_dev, (const double*)cur_vel_dev, (const double*)cur_yaw_dev,
                        (const double*)vp_pos_dev, (const double*)vp_yaw_dev, (FuelLocalTourInfo*)info_dev,
                        (int32_t*)refined_dev, (double*)tour_dev, (double*)edge_cost_dev, kmax, tour_max };
  return local_tour_impl(m, B, prob_off, group_off, p, io);
}

int fuelgpu_local_tour_batch(FuelMap* m, int32_t B, const int32_t* prob_off, const int32_t* group_off,
                             const double* cur_pos, const double* cur_vel, const double* cur_yaw, const double* vp_pos,
                             const double* vp_yaw, const FuelLocalTourParams* p, FuelLocalTourInfo* info, int32_t kmax,
                             int32_t* refined, int32_t tour_max, double* tour, double* edge_cost) {
  int32_t G, N;
  int64_t E;
  int rc = check_local_tour_args(m, B, prob_off, group_off, p, kmax, tour_max, cur_pos, cur_vel, cur_yaw, vp_pos,
                                 vp_yaw, info, refined, tour, &G, &N, &E);
  if (rc || B == 0) return rc;
  FUEL_CUDA(m, cudaSetDevice(m->dev));
  const size_t nb = (size_t)B, nn = (size_t)N;
  double *d_pos, *d_vel, *d_yaw, *d_vpp, *d_vpy, *d_tour, *d_ec;
  FuelLocalTourInfo* d_info;
  int32_t* d_ref;
  HostStaging st(m);
  st.in(&d_pos, cur_pos, nb * 3).in(&d_vel, cur_vel, nb * 3).in(&d_yaw, cur_yaw, nb);
  st.in(&d_vpp, vp_pos, nn * 3).in(&d_vpy, vp_yaw, nn);
  st.out(&d_info, info, nb).out(&d_ref, refined, nb * kmax).out(&d_tour, tour, nb * tour_max * 3);
  st.out(&d_ec, edge_cost, (size_t)E);
  rc = st.upload();
  if (rc) return rc;
  const LocalTourIO io{ d_pos, d_vel, d_yaw, d_vpp, d_vpy, d_info, d_ref, d_tour, d_ec, kmax, tour_max };
  rc = local_tour_impl(m, B, prob_off, group_off, p, io);
  if (rc) return rc;
  return st.download();
}

// The shape of a global-tour batch: returns 0 and the matrix and index entry counts, or FUELGPU_EINVAL.
static int check_global_tour_args(FuelMap* m, int32_t B, const int32_t* dims, const void* cost, const void* info,
                                  const void* indices, int64_t* n_cost, int64_t* n_idx) {
  if (!m) return fuel_fail(nullptr, FUELGPU_EINVAL, "null map");
  if (B < 0) return fuel_fail(m, FUELGPU_EINVAL, "negative batch");
  *n_cost = 0, *n_idx = 0;
  if (B == 0) return 0;
  if (!dims || !cost || !info || !indices) return fuel_fail(m, FUELGPU_EINVAL, "null argument");
  for (int32_t b = 0; b < B; ++b) {
    const int64_t d = dims[b];
    if (d < 2) return fuel_fail(m, FUELGPU_EINVAL, "instance %s%lld has no cluster (dims < 2)", "", (long long)b);
    if (*n_cost > (INT64_MAX >> 4) - d * d) return fuel_fail(m, FUELGPU_EINVAL, "matrices too large");
    *n_cost += d * d;
    *n_idx += d - 1;
  }
  return 0;
}

int fuelgpu_global_tour_batch_dev(FuelMap* m, int32_t B, const int32_t* dims, const void* cost_dev, void* info_dev,
                                  void* indices_dev) {
  int64_t nc, ni;
  const int rc = check_global_tour_args(m, B, dims, cost_dev, info_dev, indices_dev, &nc, &ni);
  if (rc || B == 0) return rc;
  FUEL_CUDA(m, cudaSetDevice(m->dev));
  return global_tour_impl(m, B, dims, (const double*)cost_dev, (FuelGlobalTourInfo*)info_dev, (int32_t*)indices_dev);
}

int fuelgpu_global_tour_batch(FuelMap* m, int32_t B, const int32_t* dims, const double* cost,
                              FuelGlobalTourInfo* info, int32_t* indices) {
  int64_t nc, ni;
  int rc = check_global_tour_args(m, B, dims, cost, info, indices, &nc, &ni);
  if (rc || B == 0) return rc;
  FUEL_CUDA(m, cudaSetDevice(m->dev));
  double* d_cost;
  FuelGlobalTourInfo* d_info;
  int32_t* d_idx;
  HostStaging st(m);
  st.in(&d_cost, cost, (size_t)nc).out(&d_info, info, (size_t)B).out(&d_idx, indices, (size_t)ni);
  rc = st.upload();
  if (rc) return rc;
  rc = global_tour_impl(m, B, dims, d_cost, d_info, d_idx);
  if (rc) return rc;
  return st.download();
}

}  // extern "C"

