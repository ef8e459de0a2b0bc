// global_tour.cu -- the tour of FastExplorationManager::findGlobalTour (exploration_manager/src/
// fast_exploration_manager.cpp:327-427) on sm_90a: the ATSP over getFullCostMatrix's (n + 1) x (n + 1) matrix that the
// reference hands to LKH, solved exactly by Held-Karp dynamic programming over subsets, for a batch of instances.
//
// Clusters are 0 .. n-1 (matrix node k + 1); node 0 is the current state.  With c the reference's integer matrix
// (int(cost * 100), truncated) the suffix table is
//   h[S][j] = the cheapest path from cluster j through every cluster of S (j not in S), then back to node 0
//   h[{}][j] = c[j+1][0],   h[S][j] = min over k in S of c[j+1][k+1] + h[S \ k][k]
// and cnt[S][j] counts the paths that reach that minimum, saturating at INT32_MAX.  The tour costs
// min over k of c[0][k+1] + h[all \ k][k]; the forward walk that takes the smallest tight k at each step returns the
// lexicographically smallest optimal sequence.
//
// Per group of instances, on the map's main stream with no host synchronisation:
//   1. gt_convert_kernel: one block per instance converts its matrix to int32 and marks BAD_INPUT / TOO_LARGE;
//   2. gt_layer_kernel, once per subset size s = 0 .. n_max - 1: one thread per (S, j not in S) with |S| = s, S from
//      its rank in the combinatorial number system, j the rank's remaining index among the clusters outside S;
//   3. gt_tour_kernel: one warp per instance, a lane per cluster: the cost, n_optimal and the tour, and the status.
// Scratch (FuelMap::gt_buf): the instance table and statuses for the whole batch, then per instance of the group
// al(4 (n+1)^2) + al(8 n 2^n) + al(4 n 2^n) bytes (al: up to a multiple of 256), about 252 MB at n = 20 and 2.8 MB at
// n = 14.  Groups are consecutive instances whose areas sum to at most GT_GROUP_BYTES (4 GiB); TOO_LARGE instances
// take none.
#include "common.cuh"

#include <stdint.h>

#include <algorithm>
#include <vector>

namespace {

constexpr int GT_MAX = FUELGPU_GTOUR_MAX_CLUSTERS;
constexpr int GT_THREADS = 256;
constexpr int GT_TOUR_THREADS = 128;
constexpr int GT_TOUR_WARPS = GT_TOUR_THREADS / 32;
constexpr size_t GT_GROUP_BYTES = (size_t)4 << 30;

struct Binom {
  uint32_t v[GT_MAX + 1][GT_MAX + 1];
};
constexpr Binom make_binom() {
  Binom b{};
  for (int n = 0; n <= GT_MAX; ++n) {
    b.v[n][0] = 1;
    for (int k = 1; k <= n; ++k) b.v[n][k] = b.v[n - 1][k - 1] + (k < n ? b.v[n - 1][k] : 0);
  }
  return b;
}
__device__ constexpr Binom gt_binom = make_binom();
constexpr Binom host_binom = make_binom();

struct GtInst {
  int n;            // clusters (the matrix has n + 1 rows)
  int pad;
  long long cost;   // its first entry in the concatenated matrices
  long long idx;    // its first entry in the concatenated indices
  long long area;   // its bytes in the group area: int32 matrix, h, cnt (0 when TOO_LARGE)
};

__device__ __forceinline__ int* gt_cint(uint8_t* area) { return (int*)area; }
__device__ __forceinline__ size_t gt_al(size_t x) { return (x + 255) & ~(size_t)255; }
__device__ __forceinline__ long long* gt_h(uint8_t* area, int n) {
  return (long long*)(area + gt_al(4 * (size_t)(n + 1) * (n + 1)));
}
__device__ __forceinline__ int* gt_cnt(uint8_t* area, int n) {
  return (int*)((uint8_t*)gt_h(area, n) + gt_al(8 * ((size_t)n << n)));
}

// stage 1: instance blockIdx.x of the group -> its int32 matrix (int int_cost = cost_mat(i, j) * scale, :357-376) and
// its status; the diagonal is never read
__global__ void __launch_bounds__(GT_THREADS)
gt_convert_kernel(const GtInst* __restrict__ inst, const double* __restrict__ cost, uint8_t* group_area,
                  int* __restrict__ status) {
  const GtInst in = inst[blockIdx.x];
  if (in.n > GT_MAX) {
    if (threadIdx.x == 0) status[blockIdx.x] = FUELGPU_GTOUR_TOO_LARGE;
    return;
  }
  const int d = in.n + 1;
  int* c = gt_cint(group_area + in.area);
  const double* src = cost + in.cost;
  bool bad = false;
  for (int e = threadIdx.x; e < d * d; e += GT_THREADS) {
    const double p = src[e] * 100.0;
    // truncation toward zero fits int32 exactly when -2^31 - 1 < p < 2^31; NaN fails both
    const bool ok = p > -2147483649.0 && p < 2147483648.0;
    if (e / d != e % d) bad = bad || !ok;
    c[e] = ok ? __double2int_rz(p) : 0;
  }
  bad = __syncthreads_or(bad);
  if (threadIdx.x == 0) status[blockIdx.x] = bad ? FUELGPU_GTOUR_BAD_INPUT : FUELGPU_GTOUR_OK;
}

// stage 2: the subsets of size s.  Thread t of instance blockIdx.x: rank t / (n - s) -> S (colex order), and the
// (t % (n - s))-th cluster outside S -> j.  Reads layer s - 1 only.
__global__ void __launch_bounds__(GT_THREADS)
gt_layer_kernel(const GtInst* __restrict__ inst, uint8_t* group_area, const int* __restrict__ status, int s) {
  const GtInst in = inst[blockIdx.x];
  const int n = in.n;
  if (n > GT_MAX || s >= n || status[blockIdx.x] != FUELGPU_GTOUR_OK) return;
  const int out = n - s;
  const uint32_t t = blockIdx.y * GT_THREADS + threadIdx.x;
  if (t >= gt_binom.v[n][s] * (uint32_t)out) return;
  uint32_t r = t / out;
  const int jr = t - r * out;
  uint32_t S = 0;
  int p = n - 1;
  for (int i = s; i >= 1; --i) {
    while (gt_binom.v[p][i] > r) --p;
    r -= gt_binom.v[p][i];
    S |= 1u << p;
    --p;
  }
  const uint32_t outside = ~S & ((1u << n) - 1);
  const int j = __fns(outside, 0, jr + 1);
  uint8_t* area = group_area + in.area;
  const int* crow = gt_cint(area) + (size_t)(j + 1) * (n + 1);
  long long* h = gt_h(area, n);
  int* cnt = gt_cnt(area, n);
  long long best;
  int ways;
  if (s == 0) {
    best = crow[0];
    ways = 1;
  } else {
    best = LLONG_MAX;
    ways = 0;
    for (uint32_t rem = S; rem; rem &= rem - 1) {
      const int k = __ffs(rem) - 1;
      const size_t q = (size_t)(S ^ (1u << k)) * n + k;
      const long long v = crow[k + 1] + h[q];
      const int w = cnt[q];
      if (v < best) {
        best = v;
        ways = w;
      } else if (v == best) {
        ways = (int)min((long long)ways + w, (long long)INT32_MAX);
      }
    }
  }
  const size_t q = (size_t)S * n + j;
  h[q] = best;
  cnt[q] = ways;
}

__device__ __forceinline__ long long warp_min_ll(long long v) {
#pragma unroll
  for (int o = 16; o; o >>= 1) v = min(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// stage 3: instance gi of the group per warp -> info and indices
__global__ void __launch_bounds__(GT_TOUR_THREADS)
gt_tour_kernel(int ng, const GtInst* __restrict__ inst, uint8_t* group_area, const int* __restrict__ status,
               FuelGlobalTourInfo* __restrict__ info, int32_t* __restrict__ indices) {
  const int gi = blockIdx.x * GT_TOUR_WARPS + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (gi >= ng) return;
  const GtInst in = inst[gi];
  const int n = in.n, st = status[gi];
  int32_t* idx = indices + in.idx;
  FuelGlobalTourInfo r;
  r.status = st;
  r.n = n;
  r.n_optimal = 0;
  r.reserved = 0;
  r.cost = 0;
  if (st != FUELGPU_GTOUR_OK) {
    for (int i = lane; i < n; i += 32) idx[i] = -1;
    if (lane == 0) info[gi] = r;
    return;
  }
  uint8_t* area = group_area + in.area;
  const int* c = gt_cint(area);
  const long long* h = gt_h(area, n);
  const int* cnt = gt_cnt(area, n);
  const bool mine = lane < n;
  uint32_t S = (1u << n) - 1;
  // the first step from node 0: the tour's cost and its number of optima
  long long v = LLONG_MAX;
  long long w = 0;
  if (mine) {
    const size_t q = (size_t)(S ^ (1u << lane)) * n + lane;
    v = c[lane + 1] + h[q];
    w = cnt[q];
  }
  long long target = warp_min_ll(v);
  long long ways = v == target ? w : 0;
#pragma unroll
  for (int o = 16; o; o >>= 1) ways += __shfl_xor_sync(0xffffffffu, ways, o);
  r.cost = target;
  r.n_optimal = (int)min(ways, (long long)INT32_MAX);
  // forwards: the smallest tight k at each step
  int row = 0;
  for (int step = 0; step < n; ++step) {
    bool tight = false;
    long long hk = 0;
    if (mine && ((S >> lane) & 1u)) {
      hk = h[(size_t)(S ^ (1u << lane)) * n + lane];
      tight = c[(size_t)row * (n + 1) + lane + 1] + hk == target;
    }
    const int k = __ffs(__ballot_sync(0xffffffffu, tight)) - 1;
    target = __shfl_sync(0xffffffffu, hk, k);
    if (lane == 0) idx[step] = k;
    S ^= 1u << k;
    row = k + 1;
  }
  if (lane == 0) info[gi] = r;
}

size_t gt_area_bytes(int n) {
  if (n > GT_MAX) return 0;
  auto al = [](size_t x) { return (x + 255) & ~(size_t)255; };
  return al(4 * (size_t)(n + 1) * (n + 1)) + al(8 * ((size_t)n << n)) + al(4 * ((size_t)n << n));
}

}  // namespace

int global_tour_impl(FuelMap* m, int B, const int32_t* dims, const double* cost, FuelGlobalTourInfo* info,
                     int32_t* indices) {
  if (B == 0) return 0;
  auto al = [](size_t x) { return (x + 255) & ~(size_t)255; };
  std::vector<GtInst> inst((size_t)B);
  std::vector<int> group_start{ 0 };
  size_t area = 0, group_max = 0;
  long long co = 0, io = 0;
  for (int b = 0; b < B; ++b) {
    const int n = dims[b] - 1;
    const size_t need = gt_area_bytes(n);
    if (area + need > GT_GROUP_BYTES && b > group_start.back()) {
      group_start.push_back(b);
      area = 0;
    }
    inst[b] = GtInst{ n, 0, co, io, (long long)area };
    area += need;
    group_max = std::max(group_max, area);
    co += (long long)dims[b] * dims[b];
    io += n;
  }
  group_start.push_back(B);
  const size_t o_inst = 0, o_status = al(sizeof(GtInst) * (size_t)B), o_area = o_status + al(4 * (size_t)B);
  int rc = m->gt_buf.ensure(m, o_area + group_max);
  if (rc) return rc;
  uint8_t* base = m->gt_buf.p;
  GtInst* d_inst = (GtInst*)(base + o_inst);
  int* d_status = (int*)(base + o_status);
  uint8_t* d_area = base + o_area;
  FUEL_CUDA(m, cudaMemcpyAsync(d_inst, inst.data(), sizeof(GtInst) * (size_t)B, cudaMemcpyHostToDevice, m->stream));
  for (size_t g = 0; g + 1 < group_start.size(); ++g) {
    const int b0 = group_start[g], ng = group_start[g + 1] - b0;
    int n_max = 0;
    for (int b = b0; b < b0 + ng; ++b)
      if (inst[b].n <= GT_MAX) n_max = std::max(n_max, inst[b].n);
    gt_convert_kernel<<<ng, GT_THREADS, 0, m->stream>>>(d_inst + b0, cost, d_area, d_status + b0);
    FUEL_LAUNCHES(m, 1);
    FUEL_CUDA(m, cudaGetLastError());
    for (int s = 0; s < n_max; ++s) {
      uint32_t work = 0;  // the most threads one instance needs at this size
      for (int b = b0; b < b0 + ng; ++b)
        if (inst[b].n <= GT_MAX && s < inst[b].n)
          work = std::max(work, host_binom.v[inst[b].n][s] * (uint32_t)(inst[b].n - s));
      const dim3 grid((unsigned)ng, (work + GT_THREADS - 1) / GT_THREADS);
      gt_layer_kernel<<<grid, GT_THREADS, 0, m->stream>>>(d_inst + b0, d_area, d_status + b0, s);
      FUEL_LAUNCHES(m, 1);
      FUEL_CUDA(m, cudaGetLastError());
    }
    gt_tour_kernel<<<(ng + GT_TOUR_WARPS - 1) / GT_TOUR_WARPS, GT_TOUR_THREADS, 0, m->stream>>>(
        ng, d_inst + b0, d_area, d_status + b0, info + b0, indices);
    FUEL_LAUNCHES(m, 1);
    FUEL_CUDA(m, cudaGetLastError());
  }
  return 0;
}
