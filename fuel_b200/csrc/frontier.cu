// frontier.cu -- frontier voxel sweep, region-grow clustering and PCA split on sm_90a.
//
// Replaces FrontierFinder::searchFrontiers' voxel-scale work
// (active_perception/src/frontier_finder.cpp:94-118), expandFrontier (:123-164),
// computeFrontierInfo (:374-390), downsample (:757-774, PCL VoxelGrid restated) and
// splitLargeFrontiers/splitHorizontally (:166-242, Eigen EigenSolver<Matrix2d> restated).
//
// The reference grows clusters one BFS at a time in scan order.  The same partition is
// obtained here without any sequential walk (DESIGN.md "frontier clustering"):
//   P(c)  = flag==0 && FREE && a 6-neighbour is UNKNOWN            (:113, :862-877)
//   E     = P && isInBox(idx) && pos.z >= min_z                    (cells a BFS may absorb, :146-152)
//   S     = P && inside the search box && !E                       (cells that can only be seeds)
//   1. ordered compaction of E and S cells (ascending address)
//   2. union-find over E with 26-connectivity (allNeighbors, :848-860)
//   3. claimer(component) = min( first E cell of the component inside the search box,
//                                first S cell 26-adjacent to the component )
//      -- exactly the seed whose BFS reaches the component first in the reference's scan.
//      Components with no claimer are never reached (flags untouched).
//   4. cluster = all components sharing a claimer (+ the S seed itself); clusters in
//      ascending seed address = tmp_frontiers_ order; size <= cluster_min dropped but flagged.
//   5. level-synchronous PCA split of all clusters at once.
#include "common.cuh"

#include <cooperative_groups.h>

#include <algorithm>
#include <vector>

namespace cg = cooperative_groups;

namespace {

constexpr int NONE = 0x7fffffff;

struct FParams {
  int dom_lo[3], dom_n[3];   // sweep domain (index box, inclusive lo, extent)
  int s_lo[3], s_hi[3];      // search box, inclusive
  int z_min_idx;             // first z index with pos.z >= min_z
  int cluster_min;
  double size_xy;
  float leaf, leaf_inv;      // PCL leaf size (float) and its float inverse
};

__device__ __forceinline__ int tri_at(const Geom& g, const uint8_t* __restrict__ occ, int x, int y,
                                      int z) {
  // getOccupancy(idx): -1 outside the map (sdf_map.h:194-196)
  if (x < 0 || y < 0 || z < 0 || x >= g.nx || y >= g.ny || z >= g.nz) return -1;
  return __ldg(occ + addr_of(g, x, y, z)) & 3;
}

__device__ __forceinline__ bool frontier_pred(const Geom& g, const uint8_t* __restrict__ occ, int x,
                                              int y, int z) {
  // knownfree && isNeighborUnknown (frontier_finder.cpp:862-877)
  if (tri_at(g, occ, x, y, z) != FUELGPU_FREE) return false;
  return tri_at(g, occ, x - 1, y, z) == FUELGPU_UNKNOWN || tri_at(g, occ, x + 1, y, z) == FUELGPU_UNKNOWN ||
         tri_at(g, occ, x, y - 1, z) == FUELGPU_UNKNOWN || tri_at(g, occ, x, y + 1, z) == FUELGPU_UNKNOWN ||
         tri_at(g, occ, x, y, z - 1) == FUELGPU_UNKNOWN || tri_at(g, occ, x, y, z + 1) == FUELGPU_UNKNOWN;
}

// ---- 1. classify + ordered compaction -------------------------------------------------
// One thread per domain voxel (z fastest).  Writes a class byte word per warp (two ballot
// masks) and the per-block count; a second kernel turns masks + scanned block offsets into
// the compact, address-ordered cell list.
constexpr int CLS_BLOCK = 1024;

__global__ void __launch_bounds__(CLS_BLOCK) classify_kernel(Geom g, FParams fp,
                                                             const uint8_t* __restrict__ occ,
                                                             const int8_t* __restrict__ flag,
                                                             uint32_t* __restrict__ maskE,
                                                             uint32_t* __restrict__ maskS,
                                                             int* __restrict__ blockcnt, int64_t ndom) {
  const int64_t L = (int64_t)blockIdx.x * CLS_BLOCK + threadIdx.x;
  bool isE = false, isS = false;
  if (L < ndom) {
    const unsigned Lu = (unsigned)L;  // ndom < 2^31 (checked by the host)
    const unsigned row = Lu / (unsigned)fp.dom_n[2];
    const int z = fp.dom_lo[2] + (int)(Lu - row * (unsigned)fp.dom_n[2]);
    const unsigned xr = row / (unsigned)fp.dom_n[1];
    const int y = fp.dom_lo[1] + (int)(row - xr * (unsigned)fp.dom_n[1]);
    const int x = fp.dom_lo[0] + (int)xr;
    if (flag[addr_of(g, x, y, z)] == 0 && frontier_pred(g, occ, x, y, z)) {
      const bool inbox = x >= g.box_min[0] && x < g.box_max[0] && y >= g.box_min[1] &&
                         y < g.box_max[1] && z >= g.box_min[2] && z < g.box_max[2];
      isE = inbox && z >= fp.z_min_idx;
      const bool ins = x >= fp.s_lo[0] && x <= fp.s_hi[0] && y >= fp.s_lo[1] && y <= fp.s_hi[1] &&
                       z >= fp.s_lo[2] && z <= fp.s_hi[2];
      isS = ins && !isE;
    }
  }
  const unsigned mE = __ballot_sync(0xffffffffu, isE);
  const unsigned mS = __ballot_sync(0xffffffffu, isS);
  const int lane = threadIdx.x & 31;
  if (lane == 0) {
    maskE[L >> 5] = mE;
    maskS[L >> 5] = mS;
  }
  __shared__ int wsum[CLS_BLOCK / 32];
  if (lane == 0) wsum[threadIdx.x >> 5] = __popc(mE) + __popc(mS);
  __syncthreads();
  if (threadIdx.x < 32) {
    int v = wsum[threadIdx.x];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
    if (threadIdx.x == 0) blockcnt[blockIdx.x] = v;
  }
}

// exclusive scan of n ints by one CTA of 1024 threads (n up to a few million)
__device__ void block_scan(const int* __restrict__ in, int* __restrict__ out, int n,
                           int* __restrict__ total) {
  __shared__ int sh[1024];
  __shared__ int carry;
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  for (int base = 0; base < n; base += 1024) {
    const int i = base + threadIdx.x;
    const int v = i < n ? in[i] : 0;
    sh[threadIdx.x] = v;
    __syncthreads();
    for (int o = 1; o < 1024; o <<= 1) {
      int t = threadIdx.x >= o ? sh[threadIdx.x - o] : 0;
      __syncthreads();
      sh[threadIdx.x] += t;
      __syncthreads();
    }
    if (i < n) out[i] = carry + sh[threadIdx.x] - v;
    __syncthreads();
    if (threadIdx.x == 1023) carry += sh[1023];
    __syncthreads();
  }
  if (threadIdx.x == 0 && total) *total = carry;
  __syncthreads();
}
__global__ void __launch_bounds__(1024) scan_kernel(const int* __restrict__ in, int* __restrict__ out,
                                                    int n, int* __restrict__ total) {
  block_scan(in, out, n, total);
}

// large arrays: (a) every CTA scans its own 1024-element chunk, (b) one CTA scans the chunk totals,
// (c) the chunk offsets are added back.
__global__ void __launch_bounds__(1024) scan_chunks_kernel(const int* __restrict__ in, int* __restrict__ out,
                                                           int n, int* __restrict__ chunk_tot) {
  __shared__ int wtot[32];
  const int i = blockIdx.x * 1024 + threadIdx.x;
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int v = i < n ? in[i] : 0;
  int inc = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int u = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += u;
  }
  if (lane == 31) wtot[w] = inc;
  __syncthreads();
  if (w == 0) {
    const int t = wtot[lane];
    int ti = t;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int u = __shfl_up_sync(0xffffffffu, ti, o);
      if (lane >= o) ti += u;
    }
    wtot[lane] = ti - t;
    if (lane == 31) chunk_tot[blockIdx.x] = ti;
  }
  __syncthreads();
  if (i < n) out[i] = wtot[w] + inc - v;
}
__global__ void __launch_bounds__(1024) scan_add_kernel(int* __restrict__ out, int n, const int* __restrict__ chunk_off) {
  const int i = blockIdx.x * 1024 + threadIdx.x;
  if (i < n) out[i] += chunk_off[blockIdx.x];
}

// two exclusive scans at once (both sums < 2^16 are packed in one int): n <= 32768
__device__ void block_scan_small(const int* __restrict__ in, int* __restrict__ out, int n, int* __restrict__ total);
__device__ void block_scan_small2(const int* __restrict__ ina, const int* __restrict__ inb, int* __restrict__ outa,
                                  int* __restrict__ outb, int n, int* __restrict__ tota, int* __restrict__ totb) {
  __shared__ unsigned wtot[32];
  const int t = threadIdx.x, lane = t & 31, w = t >> 5;
  const int chunk = (n + 1023) / 1024;
  const int b0 = t * chunk, b1 = min(b0 + chunk, n);
  unsigned s = 0;
  for (int i = b0; i < b1; ++i) s += ((unsigned)ina[i] << 16) + (unsigned)inb[i];
  unsigned inc = s;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const unsigned v = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += v;
  }
  if (lane == 31) wtot[w] = inc;
  __syncthreads();
  if (w == 0) {
    const unsigned v = wtot[lane];
    unsigned vi = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const unsigned u = __shfl_up_sync(0xffffffffu, vi, o);
      if (lane >= o) vi += u;
    }
    wtot[lane] = vi - v;
    if (lane == 31) {
      *tota = (int)(vi >> 16);
      *totb = (int)(vi & 0xffffu);
    }
  }
  __syncthreads();
  unsigned run = wtot[w] + inc - s;
  for (int i = b0; i < b1; ++i) {
    const unsigned v = ((unsigned)ina[i] << 16) + (unsigned)inb[i];
    outa[i] = (int)(run >> 16);
    outb[i] = (int)(run & 0xffffu);
    run += v;
  }
  __syncthreads();
}

// exclusive scan of a short array (n <= 32 * 1024) by one CTA: every thread owns a contiguous
// chunk, chunk sums are scanned with two levels of warp shuffles.
__device__ void block_scan_small(const int* __restrict__ in, int* __restrict__ out, int n,
                                 int* __restrict__ total) {
  __shared__ int wtot[32];
  const int t = threadIdx.x, lane = t & 31, w = t >> 5;
  const int chunk = (n + 1023) / 1024;
  const int b0 = t * chunk, b1 = min(b0 + chunk, n);
  int s = 0;
  for (int i = b0; i < b1; ++i) s += in[i];
  int inc = s;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int v = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += v;
  }
  if (lane == 31) wtot[w] = inc;
  __syncthreads();
  if (w == 0) {
    int v = wtot[lane];
    int vi = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int u = __shfl_up_sync(0xffffffffu, vi, o);
      if (lane >= o) vi += u;
    }
    wtot[lane] = vi - v;  // exclusive warp offsets
    if (lane == 31 && total) *total = vi;
  }
  __syncthreads();
  int run = wtot[w] + inc - s;
  for (int i = b0; i < b1; ++i) {
    const int v = in[i];
    out[i] = run;
    run += v;
  }
  __syncthreads();
}

__global__ void __launch_bounds__(CLS_BLOCK) compact_kernel(Geom g, FParams fp,
                                                            const uint32_t* __restrict__ maskE,
                                                            const uint32_t* __restrict__ maskS,
                                                            const int* __restrict__ blockoff,
                                                            int* __restrict__ cell_addr,
                                                            uint8_t* __restrict__ cell_cls,
                                                            int* __restrict__ cellidx, int64_t ndom, int cap) {
  const int64_t L = (int64_t)blockIdx.x * CLS_BLOCK + threadIdx.x;
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  unsigned mE = 0, mS = 0;
  if ((L - lane) < ndom) {
    mE = maskE[L >> 5];
    mS = maskS[L >> 5];
  }
  const unsigned m = mE | mS;
  __shared__ int wsum[CLS_BLOCK / 32];
  if (lane == 0) wsum[w] = __popc(m);
  __syncthreads();
  int woff = 0;
  for (int i = 0; i < w; ++i) woff += wsum[i];
  if ((m >> lane) & 1u) {
    const int idx = blockoff[blockIdx.x] + woff + __popc(m & ((1u << lane) - 1u));
    if (idx >= cap) return;  // small-path capacity exceeded: the caller falls back and recompacts
    const unsigned Lu = (unsigned)L;  // ndom < 2^31 (checked by the host)
    const unsigned row = Lu / (unsigned)fp.dom_n[2];
    const int z = fp.dom_lo[2] + (int)(Lu - row * (unsigned)fp.dom_n[2]);
    const unsigned xr = row / (unsigned)fp.dom_n[1];
    const int y = fp.dom_lo[1] + (int)(row - xr * (unsigned)fp.dom_n[1]);
    const int x = fp.dom_lo[0] + (int)xr;
    const int a = (int)addr_of(g, x, y, z);
    cell_addr[idx] = a;
    cell_cls[idx] = ((mE >> lane) & 1u) ? 1 : 2;  // 1 = E, 2 = S
    if (cellidx) cellidx[a] = idx;
  }
}

// ---- 1b. the same sweep, 32 voxels per thread (maps with nz % 32 == 0) -----------------------------------
// One thread per map-aligned 32-voxel z word of a domain row (x, y): the word and its four x/y neighbour words come
// in as 16-byte loads (10 + 2 for frontier_flag_), the predicates are byte-parallel bit operations, the z neighbours
// are shifts of the word's own UNKNOWN mask plus the two bytes beyond its ends.  Word index = row * NW + w, so the
// cells still come out in ascending address.  HBM sees the occupancy byte and the flag byte once: 2 B/voxel.
constexpr int WORD_BLOCK = 256;

struct WordGeom {
  int NW;   // words per row
  int wz0;  // first map word (z >> 5) of the domain
  int64_t nwords;
};

__device__ __forceinline__ uint32_t bits4(uint32_t t) { return ((t & 0x01010101u) * 0x01020408u) >> 24; }
// bit i <-> voxel i of the 32 bytes (v0 = bytes 0..15, v1 = bytes 16..31)
__device__ __forceinline__ uint32_t unknown_mask32(const uint4& v0, const uint4& v1) {
  auto u = [](uint32_t w) { return bits4(~(w | (w >> 1))); };  // (b & 3) == 0
  return u(v0.x) | (u(v0.y) << 4) | (u(v0.z) << 8) | (u(v0.w) << 12) | (u(v1.x) << 16) | (u(v1.y) << 20) |
         (u(v1.z) << 24) | (u(v1.w) << 28);
}
__device__ __forceinline__ uint32_t free_mask32(const uint4& v0, const uint4& v1) {
  auto u = [](uint32_t w) { return bits4(w & ~(w >> 1)); };  // (b & 3) == 1
  return u(v0.x) | (u(v0.y) << 4) | (u(v0.z) << 8) | (u(v0.w) << 12) | (u(v1.x) << 16) | (u(v1.y) << 20) |
         (u(v1.z) << 24) | (u(v1.w) << 28);
}
__device__ __forceinline__ uint32_t zero_mask32(const uint4& v0, const uint4& v1) {
  // byte == 0: bit 7 of ((b & 0x7f) + 0x7f) | b is clear
  auto u = [](uint32_t w) { return bits4(~((((w & 0x7f7f7f7fu) + 0x7f7f7f7fu) | w) >> 7)); };
  return u(v0.x) | (u(v0.y) << 4) | (u(v0.z) << 8) | (u(v0.w) << 12) | (u(v1.x) << 16) | (u(v1.y) << 20) |
         (u(v1.z) << 24) | (u(v1.w) << 28);
}
// bits of the word starting at zb whose z lies in [lo, hi] (inclusive)
__device__ __forceinline__ uint32_t zrange_mask(int zb, int lo, int hi) {
  const int a = max(lo - zb, 0), b = min(hi - zb, 31);
  if (a > b) return 0u;
  return (0xffffffffu >> (31 - b)) & (0xffffffffu << a);
}

__device__ __forceinline__ void word_coords(const FParams& fp, const WordGeom& wg, int64_t W, int& x, int& y, int& zb) {
  const unsigned row = (unsigned)(W / wg.NW);
  const int w = (int)(W - (int64_t)row * wg.NW);
  const unsigned xr = row / (unsigned)fp.dom_n[1];
  y = fp.dom_lo[1] + (int)(row - xr * (unsigned)fp.dom_n[1]);
  x = fp.dom_lo[0] + (int)xr;
  zb = (wg.wz0 + w) << 5;
}

__global__ void __launch_bounds__(WORD_BLOCK) classify_words_kernel(Geom g, FParams fp, WordGeom wg,
                                                                    const uint8_t* __restrict__ occ,
                                                                    const int8_t* __restrict__ flag,
                                                                    uint32_t* __restrict__ maskE,
                                                                    uint32_t* __restrict__ maskS,
                                                                    int* __restrict__ blockcnt) {
  const int64_t W = (int64_t)blockIdx.x * WORD_BLOCK + threadIdx.x;
  uint32_t mE = 0, mS = 0;
  if (W < wg.nwords) {
    int x, y, zb;
    word_coords(fp, wg, W, x, y, zb);
    const int64_t a0 = addr_of(g, x, y, zb);
    const uint4* c = reinterpret_cast<const uint4*>(occ + a0);
    const uint4 c0 = __ldg(c), c1 = __ldg(c + 1);
    const uint32_t fr = free_mask32(c0, c1);
    const uint32_t dz = zrange_mask(zb, fp.dom_lo[2], fp.dom_lo[2] + fp.dom_n[2] - 1);
    if (fr & dz) {
      const uint32_t uc = unknown_mask32(c0, c1);
      uint32_t un = (uc << 1) | (uc >> 1);
      if (zb > 0 && (__ldg(occ + a0 - 1) & 3) == FUELGPU_UNKNOWN) un |= 1u;
      if (zb + 32 < g.nz && (__ldg(occ + a0 + 32) & 3) == FUELGPU_UNKNOWN) un |= 0x80000000u;
      const int64_t sx = (int64_t)g.ny * g.nz;
      if (x > 0) {
        const uint4* q = reinterpret_cast<const uint4*>(occ + a0 - sx);
        un |= unknown_mask32(__ldg(q), __ldg(q + 1));
      }
      if (x + 1 < g.nx) {
        const uint4* q = reinterpret_cast<const uint4*>(occ + a0 + sx);
        un |= unknown_mask32(__ldg(q), __ldg(q + 1));
      }
      if (y > 0) {
        const uint4* q = reinterpret_cast<const uint4*>(occ + a0 - g.nz);
        un |= unknown_mask32(__ldg(q), __ldg(q + 1));
      }
      if (y + 1 < g.ny) {
        const uint4* q = reinterpret_cast<const uint4*>(occ + a0 + g.nz);
        un |= unknown_mask32(__ldg(q), __ldg(q + 1));
      }
      uint32_t P = fr & un & dz;
      if (P) {
        const uint4* fq = reinterpret_cast<const uint4*>(flag + a0);
        P &= zero_mask32(__ldg(fq), __ldg(fq + 1));
      }
      if (P) {
        const bool inbox = x >= g.box_min[0] && x < g.box_max[0] && y >= g.box_min[1] && y < g.box_max[1];
        const bool ins = x >= fp.s_lo[0] && x <= fp.s_hi[0] && y >= fp.s_lo[1] && y <= fp.s_hi[1];
        if (inbox) mE = P & zrange_mask(zb, max(g.box_min[2], fp.z_min_idx), g.box_max[2] - 1);
        if (ins) mS = P & zrange_mask(zb, fp.s_lo[2], fp.s_hi[2]) & ~mE;
      }
    }
    maskE[W] = mE;
    maskS[W] = mS;
  }
  __shared__ int wsum[WORD_BLOCK / 32];
  int v = __popc(mE) + __popc(mS);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
  if ((threadIdx.x & 31) == 0) wsum[threadIdx.x >> 5] = v;
  __syncthreads();
  if (threadIdx.x == 0) {
    int t = 0;
#pragma unroll
    for (int i = 0; i < WORD_BLOCK / 32; ++i) t += wsum[i];
    blockcnt[blockIdx.x] = t;
  }
}

__global__ void __launch_bounds__(WORD_BLOCK) compact_words_kernel(Geom g, FParams fp, WordGeom wg,
                                                                   const uint32_t* __restrict__ maskE,
                                                                   const uint32_t* __restrict__ maskS,
                                                                   const int* __restrict__ blockoff,
                                                                   int* __restrict__ cell_addr,
                                                                   uint8_t* __restrict__ cell_cls,
                                                                   int* __restrict__ cellidx, int cap) {
  const int64_t W = (int64_t)blockIdx.x * WORD_BLOCK + threadIdx.x;
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  uint32_t mE = 0, mS = 0;
  if (W < wg.nwords) {
    mE = maskE[W];
    mS = maskS[W];
  }
  uint32_t m = mE | mS;
  const int cnt = __popc(m);
  int inc = cnt;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int u = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += u;
  }
  __shared__ int wsum[WORD_BLOCK / 32];
  if (lane == 31) wsum[w] = inc;
  __syncthreads();
  if (!m) return;
  int idx = blockoff[blockIdx.x] + inc - cnt;
  for (int i = 0; i < w; ++i) idx += wsum[i];
  int x, y, zb;
  word_coords(fp, wg, W, x, y, zb);
  const int a0 = (int)addr_of(g, x, y, zb);
  while (m) {
    const int b = __ffs(m) - 1;
    m &= m - 1;
    if (idx >= cap) return;  // small-path capacity exceeded: the caller falls back and recompacts
    cell_addr[idx] = a0 + b;
    cell_cls[idx] = ((mE >> b) & 1u) ? 1 : 2;  // 1 = E, 2 = S
    if (cellidx) cellidx[a0 + b] = idx;
    ++idx;
  }
}

// ---- 2. union-find over E cells, 26-connectivity -----------------------------------------
// find with path halving.  The plain stores race benignly with the atomicMin hooks: a parent
// entry is only ever replaced by another member of the same set with a smaller index, so the
// pointers stay acyclic and the component minimum stays the root.
__device__ __forceinline__ int uf_find(int* parent, int i) {
  int p = parent[i];
  while (p != i) {
    const int gp = parent[p];
    if (gp != p) parent[i] = gp;
    i = p;
    p = gp;
  }
  return i;
}
__device__ __forceinline__ int uf_find_ro(const int* parent, int i) {
  int p = parent[i];
  while (p != i) {
    i = p;
    p = parent[i];
  }
  return i;
}
__device__ __forceinline__ void uf_union(int* parent, int a, int b) {
  while (true) {
    a = uf_find(parent, a);
    b = uf_find(parent, b);
    if (a == b) return;
    if (a < b) {
      int t = a;
      a = b;
      b = t;
    }
    const int old = atomicMin(&parent[a], b);
    if (old == a) return;
    a = old;
  }
}

// as uf_union, returning the root of the merged set as far as this thread has seen it
__device__ __forceinline__ int uf_union_root(int* parent, int a, int b) {
  while (true) {
    a = uf_find(parent, a);
    b = uf_find(parent, b);
    if (a == b) return a;
    if (a < b) {
      const int t = a;
      a = b;
      b = t;
    }
    const int old = atomicMin(&parent[a], b);
    if (old == a) return b;
    a = old;
  }
}

__device__ __forceinline__ void init_parent_item(int* parent, int* claim, int* csize, int n, int _tid) {
  const int i = _tid;
  if (i < n) {
    parent[i] = i;
    claim[i] = NONE;
    csize[i] = 0;
  }
}

__device__ __forceinline__ void addr_to_idx(const Geom& g, int a, int& x, int& y, int& z) {
  z = a % g.nz;
  const int r = a / g.nz;
  y = r % g.ny;
  x = r / g.ny;
}

__device__ __forceinline__ void union_item(Geom g, const int* __restrict__ cell_addr,
                             const uint8_t* __restrict__ cell_cls, const int* __restrict__ cellidx,
                             int* parent, int n, int _tid) {
  const int i = _tid;
  if (i >= n || cell_cls[i] != 1) return;
  int x, y, z;
  addr_to_idx(g, cell_addr[i], x, y, z);
  // the 13 neighbours with smaller address: all lookups are issued before any is consumed
  int jn[13];
  int t = 0;
#pragma unroll
  for (int dx = -1; dx <= 0; ++dx)
#pragma unroll
    for (int dy = -1; dy <= 1; ++dy)
#pragma unroll
      for (int dz = -1; dz <= 1; ++dz) {
        if (dx == 0 && (dy > 0 || (dy == 0 && dz >= 0))) continue;
        const int X = x + dx, Y = y + dy, Z = z + dz;
        const bool ok = !(X < 0 || Y < 0 || Z < 0 || Y >= g.ny || Z >= g.nz);
        jn[t++] = ok ? cellidx[addr_of(g, X, Y, Z)] : -1;
      }
#pragma unroll
  for (int q = 0; q < 13; ++q) {
    const int j = jn[q];
    jn[q] = (j >= 0 && cell_cls[j] == 1) ? j : -1;
  }
  // Any ancestor is a valid start for a find: the neighbours' parents are fetched together (one round trip), the
  // unions then run from them and from this cell's current root; equal consecutive parents are the same set already.
#pragma unroll
  for (int q = 0; q < 13; ++q) jn[q] = jn[q] >= 0 ? parent[jn[q]] : -1;
  int r = i, last = -1;
#pragma unroll
  for (int q = 0; q < 13; ++q) {
    const int pj = jn[q];
    if (pj >= 0 && pj != last && pj != r) r = uf_union_root(parent, r, pj);
    if (pj >= 0) last = pj;
  }
}
__device__ __forceinline__ void flatten_item(int* parent, const uint8_t* __restrict__ cell_cls, int n, int _tid) {
  const int i = _tid;
  if (i >= n || cell_cls[i] != 1) return;
  parent[i] = uf_find_ro(parent, i);
}

// ---- 3. claimers ----------------------------------------------------------------------------
__device__ __forceinline__ void claim_item(Geom g, FParams fp, const int* __restrict__ cell_addr,
                             const uint8_t* __restrict__ cell_cls, const int* __restrict__ cellidx,
                             const int* __restrict__ label, int* claim, int n, int _tid) {
  const int i = _tid;
  if (i >= n) return;
  int x, y, z;
  addr_to_idx(g, cell_addr[i], x, y, z);
  if (cell_cls[i] == 1) {
    const bool ins = x >= fp.s_lo[0] && x <= fp.s_hi[0] && y >= fp.s_lo[1] && y <= fp.s_hi[1] &&
                     z >= fp.s_lo[2] && z <= fp.s_hi[2];
    // neighbouring cells mostly share a component: one atomic per component and warp instead of one per cell
    const int key = ins ? label[i] : -1;
    const unsigned grp = __match_any_sync(__activemask(), key);
    if (key >= 0) {
      const int mn = __reduce_min_sync(grp, i);
      if ((int)(threadIdx.x & 31) == __ffs(grp) - 1) atomicMin(&claim[key], mn);
    }
  } else {
    // the 26 lookups go out together, then the classes, then the labels: three round trips instead of one per neighbour
    int jn[26];
    int t = 0;
#pragma unroll
    for (int dx = -1; dx <= 1; ++dx)
#pragma unroll
      for (int dy = -1; dy <= 1; ++dy)
#pragma unroll
        for (int dz = -1; dz <= 1; ++dz) {
          if (dx == 0 && dy == 0 && dz == 0) continue;
          const int X = x + dx, Y = y + dy, Z = z + dz;
          const bool ok = !(X < 0 || Y < 0 || Z < 0 || X >= g.nx || Y >= g.ny || Z >= g.nz);
          jn[t++] = ok ? cellidx[addr_of(g, X, Y, Z)] : -1;
        }
#pragma unroll
    for (int q = 0; q < 26; ++q) {
      const int j = jn[q];
      jn[q] = (j >= 0 && cell_cls[j] == 1) ? j : -1;
    }
#pragma unroll
    for (int q = 0; q < 26; ++q) jn[q] = jn[q] >= 0 ? label[jn[q]] : -1;
    int last = -1;
#pragma unroll
    for (int q = 0; q < 26; ++q) {
      if (jn[q] >= 0 && jn[q] != last) atomicMin(&claim[jn[q]], i);
      if (jn[q] >= 0) last = jn[q];
    }
  }
}

// ---- 4. cluster id (= seed cell index) per cell, sizes, flags --------------------------------
__device__ __forceinline__ void assign_item(const int* __restrict__ cell_addr, const uint8_t* __restrict__ cell_cls,
                              const int* __restrict__ label, const int* __restrict__ claim,
                              int* __restrict__ seed, int* csize, int8_t* __restrict__ flag, int n, int _tid) {
  const int i = _tid;
  int key = -1;
  if (i < n) {
    const int s = cell_cls[i] == 1 ? claim[label[i]] : i;
    seed[i] = s;
    if (s != NONE) {
      key = s;
      flag[cell_addr[i]] = 1;  // frontier_flag_ set for every absorbed cell (:132,:155)
    }
  }
  // cells of a warp mostly share their seed: one size update per seed and warp
  const unsigned grp = __match_any_sync(__activemask(), key);
  if (key >= 0 && (int)(threadIdx.x & 31) == __ffs(grp) - 1) atomicAdd(&csize[key], __popc(grp));
}

// per cell: 1 if it is the seed of a kept cluster (for the rank scan), and kept-cell marks
__device__ __forceinline__ void mark_item(const int* __restrict__ seed, const int* __restrict__ csize, int cluster_min,
                            int* __restrict__ is_root, int* __restrict__ is_kept, int n, int _tid) {
  const int i = _tid;
  if (i >= n) return;
  const int s = seed[i];
  const bool kept = s != NONE && csize[s] > cluster_min;  // expanded.size() > cluster_min_ (:157)
  is_kept[i] = kept ? 1 : 0;
  is_root[i] = (kept && s == i) ? 1 : 0;
}

__device__ __forceinline__ void reset_cellidx_item(const int* __restrict__ cell_addr, int* __restrict__ cellidx, int n, int _tid) {
  const int i = _tid;
  if (i < n) cellidx[cell_addr[i]] = -1;
}

// kept cells -> dense arrays; cellidx now maps voxel -> kept index
__device__ __forceinline__ void gather_kept_item(const int* __restrict__ cell_addr, const int* __restrict__ seed,
                                   const int* __restrict__ is_kept, const int* __restrict__ kept_off,
                                   const int* __restrict__ root_rank, int* __restrict__ k_addr,
                                   int* __restrict__ k_cl, int* __restrict__ cellidx, int n, int _tid) {
  const int i = _tid;
  if (i >= n) return;
  if (is_kept[i]) {
    const int k = kept_off[i];
    k_addr[k] = cell_addr[i];
    k_cl[k] = root_rank[seed[i]];
    cellidx[cell_addr[i]] = k;
  } else {
    cellidx[cell_addr[i]] = -1;
  }
}

// ---- 5. split levels ----------------------------------------------------------------------------
struct ClusterMeta {  // persistent per cluster
  int root;           // rank of the root cluster (tmp_frontiers_ order before the split)
  unsigned path;      // split path, left aligned (bit 31 = first split; 0 = ftr1, 1 = ftr2)
  int depth;
  int active;         // 1 while the cluster may still split
  double mean[3];
  double pc[2];
  int do_split;
  int new_id;
};

struct ClusterStat {  // per cluster, rebuilt every level while the cluster is active
  long long sx, sy, sz;
  int n;
  int lo[3], hi[3];
  // covariance of filtered cells in exact two-part fixed point
  long long cxx_hi, cxx_lo, cxy_hi, cxy_lo, cyy_hi, cyy_lo;
  int nfilt;
  int need_split;
  int cnt0, cnt1;  // partition sizes
};


__device__ __forceinline__ void stat_reset_item(ClusterStat* st, const ClusterMeta* __restrict__ meta, int C, int _tid) {
  const int c = _tid;
  if (c >= C || !meta[c].active) return;  // finished clusters keep their last statistics
  ClusterStat s;
  memset(&s, 0, sizeof(s));
  s.lo[0] = s.lo[1] = s.lo[2] = NONE;
  s.hi[0] = s.hi[1] = s.hi[2] = -1;
  st[c] = s;
}

__device__ __forceinline__ void stat_accum_item(Geom g, const int* __restrict__ k_addr, const int* __restrict__ k_cl,
                                  const ClusterMeta* __restrict__ meta, ClusterStat* st, int K, int _tid) {
  // Cells arrive in address order, so the lanes of a warp mostly share a cluster: lanes with the
  // same cluster id are reduced in-warp (match_any + reduce_sync) and ONE lane issues the atomics.
  // All sums are exact integers -> the result does not depend on the grouping.
  const int k = _tid;
  int c = -1, x = 0, y = 0, z = 0;
  if (k < K) {
    c = k_cl[k];
    if (!meta[c].active)
      c = -1;
    else
      addr_to_idx(g, k_addr[k], x, y, z);
  }
  const unsigned act = __activemask();
  const unsigned grp = __match_any_sync(act, c);
  if (c < 0) return;
  const int sx = __reduce_add_sync(grp, x), sy = __reduce_add_sync(grp, y), sz = __reduce_add_sync(grp, z);
  const int lx = __reduce_min_sync(grp, x), ly = __reduce_min_sync(grp, y), lz = __reduce_min_sync(grp, z);
  const int hx = __reduce_max_sync(grp, x), hy = __reduce_max_sync(grp, y), hz = __reduce_max_sync(grp, z);
  if ((int)(threadIdx.x & 31) != __ffs(grp) - 1) return;
  ClusterStat* s = &st[c];
  atomicAdd((unsigned long long*)&s->sx, (unsigned long long)sx);
  atomicAdd((unsigned long long*)&s->sy, (unsigned long long)sy);
  atomicAdd((unsigned long long*)&s->sz, (unsigned long long)sz);
  atomicAdd(&s->n, __popc(grp));
  atomicMin(&s->lo[0], lx);
  atomicMin(&s->lo[1], ly);
  atomicMin(&s->lo[2], lz);
  atomicMax(&s->hi[0], hx);
  atomicMax(&s->hi[1], hy);
  atomicMax(&s->hi[2], hz);
}

// average_ of computeFrontierInfo (:376-386).  The reference sums positions sequentially in
// fp64; here the index sums are exact integers and the mean is formed once (differs from
// the sequential sum by rounding only, ~1e-16 relative).
__device__ __forceinline__ void mean_item(Geom g, ClusterMeta* meta, const ClusterStat* __restrict__ st, int C, int _tid) {
  const int c = _tid;
  if (c >= C || !meta[c].active) return;
  const ClusterStat& s = st[c];
  const double inv = 1.0 / (double)s.n;
  meta[c].mean[0] = ((double)s.sx * inv + 0.5) * g.res + g.origin[0];
  meta[c].mean[1] = ((double)s.sy * inv + 0.5) * g.res + g.origin[1];
  meta[c].mean[2] = ((double)s.sz * inv + 0.5) * g.res + g.origin[2];
}

__device__ __forceinline__ float cell_posf(const Geom& g, int id, int axis) {
  // (float) of indexToPos (sdf_map.h:132-135); PointXYZ narrowing at frontier_finder.cpp:762
  return (float)((id + 0.5) * g.res + g.origin[axis]);
}
// leaf coordinate of PCL VoxelGrid: (int)(floorf(p * inv_leaf) - (float)min_b)
__device__ __forceinline__ int leaf_coord(const Geom& g, const FParams& fp, int id, int axis, int min_b) {
  return (int)(floorf(cell_posf(g, id, axis) * fp.leaf_inv) - (float)min_b);
}

// PCL VoxelGrid restated per cell: the min-address cell of every occupied leaf computes the
// leaf centroid (float accumulation in ascending address order) and contributes to the split
// test (:183-189) and the covariance (:194-200).
template <bool LOCALMEAN = false>  // true: form the cluster mean from the statistics here (same expression as mean_item)
__device__ __forceinline__ void downsample_item(Geom g, FParams fp, const int* __restrict__ k_addr,
                                  const int* __restrict__ k_cl, const int* __restrict__ cellidx,
                                  const ClusterMeta* __restrict__ meta, ClusterStat* st,
                                  float* __restrict__ k_cent, int* __restrict__ k_leaf, int K, int _tid) {
  const int k = _tid;
  if (k >= K) return;
  const int c = k_cl[k];
  if (!meta[c].active) return;
  k_leaf[k] = -1;
  int id[3];
  addr_to_idx(g, k_addr[k], id[0], id[1], id[2]);
  const ClusterStat& s = st[c];
  int min_b[3], lc[3], lo[3], hi[3], div_b[3];
  const int nmax[3] = { g.nx, g.ny, g.nz };
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    min_b[a] = (int)floorf(cell_posf(g, s.lo[a], a) * fp.leaf_inv);
    const int max_b = (int)floorf(cell_posf(g, s.hi[a], a) * fp.leaf_inv);
    div_b[a] = max_b - min_b[a] + 1;
    lc[a] = leaf_coord(g, fp, id[a], a, min_b[a]);
    lo[a] = id[a];
    hi[a] = id[a];
    while (lo[a] - 1 >= 0 && lo[a] - 1 >= s.lo[a] && leaf_coord(g, fp, lo[a] - 1, a, min_b[a]) == lc[a]) --lo[a];
    while (hi[a] + 1 < nmax[a] && hi[a] + 1 <= s.hi[a] && leaf_coord(g, fp, hi[a] + 1, a, min_b[a]) == lc[a]) ++hi[a];
  }
  // The leaf's voxels in ascending address order (a leaf spans at most 4 voxels per axis).  All
  // cellidx lookups are issued first, then all cluster-id lookups (two memory round trips
  // instead of one per voxel), then the float accumulation runs in the reference order.
  int jj[64];
  const int a0 = (int)addr_of(g, lo[0], lo[1], lo[2]);
  const int sx = g.ny * g.nz, sy = g.nz;
  const int ex = hi[0] - lo[0], ey = hi[1] - lo[1], ez = hi[2] - lo[2];
#pragma unroll
  for (int dx = 0; dx < 4; ++dx)
#pragma unroll
    for (int dy = 0; dy < 4; ++dy)
#pragma unroll
      for (int dz = 0; dz < 4; ++dz) {
        const bool ok = dx <= ex && dy <= ey && dz <= ez;
        jj[(dx * 4 + dy) * 4 + dz] = ok ? cellidx[a0 + dx * sx + dy * sy + dz] : -1;
      }
#pragma unroll
  for (int v = 0; v < 64; ++v) {
    const int j = jj[v];
    jj[v] = (j >= 0 && k_cl[j] == c) ? j : -1;
  }
  float px[4], py[4], pz[4];  // the (float) positions of the leaf's voxel rows, formed once
#pragma unroll
  for (int d = 0; d < 4; ++d) {
    px[d] = cell_posf(g, lo[0] + d, 0);
    py[d] = cell_posf(g, lo[1] + d, 1);
    pz[d] = cell_posf(g, lo[2] + d, 2);
  }
  float sum[3] = { 0.f, 0.f, 0.f };
  int cnt = 0;
  bool owner = true;
#pragma unroll
  for (int v = 0; v < 64; ++v) {
    const int j = jj[v];
    if (j >= 0 && owner) {
      if (cnt == 0 && j != k) owner = false;  // a smaller-address cell owns this leaf
      sum[0] += px[v / 16];
      sum[1] += py[(v / 4) % 4];
      sum[2] += pz[v % 4];
      ++cnt;
    }
  }
  if (!owner) return;
  const float fc = (float)cnt;
  const float cx = sum[0] / fc, cy = sum[1] / fc, cz = sum[2] / fc;
  k_cent[3 * k] = cx;
  k_cent[3 * k + 1] = cy;
  k_cent[3 * k + 2] = cz;
  k_leaf[k] = lc[0] + lc[1] * div_b[0] + lc[2] * div_b[0] * div_b[1];
  atomicAdd(&st[c].nfilt, 1);
  double m0 = meta[c].mean[0], m1 = meta[c].mean[1];
  if (LOCALMEAN) {
    const double inv = 1.0 / (double)s.n;
    m0 = ((double)s.sx * inv + 0.5) * g.res + g.origin[0];
    m1 = ((double)s.sy * inv + 0.5) * g.res + g.origin[1];
  }
  const double dx = (double)cx - m0, dy = (double)cy - m1;
  if (sqrt(dx * dx + dy * dy) > fp.size_xy) atomicOr(&st[c].need_split, 1);
}

// covariance terms as exact two-part fixed point: p = hi*2^-20 + lo*2^-82
__device__ __forceinline__ double fx_get(long long hi, long long lo) {
  return (double)hi * (1.0 / 1048576.0) + (double)lo * (1.0 / 4835703278458516698824704.0);
}

// sum of a 64-bit value over the lanes of grp (mod 2^64, like the atomics it replaces): three 21/21/22-bit limbs
// go through the 32-bit warp reduction
__device__ __forceinline__ unsigned long long group_sum_u64(unsigned grp, unsigned long long v) {
  const unsigned a = (unsigned)(v & 0x1fffffull), b = (unsigned)((v >> 21) & 0x1fffffull), c = (unsigned)(v >> 42);
  const unsigned long long sa = __reduce_add_sync(grp, a), sb = __reduce_add_sync(grp, b), sc = __reduce_add_sync(grp, c);
  return sa + (sb << 21) + (sc << 42);
}
__device__ __forceinline__ void fx_split(double p, unsigned long long* hi, unsigned long long* lo) {
  const double h = rint(p * 1048576.0);          // 2^20
  const double l = (p - h * (1.0 / 1048576.0));  // exact, |l| <= 2^-21
  *hi = (unsigned long long)(long long)h;
  *lo = (unsigned long long)(long long)rint(l * 4835703278458516698824704.0);  // 2^82
}

// The sums are exact integers (two-part fixed point), so the lanes of a warp that share a cluster are added up in the
// warp first and ONE lane issues the six atomics: same result, a fraction of the atomic traffic on the cluster's record.
template <bool LOCALMEAN = false>  // true: form the cluster mean from the statistics here (same expression as mean_item)
__device__ __forceinline__ void cov_item(Geom g, const int* __restrict__ k_cl, const int* __restrict__ k_leaf,
                           const float* __restrict__ k_cent, const ClusterMeta* __restrict__ meta,
                           ClusterStat* st, int K, int _tid) {
  const int k = _tid;
  int c = -1;
  if (k < K) {
    c = k_cl[k];
    if (!meta[c].active || k_leaf[k] < 0 || !st[c].need_split) c = -1;
  }
  const unsigned grp = __match_any_sync(__activemask(), c);
  if (c < 0) return;
  double m0 = meta[c].mean[0], m1 = meta[c].mean[1];
  if (LOCALMEAN) {
    const ClusterStat& s = st[c];
    const double inv = 1.0 / (double)s.n;
    m0 = ((double)s.sx * inv + 0.5) * g.res + g.origin[0];
    m1 = ((double)s.sy * inv + 0.5) * g.res + g.origin[1];
  }
  const double dx = (double)k_cent[3 * k] - m0;
  const double dy = (double)k_cent[3 * k + 1] - m1;
  unsigned long long v[6];
  fx_split(dx * dx, &v[0], &v[1]);
  fx_split(dx * dy, &v[2], &v[3]);
  fx_split(dy * dy, &v[4], &v[5]);
  if (grp & (grp - 1)) {
#pragma unroll
    for (int q = 0; q < 6; ++q) v[q] = group_sum_u64(grp, v[q]);
  }
  if ((int)(threadIdx.x & 31) != __ffs(grp) - 1) return;
  ClusterStat* sc = &st[c];
  atomicAdd((unsigned long long*)&sc->cxx_hi, v[0]);
  atomicAdd((unsigned long long*)&sc->cxx_lo, v[1]);
  atomicAdd((unsigned long long*)&sc->cxy_hi, v[2]);
  atomicAdd((unsigned long long*)&sc->cxy_lo, v[3]);
  atomicAdd((unsigned long long*)&sc->cyy_hi, v[4]);
  atomicAdd((unsigned long long*)&sc->cyy_lo, v[5]);
}

// Eigen 3.3 EigenSolver<Matrix2d> restated for a symmetric matrix: RealSchur (findSmallSubdiagEntry,
// splitOffTwoRows, JacobiRotation::makeGivens) + doComputeEigenvectors back-substitution
// (third-party convention reconstructed from the published algorithm; unpinned, SURVEY 8c).
__device__ void make_givens(double p, double q, double* c, double* s) {
  if (q == 0.0) {
    *c = p < 0 ? -1.0 : 1.0;
    *s = 0.0;
  } else if (p == 0.0) {
    *c = 0.0;
    *s = q < 0 ? 1.0 : -1.0;
  } else if (fabs(p) > fabs(q)) {
    double t = q / p;
    double u = sqrt(1.0 + t * t);
    if (p < 0) u = -u;
    *c = 1.0 / u;
    *s = -t * (*c);
  } else {
    double t = p / q;
    double u = sqrt(1.0 + t * t);
    if (q < 0) u = -u;
    *s = -1.0 / u;
    *c = -t * (*s);
  }
}
// products and sums are kept un-contracted (no FMA) to follow the host arithmetic
#define MUL(a, b) __dmul_rn((a), (b))
#define ADD(a, b) __dadd_rn((a), (b))
__device__ void principal_axis_2x2(double a, double b, double d, double pc[2]) {
  const double eps = 2.220446049250313e-16;
  double T[2][2] = { { a, b }, { b, d } };
  double U[2][2] = { { 1, 0 }, { 0, 1 } };
  const double norm = fabs(a) + fabs(b) + fabs(b) + fabs(d);
  if (norm != 0.0) {
    const double s = fabs(T[0][0]) + fabs(T[1][1]);
    const double thr = MUL(s, eps);
    if (!(fabs(T[1][0]) <= thr)) {
      const double p = MUL(0.5, T[0][0] - T[1][1]);
      const double q = ADD(MUL(p, p), MUL(T[1][0], T[0][1]));
      if (q >= 0) {
        const double z = sqrt(fabs(q));
        double c, sn;
        if (p >= 0)
          make_givens(p + z, T[1][0], &c, &sn);
        else
          make_givens(p - z, T[1][0], &c, &sn);
        for (int j = 0; j < 2; ++j) {
          const double x = T[0][j], y = T[1][j];
          T[0][j] = ADD(MUL(c, x), -MUL(sn, y));
          T[1][j] = ADD(MUL(sn, x), MUL(c, y));
        }
        for (int i = 0; i < 2; ++i) {
          const double x = T[i][0], y = T[i][1];
          T[i][0] = ADD(MUL(c, x), -MUL(sn, y));
          T[i][1] = ADD(MUL(sn, x), MUL(c, y));
        }
        T[1][0] = 0.0;
        for (int i = 0; i < 2; ++i) {
          const double x = U[i][0], y = U[i][1];
          U[i][0] = ADD(MUL(c, x), -MUL(sn, y));
          U[i][1] = ADD(MUL(sn, x), MUL(c, y));
        }
      }
    } else {
      T[1][0] = 0.0;
    }
  }
  double e1[2];
  {
    const double w = T[0][0] - T[1][1];
    const double r = T[0][1];
    e1[0] = (w != 0.0) ? -r / w : -r / MUL(eps, norm);
    e1[1] = 1.0;
  }
  double v0[2] = { ADD(MUL(U[0][0], 1.0), MUL(U[0][1], 0.0)), ADD(MUL(U[1][0], 1.0), MUL(U[1][1], 0.0)) };
  double v1[2] = { ADD(MUL(U[0][0], e1[0]), MUL(U[0][1], e1[1])), ADD(MUL(U[1][0], e1[0]), MUL(U[1][1], e1[1])) };
  const double n0 = sqrt(ADD(MUL(v0[0], v0[0]), MUL(v0[1], v0[1])));
  const double n1 = sqrt(ADD(MUL(v1[0], v1[0]), MUL(v1[1], v1[1])));
  if (n0 > 0) { v0[0] /= n0; v0[1] /= n0; }
  if (n1 > 0) { v1[0] /= n1; v1[1] /= n1; }
  const int max_idx = (T[1][1] > T[0][0]) ? 1 : 0;  // ties -> 0 (:207-212)
  pc[0] = max_idx == 0 ? v0[0] : v1[0];
  pc[1] = max_idx == 0 ? v0[1] : v1[1];
}

__device__ __forceinline__ void pca_item(ClusterMeta* meta, const ClusterStat* __restrict__ st, int C, int _tid) {
  const int c = _tid;
  if (c >= C || !meta[c].active) return;
  const ClusterStat& s = st[c];
  meta[c].do_split = 0;
  if (!s.need_split || meta[c].depth >= 32) return;
  const double m = (double)s.nfilt;
  const double cxx = fx_get(s.cxx_hi, s.cxx_lo) / m, cxy = fx_get(s.cxy_hi, s.cxy_lo) / m,
               cyy = fx_get(s.cyy_hi, s.cyy_lo) / m;
  principal_axis_2x2(cxx, cxy, cyy, meta[c].pc);
  meta[c].do_split = 1;
}

__device__ __forceinline__ int cell_side(const Geom& g, const ClusterMeta& mt, int addr) {
  int x, y, z;
  addr_to_idx(g, addr, x, y, z);
  const double px = (x + 0.5) * g.res + g.origin[0], py = (y + 0.5) * g.res + g.origin[1];
  // (cell.head<2>() - mean).dot(first_pc) >= 0 -> ftr1 (:218-223)
  const double d = ADD(MUL(px - mt.mean[0], mt.pc[0]), MUL(py - mt.mean[1], mt.pc[1]));
  return d >= 0 ? 0 : 1;
}

__device__ __forceinline__ void side_count_item(Geom g, const int* __restrict__ k_addr, const int* __restrict__ k_cl,
                                  const ClusterMeta* __restrict__ meta, ClusterStat* st, int K, int _tid) {
  const int k = _tid;
  int c = -1, side = 0;
  if (k < K) {
    c = k_cl[k];
    if (!meta[c].active || !meta[c].do_split)
      c = -1;
    else
      side = cell_side(g, meta[c], k_addr[k]);
  }
  const unsigned act = __activemask();
  const unsigned grp = __match_any_sync(act, c);
  if (c < 0) return;
  const int n1 = __reduce_add_sync(grp, side);
  if ((int)(threadIdx.x & 31) != __ffs(grp) - 1) return;
  const int n0 = __popc(grp) - n1;
  if (n0) atomicAdd(&st[c].cnt0, n0);
  if (n1) atomicAdd(&st[c].cnt1, n1);
}

// decide splits, allocate ids for the ftr2 halves, update metadata.  Single thread block
// scan over clusters keeps ids deterministic.
__device__ void split_alloc(ClusterMeta* meta, const ClusterStat* __restrict__ st, int C,
                            int* __restrict__ n_new) {
  __shared__ int sh[1024];
  __shared__ int carry;
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  for (int base = 0; base < C; base += 1024) {
    const int c = base + threadIdx.x;
    int v = 0;
    if (c < C && meta[c].active) {
      if (meta[c].do_split && st[c].cnt0 > 0 && st[c].cnt1 > 0)
        v = 1;
      else {
        meta[c].do_split = 0;
        meta[c].active = 0;  // final
      }
    }
    sh[threadIdx.x] = v;
    __syncthreads();
    for (int o = 1; o < 1024; o <<= 1) {
      int t = threadIdx.x >= o ? sh[threadIdx.x - o] : 0;
      __syncthreads();
      sh[threadIdx.x] += t;
      __syncthreads();
    }
    if (v) {
      const int nid = C + carry + sh[threadIdx.x] - 1;
      ClusterMeta& p = meta[c];
      ClusterMeta ch = p;
      p.new_id = nid;
      ch.path = p.path | (1u << (31 - p.depth));
      ch.depth = p.depth + 1;
      ch.active = 1;
      ch.do_split = 0;
      p.depth += 1;
      meta[nid] = ch;  // child fields that matter: root, path, depth, active
      // parent's mean/pc are still needed by relabel_kernel this level; child's copy is unused
    }
    __syncthreads();
    if (threadIdx.x == 1023) carry += sh[1023];
    __syncthreads();
  }
  if (threadIdx.x == 0) *n_new = carry;
}

__device__ __forceinline__ void relabel_item(Geom g, const int* __restrict__ k_addr, int* __restrict__ k_cl,
                               const ClusterMeta* __restrict__ meta, int K, int C_old, int _tid) {
  const int k = _tid;
  if (k >= K) return;
  const int c = k_cl[k];
  if (c >= C_old || !meta[c].do_split) return;
  if (cell_side(g, meta[c], k_addr[k]) == 1) k_cl[k] = meta[c].new_id;
}

__device__ __forceinline__ void clear_do_split_item(ClusterMeta* meta, int C, int _tid) {
  const int c = _tid;
  if (c < C) meta[c].do_split = 0;
}

__device__ __forceinline__ void init_meta_item(ClusterMeta* meta, int R, int _tid) {
  const int c = _tid;
  if (c >= R) return;
  ClusterMeta m;
  memset(&m, 0, sizeof(m));
  m.root = c;
  m.active = 1;
  meta[c] = m;
}

// ---- grid-stride wrappers of the per-item functions (large inputs) ----
__global__ void init_parent_kernel(int* parent, int* claim, int* csize, int n) {
  init_parent_item(parent, claim, csize, n, blockIdx.x * blockDim.x + threadIdx.x);
}

__global__ void union_kernel(Geom g, const int* __restrict__ cell_addr,
                             const uint8_t* __restrict__ cell_cls, const int* __restrict__ cellidx,
                             int* parent, int n) {
  union_item(g, cell_addr, cell_cls, cellidx, parent, n, blockIdx.x * blockDim.x + threadIdx.x);
}

__global__ void flatten_kernel(int* parent, const uint8_t* __restrict__ cell_cls, int n) {
  flatten_item(parent, cell_cls, n, blockIdx.x * blockDim.x + threadIdx.x);
}

__global__ void claim_kernel(Geom g, FParams fp, const int* __restrict__ cell_addr,
                             const uint8_t* __restrict__ cell_cls, const int* __restrict__ cellidx,
                             const int* __restrict__ label, int* claim, int n) {
  claim_item(g, fp, cell_addr, cell_cls, cellidx, label, claim, n, blockIdx.x * blockDim.x + threadIdx.x);
}

__global__ void assign_kernel(const int* __restrict__ cell_addr, const uint8_t* __restrict__ cell_cls,
                              const int* __restrict__ label, const int* __restrict__ claim,
                              int* __restrict__ seed, int* csize, int8_t* __restrict__ flag, int n) {
  assign_item(cell_addr, cell_cls, label, claim, seed, csize, flag, n, blockIdx.x * blockDim.x + threadIdx.x);
}

__global__ void mark_kernel(const int* __restrict__ seed, const int* __restrict__ csize, int cluster_min,
                            int* __restrict__ is_root, int* __restrict__ is_kept, int n) {
  mark_item(seed, csize, cluster_min, is_root, is_kept, n, blockIdx.x * blockDim.x + threadIdx.x);
}

__global__ void reset_cellidx_kernel(const int* __restrict__ cell_addr, int* __restrict__ cellidx, int n) {
  reset_cellidx_item(cell_addr, cellidx, n, blockIdx.x * blockDim.x + threadIdx.x);
}

__global__ void gather_kept_kernel(const int* __restrict__ cell_addr, const int* __restrict__ seed,
                                   const int* __restrict__ is_kept, const int* __restrict__ kept_off,
                                   const int* __restrict__ root_rank, int* __restrict__ k_addr,
                                   int* __restrict__ k_cl, int* __restrict__ cellidx, int n) {
  gather_kept_item(cell_addr, seed, is_kept, kept_off, root_rank, k_addr, k_cl, cellidx, n, blockIdx.x * blockDim.x + threadIdx.x);
}

// The split levels run without the host: the counts live in device memory (ctl), every level kernel leaves at once
// when the previous level made no new cluster (ctl->n_new == 0), so the host enqueues levels blind and looks at the
// counters once per batch.  The cluster count of level L is read from ccur and written (by the single-CTA
// split_alloc) to cnext: the two slots alternate, so no kernel of a level races with the update.
struct LevelCtl {
  const int* R;    // root clusters (scan total)
  const int* K;    // kept cells (scan total)
  int* n_new;      // clusters created by the last level that ran; doubles as the "keep going" flag
  int* c_final;    // cluster count after the last level that ran
  int* ccur;       // cluster count at the start of this level
  int* cnext;      // ... of the next one
};

__global__ void stat_accum_kernel(Geom g, const int* __restrict__ k_addr, const int* __restrict__ k_cl,
                                  const ClusterMeta* __restrict__ meta, ClusterStat* st, LevelCtl ctl) {
  if (*ctl.n_new == 0) return;
  stat_accum_item(g, k_addr, k_cl, meta, st, *ctl.K, blockIdx.x * blockDim.x + threadIdx.x);
}

// VoxelGrid pass and covariance form the cluster mean from the statistics themselves (LOCALMEAN: the expression of
// mean_item); the mean is stored by pca_kernel for the later consumers (side test, relabel, average_)
__global__ void downsample_kernel(Geom g, FParams fp, const int* __restrict__ k_addr,
                                  const int* __restrict__ k_cl, const int* __restrict__ cellidx,
                                  const ClusterMeta* __restrict__ meta, ClusterStat* st,
                                  float* __restrict__ k_cent, int* __restrict__ k_leaf, LevelCtl ctl) {
  if (*ctl.n_new == 0) return;
  downsample_item<true>(g, fp, k_addr, k_cl, cellidx, meta, st, k_cent, k_leaf, *ctl.K, blockIdx.x * blockDim.x + threadIdx.x);
}

__global__ void cov_kernel(Geom g, const int* __restrict__ k_cl, const int* __restrict__ k_leaf,
                           const float* __restrict__ k_cent, const ClusterMeta* __restrict__ meta,
                           ClusterStat* st, LevelCtl ctl) {
  if (*ctl.n_new == 0) return;
  cov_item<true>(g, k_cl, k_leaf, k_cent, meta, st, *ctl.K, blockIdx.x * blockDim.x + threadIdx.x);
}

__global__ void pca_kernel(Geom g, ClusterMeta* meta, const ClusterStat* __restrict__ st, LevelCtl ctl) {
  if (*ctl.n_new == 0) return;
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  mean_item(g, meta, st, *ctl.ccur, c);
  pca_item(meta, st, *ctl.ccur, c);
}

__global__ void side_count_kernel(Geom g, const int* __restrict__ k_addr, const int* __restrict__ k_cl,
                                  const ClusterMeta* __restrict__ meta, ClusterStat* st, LevelCtl ctl) {
  if (*ctl.n_new == 0) return;
  side_count_item(g, k_addr, k_cl, meta, st, *ctl.K, blockIdx.x * blockDim.x + threadIdx.x);
}

__global__ void __launch_bounds__(1024) split_alloc_kernel(ClusterMeta* meta, const ClusterStat* __restrict__ st,
                                                           LevelCtl ctl) {
  if (*ctl.n_new == 0) return;  // (uniform: nothing below has written it yet)
  const int C = *ctl.ccur;
  __shared__ int made;
  split_alloc(meta, st, C, &made);
  __syncthreads();
  if (threadIdx.x == 0) {
    *ctl.cnext = C + made;
    *ctl.c_final = C + made;
    *ctl.n_new = made;
  }
}

// the cells of the ftr2 halves take their new ids; afterwards the parents' split marks are cleared
__global__ void relabel_kernel(Geom g, const int* __restrict__ k_addr, int* __restrict__ k_cl,
                               const ClusterMeta* __restrict__ meta, LevelCtl ctl) {
  if (*ctl.n_new == 0) return;
  relabel_item(g, k_addr, k_cl, meta, *ctl.K, *ctl.ccur, blockIdx.x * blockDim.x + threadIdx.x);
}

// end of a level: the parents' split marks are cleared and the statistics of every cluster that is still active
// (children included) are reset for the next level
__global__ void next_level_kernel(ClusterMeta* meta, ClusterStat* st, LevelCtl ctl) {
  if (*ctl.n_new == 0) return;
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  clear_do_split_item(meta, *ctl.ccur, c);
  stat_reset_item(st, meta, *ctl.cnext, c);
}

__global__ void init_meta_kernel(ClusterMeta* meta, ClusterStat* st, LevelCtl ctl) {
  const int R = *ctl.R;
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  init_meta_item(meta, R, c);
  stat_reset_item(st, meta, R, c);
  if (c == 0) {
    *ctl.ccur = R;
    *ctl.c_final = R;
    *ctl.n_new = (R > 0 && *ctl.K > 0) ? 1 : 0;
  }
}


// ---- small inputs: the whole clustering + split in ONE single-CTA launch --------------------
// Per-search work on a room-sized map is a few thousand frontier cells: every phase is far
// below one launch latency, so the multi-kernel pipeline is pure launch + host-sync overhead.
// Here one CTA of 1024 threads runs all phases back to back with __syncthreads() in between
// and iterates the split levels on the device.  Same per-item functions as the large path.
constexpr int SMALL_CTAS = 8;      // one thread-block cluster (portable maximum)
constexpr int SMALL_CAP = 32768;   // candidate cells
constexpr int SMALL_CCAP = 8192;   // clusters (incl. split products)
// The small path's result block: the kernel's tail writes the arrays fuelgpu_frontier_fetch hands out, in their final
// order, and the block comes back with the counters in one copy.  A search with more kept cells, clusters or filtered
// cells than these caps is marshalled on the host from an exact-size download (frontier_marshal).
constexpr int RES_K0 = 12288, RES_C0 = 256, RES_F0 = 4096;
constexpr size_t al16(size_t b) { return (b + 15) & ~(size_t)15; }
// byte offsets in the block: int counters[16] ([0] n_cand [1] R [2] K [3] n_new [4] status [5] C [8] assembled [9] NF),
// int cell_off[C+1], int filt_off[C+1], double average[3C], int box[6C] (lo xyz, hi xyz), int cell_addr[K],
// double filtered[3 NF] -- clusters in output order
constexpr size_t RB_CELL_OFF = 64;
constexpr size_t RB_FILT_OFF = RB_CELL_OFF + al16(sizeof(int) * (RES_C0 + 1));
constexpr size_t RB_AVG = RB_FILT_OFF + al16(sizeof(int) * (RES_C0 + 1));
constexpr size_t RB_BOX = RB_AVG + al16(sizeof(double) * 3 * RES_C0);
constexpr size_t RB_ADDR = RB_BOX + al16(sizeof(int) * 6 * RES_C0);
constexpr size_t RB_FILT = RB_ADDR + al16(sizeof(int) * RES_K0);
constexpr size_t RB_BYTES = RB_FILT + al16(sizeof(double) * 3 * RES_F0);
// the tail's scratch (ints): per cluster cell count, filtered count, output rank; per kept cell its place in cell_addr
// and in its cluster's filtered range (kept order); per filtered slot its kept cell, leaf and cluster rank
constexpr size_t ASM_SCR = 3 * RES_C0 + 2 * RES_K0 + 3 * RES_F0;
constexpr unsigned TAG_PAD = 0x8000u;  // a kept cell's tag: cluster id | 0x100 if it holds a VoxelGrid centroid
static_assert(RES_C0 <= 256 && RES_C0 <= SMALL_CTAS * 32, "cluster ids fit a tag byte, one warp per cluster");
static_assert(RES_K0 % 128 == 0 && sizeof(int) * RES_F0 <= sizeof(unsigned short) * RES_K0, "tail's shared memory");


// Small path: the kept/root marks of 32 consecutive cells are one ballot, so the rank scan runs over ceil(n/32) <= 1024
// chunk counts (one pass of one CTA) instead of n cells.  Arrays reused as: is_kept[q] / is_root[q] = the ballots of
// chunk q, kept_off[q] / root_rank[q] = exclusive counts before chunk q.
__device__ __forceinline__ void mark_chunk_item(const int* __restrict__ seed, const int* __restrict__ csize, int cluster_min,
                                                int* __restrict__ root_mask, int* __restrict__ kept_mask, int n, int i) {
  bool kept = false, root = false;
  if (i < n) {
    const int s = seed[i];
    kept = s != NONE && csize[s] > cluster_min;  // expanded.size() > cluster_min_ (:157)
    root = kept && s == i;
  }
  const unsigned mk = __ballot_sync(0xffffffffu, kept), mr = __ballot_sync(0xffffffffu, root);
  if ((i & 31) == 0 && i < n) {
    kept_mask[i >> 5] = (int)mk;
    root_mask[i >> 5] = (int)mr;
  }
}
__device__ void chunk_scan_small(const int* __restrict__ root_mask, const int* __restrict__ kept_mask,
                                 int* __restrict__ root_off, int* __restrict__ kept_off, int nchunk,
                                 int* __restrict__ tot_root, int* __restrict__ tot_kept) {
  __shared__ unsigned wtot2[32];
  const int t = threadIdx.x, lane = t & 31, w = t >> 5;
  const unsigned v = t < nchunk ? ((unsigned)__popc((unsigned)root_mask[t]) << 16) + (unsigned)__popc((unsigned)kept_mask[t]) : 0u;
  unsigned inc = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const unsigned u = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += u;
  }
  if (lane == 31) wtot2[w] = inc;
  __syncthreads();
  if (w == 0) {
    const unsigned x = wtot2[lane];
    unsigned xi = x;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const unsigned u = __shfl_up_sync(0xffffffffu, xi, o);
      if (lane >= o) xi += u;
    }
    wtot2[lane] = xi - x;
    if (lane == 31) {
      *tot_root = (int)(xi >> 16);
      *tot_kept = (int)(xi & 0xffffu);
    }
  }
  __syncthreads();
  if (t < nchunk) {
    const unsigned ex = wtot2[w] + inc - v;
    root_off[t] = (int)(ex >> 16);
    kept_off[t] = (int)(ex & 0xffffu);
  }
}
__device__ __forceinline__ void gather_chunk_item(const int* __restrict__ cell_addr, const int* __restrict__ seed,
                                                  const int* __restrict__ kept_mask, const int* __restrict__ kept_off,
                                                  const int* __restrict__ root_mask, const int* __restrict__ root_off,
                                                  int* __restrict__ k_addr, int* __restrict__ k_cl,
                                                  int* __restrict__ cellidx, int n, int i) {
  if (i >= n) return;
  const unsigned mk = (unsigned)kept_mask[i >> 5];
  const int a = cell_addr[i];
  if ((mk >> (i & 31)) & 1u) {
    const int k = kept_off[i >> 5] + __popc(mk & ((1u << (i & 31)) - 1u));
    const int s = seed[i];
    k_addr[k] = a;
    k_cl[k] = root_off[s >> 5] + __popc((unsigned)root_mask[s >> 5] & ((1u << (s & 31)) - 1u));
    cellidx[a] = k;
  } else {
    cellidx[a] = -1;
  }
}

struct SmallBufs {
  int *cell_addr, *parent, *claim, *csize, *seed, *is_root, *is_kept, *root_rank, *kept_off;
  uint8_t* cell_cls;
  int *k_addr, *k_cl, *k_leaf;
  float* k_cent;
  ClusterMeta* meta;
  ClusterStat* stat;
  int* counters;  // [0] n_cand (in) [1] R [2] K [3] n_new [4] status [5] C
  char* res;      // the result block the host fetches with ONE copy (RB_* layout)
  int* scr;       // ASM_SCR ints for the tail
  int assemble;   // 0: leave the ordering to the host (counters only)
};

// ---- the tail of the small path: the result in output order ---------------------------------------------------------
// The same arrays and order as frontier_build_csr: clusters by (root, path), a cluster's cells in ascending address
// (= kept index), its filtered cells by (leaf, kept index).  Phase A: cell / filtered counts per cluster (warp-aggregated
// atomics) and the output rank of every cluster (one warp per cluster, O(C) compares).
__device__ __forceinline__ void tail_count_item(const int* __restrict__ k_cl, const int* __restrict__ k_leaf,
                                                int* __restrict__ cnt_cell, int* __restrict__ cnt_filt, int K, int k) {
  const int c = k < K ? k_cl[k] : -1;
  const int cf = (k < K && k_leaf[k] >= 0) ? c : -1;
  const unsigned pc = __match_any_sync(0xffffffffu, c), pf = __match_any_sync(0xffffffffu, cf);
  const int lane = k & 31;
  if (c >= 0 && lane == __ffs(pc) - 1) atomicAdd(cnt_cell + c, __popc(pc));
  if (cf >= 0 && lane == __ffs(pf) - 1) atomicAdd(cnt_filt + cf, __popc(pf));
}
__device__ __forceinline__ void tail_rank_warp(const ClusterMeta* __restrict__ meta, int* __restrict__ crank, int C, int c,
                                               int lane) {
  const int r0 = meta[c].root;
  const unsigned p0 = meta[c].path;
  int lt = 0;
  for (int c2 = lane; c2 < C; c2 += 32) {
    const int r2 = meta[c2].root;
    const unsigned p2 = meta[c2].path;
    lt += r2 < r0 || (r2 == r0 && (p2 < p0 || (p2 == p0 && c2 < c)));
  }
  lt = __reduce_add_sync(0xffffffffu, lt);
  if (lane == 0) crank[c] = lt;
}
// Phase B.  Every CTA first copies the tags of all kept cells into shared memory (tail_tags); then one warp per cluster c
// writes its CSR offsets (sum of the counts of the clusters ranked before it), average_ and box, and runs once over the
// tags, four cells per lane, to give each of its cells its place in cell_addr and each of its filtered cells its place
// in the cluster's filtered range, both in ascending kept index.  Only stores leave the loop.
__device__ __forceinline__ void tail_tags(const int* __restrict__ k_cl, const int* __restrict__ k_leaf,
                                          unsigned short* __restrict__ tag, int K) {
  const int Kp = (K + 127) & ~127;
  for (int k = threadIdx.x; k < Kp; k += blockDim.x)
    tag[k] = (unsigned short)(k < K ? (unsigned)k_cl[k] | (k_leaf[k] >= 0 ? 0x100u : 0u) : TAG_PAD);
}
__device__ __forceinline__ void tail_place_warp(const ClusterMeta* __restrict__ meta, const ClusterStat* __restrict__ st,
                                                const unsigned short* __restrict__ tag, int* __restrict__ scr,
                                                char* __restrict__ res, int K, int C, int c, int lane) {
  const int *cnt_cell = scr, *cnt_filt = scr + RES_C0, *crank = scr + 2 * RES_C0;
  int* pos = scr + 3 * RES_C0;
  int* fpos = pos + RES_K0;
  const int r = crank[c];
  int co = 0, fo = 0;
  for (int c2 = lane; c2 < C; c2 += 32) {
    if (crank[c2] < r) {
      co += cnt_cell[c2];
      fo += cnt_filt[c2];
    }
  }
  co = __reduce_add_sync(0xffffffffu, co);
  fo = __reduce_add_sync(0xffffffffu, fo);
  int* cell_off = (int*)(res + RB_CELL_OFF);
  int* filt_off = (int*)(res + RB_FILT_OFF);
  if (lane == 0) {
    cell_off[r] = co;
    filt_off[r] = fo;
    if (r == C - 1) {
      cell_off[C] = co + cnt_cell[c];
      filt_off[C] = fo + cnt_filt[c];
    }
  }
  if (lane < 3) {
    ((double*)(res + RB_AVG))[3 * r + lane] = meta[c].mean[lane];
    ((int*)(res + RB_BOX))[6 * r + lane] = st[c].lo[lane];
    ((int*)(res + RB_BOX))[6 * r + 3 + lane] = st[c].hi[lane];
  }
  const int Kp = (K + 127) & ~127;
  for (int base = 0; base < Kp; base += 128) {
    const uint2 w = *(const uint2*)(tag + base + 4 * lane);
    const unsigned t[4] = { w.x & 0xffffu, w.x >> 16, w.y & 0xffffu, w.y >> 16 };
    unsigned mine = 0, filt = 0;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      if ((t[j] & 0x80ffu) == (unsigned)c) {
        mine |= 1u << j;
        if (t[j] & 0x100u) filt |= 1u << j;
      }
    }
    if (!__any_sync(0xffffffffu, mine)) continue;
    // exclusive prefix over the lanes of (cells, filtered cells), packed 16/16 (at most 128 each)
    const unsigned v = (unsigned)__popc(mine) | ((unsigned)__popc(filt) << 16);
    unsigned inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const unsigned u = __shfl_up_sync(0xffffffffu, inc, o);
      if (lane >= o) inc += u;
    }
    const unsigned tot = __shfl_sync(0xffffffffu, inc, 31), ex = inc - v;
    int pm = co + (int)(ex & 0xffffu), pf = fo + (int)(ex >> 16);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      if ((mine >> j) & 1u) {
        pos[base + 4 * lane + j] = pm++;
        if ((filt >> j) & 1u) fpos[base + 4 * lane + j] = pf++;
      }
    }
    co += (int)(tot & 0xffffu);
    fo += (int)(tot >> 16);
  }
}
// Phase C, one thread per kept cell: its address to its place; a filtered cell lists (kept index, leaf, cluster rank)
// in its slot of the filtered range (kept order inside the cluster)
__device__ __forceinline__ void tail_scatter_item(const int* __restrict__ k_addr, const int* __restrict__ k_cl,
                                                  const int* __restrict__ k_leaf, const int* __restrict__ scr,
                                                  int* __restrict__ f_k, int* __restrict__ f_leaf, int* __restrict__ f_r,
                                                  char* __restrict__ res, int K, int k) {
  if (k >= K) return;
  const int *crank = scr + 2 * RES_C0, *pos = scr + 3 * RES_C0, *fpos = pos + RES_K0;
  ((int*)(res + RB_ADDR))[pos[k]] = k_addr[k];
  const int lf = k_leaf[k];
  if (lf >= 0) {
    const int s = fpos[k];
    f_k[s] = k;
    f_leaf[s] = lf;
    f_r[s] = crank[k_cl[k]];
  }
}
// Phase D, one thread per filtered slot i, the leaves of all slots in shared memory: its place in the cluster is the
// number of slots of the range with a smaller (leaf, kept index); the centroid goes there as the double fetch returns
__device__ __forceinline__ void tail_filtered_item(const float* __restrict__ k_cent, const int* __restrict__ f_k,
                                                   const int* __restrict__ s_leaf, const int* __restrict__ f_r,
                                                   char* __restrict__ res, int NF, int i) {
  if (i >= NF) return;
  const int* filt_off = (const int*)(res + RB_FILT_OFF);
  const int r = f_r[i], lo = filt_off[r], hi = filt_off[r + 1], lf = s_leaf[i];
  int pos = lo;
#pragma unroll 4
  for (int j = lo; j < hi; ++j) {
    const int l2 = s_leaf[j];
    pos += l2 < lf || (l2 == lf && j < i);
  }
  const int k = f_k[i];
  double* out = (double*)(res + RB_FILT);
  out[3 * pos] = (double)k_cent[3 * k];
  out[3 * pos + 1] = (double)k_cent[3 * k + 1];
  out[3 * pos + 2] = (double)k_cent[3 * k + 2];
}

__global__ void __cluster_dims__(SMALL_CTAS, 1, 1) __launch_bounds__(1024) cluster_small_kernel(Geom g, FParams fp, int8_t* __restrict__ flag,
                                                             int* __restrict__ cellidx, SmallBufs b) {
  cg::cluster_group cluster = cg::this_cluster();
  const int rank = (int)cluster.block_rank();
  // items go to warps round-robin over the CTAs (32 consecutive items per warp): a few thousand cells keep all 8 SMs
  // busy instead of filling the first CTAs only
  const int tid = (((int)threadIdx.x >> 5) * SMALL_CTAS + rank) * 32 + ((int)threadIdx.x & 31);
  constexpr int NT = 1024 * SMALL_CTAS;
  const int n = b.counters[0];
#ifdef FUEL_PROF
  long long* prof = (long long*)(b.counters + 8);
  int pi = 0;
#define STAMP() do { if (tid == 0) { long long t_; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t_)); prof[pi++] = t_; } } while (0)
#else
#define STAMP() do {} while (0)
#endif
  STAMP();
  int* r_counters = (int*)b.res;
  if (n > SMALL_CAP) {
    if (tid == 0) {
      b.counters[4] = 1;
      r_counters[0] = n;
      r_counters[4] = 1;
    }
    return;  // uniform over the whole cluster
  }
#define FOR_ITEMS(i, N) for (int i = tid; i - tid < (N); i += NT)  // uniform trip count per warp
  FOR_ITEMS(i, n) init_parent_item(b.parent, b.claim, b.csize, n, i);
  cluster.sync();
  STAMP();
  FOR_ITEMS(i, n) union_item(g, b.cell_addr, b.cell_cls, cellidx, b.parent, n, i);
  cluster.sync();
  STAMP();
  FOR_ITEMS(i, n) flatten_item(b.parent, b.cell_cls, n, i);
  cluster.sync();
  STAMP();
  FOR_ITEMS(i, n) claim_item(g, fp, b.cell_addr, b.cell_cls, cellidx, b.parent, b.claim, n, i);
  cluster.sync();
  STAMP();
  FOR_ITEMS(i, n) assign_item(b.cell_addr, b.cell_cls, b.parent, b.claim, b.seed, b.csize, flag, n, i);
  cluster.sync();
  STAMP();
  FOR_ITEMS(i, n) mark_chunk_item(b.seed, b.csize, fp.cluster_min, b.is_root, b.is_kept, n, i);
  cluster.sync();
  STAMP();
  if (rank == 0) chunk_scan_small(b.is_root, b.is_kept, b.root_rank, b.kept_off, (n + 31) >> 5, b.counters + 1, b.counters + 2);
  cluster.sync();
  STAMP();
  const int R = b.counters[1], K = b.counters[2];
  int C = R;
  int status = 0;
  if (R > 0 && K > 0) {
    FOR_ITEMS(i, n) gather_chunk_item(b.cell_addr, b.seed, b.is_kept, b.kept_off, b.is_root, b.root_rank, b.k_addr, b.k_cl,
                                      cellidx, n, i);
    FOR_ITEMS(c, R) {
      init_meta_item(b.meta, R, c);
      stat_reset_item(b.stat, b.meta, R, c);
    }
    if (b.assemble) FOR_ITEMS(c, 2 * RES_C0) if (c < 2 * RES_C0) b.scr[c] = 0;  // the tail's per-cluster counts
    cluster.sync();
    STAMP();
    for (int level = 0; level < 40; ++level) {
      if (2 * C > SMALL_CCAP) {
        status = 2;
        break;
      }
      FOR_ITEMS(k, K) stat_accum_item(g, b.k_addr, b.k_cl, b.meta, b.stat, K, k);
      cluster.sync();
      STAMP();
      // the cluster means are written for the later phases while the VoxelGrid pass forms its own copy
      FOR_ITEMS(c, C) mean_item(g, b.meta, b.stat, C, c);
      FOR_ITEMS(k, K) downsample_item<true>(g, fp, b.k_addr, b.k_cl, cellidx, b.meta, b.stat, b.k_cent, b.k_leaf, K, k);
      cluster.sync();
      STAMP();
      FOR_ITEMS(k, K) cov_item(g, b.k_cl, b.k_leaf, b.k_cent, b.meta, b.stat, K, k);
      cluster.sync();
      STAMP();
      FOR_ITEMS(c, C) pca_item(b.meta, b.stat, C, c);
      cluster.sync();
      STAMP();
      FOR_ITEMS(k, K) side_count_item(g, b.k_addr, b.k_cl, b.meta, b.stat, K, k);
      cluster.sync();
      STAMP();
      if (rank == 0) split_alloc(b.meta, b.stat, C, b.counters + 3);
      cluster.sync();
      STAMP();
      FOR_ITEMS(k, K) relabel_item(g, b.k_addr, b.k_cl, b.meta, K, C, k);
      cluster.sync();
      STAMP();
      const int n_new = b.counters[3];
      if (n_new == 0) break;
      FOR_ITEMS(c, C) clear_do_split_item(b.meta, C, c);
      C += n_new;
      FOR_ITEMS(c, C) stat_reset_item(b.stat, b.meta, C, c);  // for the next level (children included)
      cluster.sync();
      STAMP();
    }
  }
  FOR_ITEMS(i, n) reset_cellidx_item(b.cell_addr, cellidx, n, i);
  // the result in output order (every value the tail reads is final since the last cluster.sync(), whichever CTA
  // wrote it); the conditions are uniform over the cluster
  int assembled = 0, NF = 0;
  if (b.assemble && status == 0 && R > 0 && K > 0 && K <= RES_K0 && C <= RES_C0) {
    __shared__ __align__(16) unsigned short s_tag[RES_K0];  // phase B: kept-cell tags; phase D: the slots' leaves
    int* f_k = b.scr + 3 * RES_C0 + 2 * RES_K0;
    int* f_leaf = f_k + RES_F0;
    int* f_r = f_leaf + RES_F0;
    const int gw = tid >> 5, lane = tid & 31;  // one warp per cluster: 8 x 32 warps >= RES_C0
    FOR_ITEMS(k, K) tail_count_item(b.k_cl, b.k_leaf, b.scr, b.scr + RES_C0, K, k);
    if (gw < C) tail_rank_warp(b.meta, b.scr + 2 * RES_C0, C, gw, lane);
    cluster.sync();
    STAMP();
    tail_tags(b.k_cl, b.k_leaf, s_tag, K);
    __syncthreads();
    if (gw < C) tail_place_warp(b.meta, b.stat, s_tag, b.scr, b.res, K, C, gw, lane);
    cluster.sync();
    STAMP();
    NF = ((const int*)(b.res + RB_FILT_OFF))[C];
    if (NF <= RES_F0) {  // (uniform)
      FOR_ITEMS(k, K) tail_scatter_item(b.k_addr, b.k_cl, b.k_leaf, b.scr, f_k, f_leaf, f_r, b.res, K, k);
      cluster.sync();
      STAMP();
      int* s_leaf = (int*)s_tag;  // (RES_F0 ints fit in the tags' space)
      for (int i = threadIdx.x; i < NF; i += blockDim.x) s_leaf[i] = f_leaf[i];
      __syncthreads();
      FOR_ITEMS(i, NF) tail_filtered_item(b.k_cent, f_k, s_leaf, f_r, b.res, NF, i);
      STAMP();
      assembled = 1;
    }
  }
  if (tid == 0) {
    b.counters[4] = status;
    b.counters[5] = C;
    const int out[10] = { n, R, K, b.counters[3], status, C, b.counters[6], b.counters[7], assembled, NF };
#pragma unroll
    for (int j = 0; j < 10; ++j) r_counters[j] = out[j];
  }
#undef FOR_ITEMS
}

__global__ void is_changed_kernel(Geom g, const uint8_t* __restrict__ occ, const int* __restrict__ offs,
                                  const int* __restrict__ addr, uint8_t* __restrict__ changed, int* __restrict__ counts,
                                  int m) {
  // isFrontierChanged (:365-372) / the change count of isFrontierCovered (:703-712): one block per stored cluster
  const int c = blockIdx.x;
  if (c >= m) return;
  __shared__ int cnt;
  if (threadIdx.x == 0) cnt = 0;
  __syncthreads();
  int mine = 0;
  for (int i = offs[c] + threadIdx.x; i < offs[c + 1]; i += blockDim.x) {
    int x, y, z;
    addr_to_idx(g, addr[i], x, y, z);
    if (!frontier_pred(g, occ, x, y, z)) ++mine;
  }
  if (mine) atomicAdd(&cnt, mine);
  __syncthreads();
  if (threadIdx.x == 0) {
    if (changed) changed[c] = (uint8_t)(cnt > 0);
    if (counts) counts[c] = cnt;
  }
}

}  // namespace

struct SweepPlan {  // how the voxel sweep of a search is laid out
  bool words = false;  // 32 voxels per thread (nz % 32 == 0) or one voxel per thread
  unsigned nb = 0;     // CTAs = entries of blockcnt / blockoff
  size_t nmask = 0;    // mask words
  int64_t ndom = 0;
  WordGeom wg;
};

struct HostView {  // result arrays in pinned host memory
  const int *addr, *cl, *leaf;
  const float* cent;
  const ClusterMeta* meta;
  const ClusterStat* stat;
};

struct FrontierState {
  int* cellidx = nullptr;  // voxel -> cell index, -1 elsewhere (persistent, sparse use)
  DevBuf<uint32_t> maskE, maskS;
  DevBuf<int> blockcnt, blockoff, scan_tot, scan_off;
  DevBuf<int> cell_addr, parent, claim, csize, seed, is_root, is_kept, root_rank, kept_off;
  DevBuf<uint8_t> cell_cls;
  DevBuf<int> k_addr, k_cl, k_leaf;
  DevBuf<float> k_cent;
  DevBuf<ClusterStat> stat;
  DevBuf<ClusterMeta> meta;
  DevBuf<char> res;     // the small path's result block (RB_* layout), fetched with one copy
  DevBuf<int> asm_scr;  // scratch of the kernel's tail (ASM_SCR)
  // a search that has been enqueued (begin) but not yet collected (end)
  bool pend_active = false, pend_empty = true;
  FParams pend_fp;
  SweepPlan pend_plan;
  cudaStream_t stream = nullptr;  // the frontier subsystem's own stream
  cudaEvent_t ev_in = nullptr;
  cudaEvent_t ev_out = nullptr;  // end of the last enqueued search: writers of `occ` on the main stream wait for it
  bool ev_out_valid = false;
  DevBuf<char, true> h_pin;  // pinned host staging for the exact-size download (frontier_marshal)
  // pinned copies of the result block, used in turn: a search fills the one that does not hold the result of the last
  // collected search, so fuelgpu_frontier_fetch may still read that one after the next search_begin
  DevBuf<char, true> h_res[2];
  int pend_blk = 0;  // block the pending search is copied into
  int res_blk = -1;  // block holding the result of the last collected search; -1: the h_* vectors hold it
  int* d_counters = nullptr;  // [0] n_cand [1] n_roots [2] n_kept [3] n_new [4] small-path status [5] C
  // results of the last search marshalled on the host (CSR)
  std::vector<int32_t> h_cell_off, h_cell_addr, h_filt_off;
  std::vector<double> h_filtered, h_avg, h_bmin, h_bmax;
  int cell_order = FUELGPU_CELLS_BY_ADDRESS;  // fuelgpu_frontier_set_cell_order
  float last_leaf = 0.f;                      // PCL leaf size of the last search
};

cudaStream_t frontier_stream_raw(FuelMap* m) { return m->fs->stream; }
cudaStream_t frontier_stream(FuelMap* m) {
  FrontierState* f = m->fs;
  cudaEventRecord(f->ev_in, m->stream);
  cudaStreamWaitEvent(f->stream, f->ev_in, 0);
  return f->stream;
}

int frontier_set_cell_order(FuelMap* m, int order) {
  if (order != FUELGPU_CELLS_BY_ADDRESS && order != FUELGPU_CELLS_BFS)
    return fuel_fail(m, FUELGPU_EINVAL, "unknown cell order");
  m->fs->cell_order = order;
  return 0;
}

void frontier_order_writer(FuelMap* m) {
  FrontierState* f = m->fs;
  if (f && f->ev_out_valid) cudaStreamWaitEvent(m->stream, f->ev_out, 0);
}

int frontier_state_create(FuelMap* m) {
  m->fs = new FrontierState();
  FUEL_CUDA(m, cudaStreamCreateWithFlags(&m->fs->stream, cudaStreamNonBlocking));
  FUEL_CUDA(m, cudaEventCreateWithFlags(&m->fs->ev_in, cudaEventDisableTiming));
  FUEL_CUDA(m, cudaEventCreateWithFlags(&m->fs->ev_out, cudaEventDisableTiming));
  FUEL_CUDA(m, cudaMalloc(&m->fs->cellidx, sizeof(int) * m->nvox));
  FUEL_CUDA(m, cudaMemsetAsync(m->fs->cellidx, 0xff, sizeof(int) * m->nvox, m->stream));
  FUEL_CUDA(m, cudaMalloc(&m->fs->d_counters, sizeof(int) * 8 + sizeof(long long) * 256));
  FUEL_CUDA(m, cudaMemsetAsync(m->fs->d_counters, 0, sizeof(int) * 8 + sizeof(long long) * 256, m->stream));
  return 0;
}

void frontier_state_destroy(FuelMap* m) {
  if (!m->fs) return;
  FrontierState* f = m->fs;
  if (f->stream) {
    cudaStreamSynchronize(f->stream);
    cudaStreamDestroy(f->stream);
  }
  if (f->ev_in) cudaEventDestroy(f->ev_in);
  if (f->ev_out) cudaEventDestroy(f->ev_out);
  if (f->cellidx) cudaFree(f->cellidx);
  if (f->d_counters) cudaFree(f->d_counters);
  f->h_pin.release();
  f->maskE.release(); f->maskS.release(); f->blockcnt.release(); f->blockoff.release();
  f->scan_tot.release(); f->scan_off.release();
  f->cell_addr.release(); f->parent.release(); f->claim.release(); f->csize.release();
  f->seed.release(); f->is_root.release(); f->is_kept.release(); f->root_rank.release();
  f->kept_off.release(); f->cell_cls.release(); f->k_addr.release(); f->k_cl.release();
  f->k_leaf.release(); f->k_cent.release(); f->stat.release(); f->meta.release(); f->res.release();
  f->asm_scr.release(); f->h_res[0].release(); f->h_res[1].release();
  delete f;
  m->fs = nullptr;
}

#define ENSURE(buf, n)                      \
  do {                                      \
    const int _rc = (buf).ensure(m, (n));   \
    if (_rc) return _rc;                    \
  } while (0)

static inline unsigned nblk(int64_t n, int b) { return (unsigned)((n + b - 1) / b); }

// exclusive scan of n ints on the stream; `total` (device) receives the sum
static int scan_ints(FuelMap* m, const int* in, int* out, int n, int* total) {
  FrontierState* f = m->fs;
  cudaStream_t s = m->fs->stream;
  if (n <= 4096) {
    scan_kernel<<<1, 1024, 0, s>>>(in, out, n, total);
    FUEL_LAUNCHES(m, 1);
    return 0;
  }
  const int nchunk = (n + 1023) / 1024;
  ENSURE(f->scan_tot, nchunk);
  ENSURE(f->scan_off, nchunk);
  scan_chunks_kernel<<<nchunk, 1024, 0, s>>>(in, out, n, f->scan_tot.p);
  scan_kernel<<<1, 1024, 0, s>>>(f->scan_tot.p, f->scan_off.p, nchunk, total);
  scan_add_kernel<<<nchunk, 1024, 0, s>>>(out, n, f->scan_off.p);
  FUEL_LAUNCHES(m, 3);
  return 0;
}

static SweepPlan sweep_plan(const Geom& g, const FParams& fp) {
  SweepPlan pl;
  pl.ndom = (int64_t)fp.dom_n[0] * fp.dom_n[1] * fp.dom_n[2];
  pl.words = (g.nz % 32) == 0 && pl.ndom > 0;
  if (pl.words) {
    const int z0 = fp.dom_lo[2], z1 = fp.dom_lo[2] + fp.dom_n[2] - 1;
    pl.wg.wz0 = z0 >> 5;
    pl.wg.NW = (z1 >> 5) - pl.wg.wz0 + 1;
    pl.wg.nwords = (int64_t)fp.dom_n[0] * fp.dom_n[1] * pl.wg.NW;
    pl.nb = nblk(pl.wg.nwords, WORD_BLOCK);
    pl.nmask = (size_t)pl.nb * WORD_BLOCK;
  } else {
    pl.nb = nblk(pl.ndom, CLS_BLOCK);
    pl.nmask = (size_t)pl.nb * (CLS_BLOCK / 32);
  }
  return pl;
}

// classification sweep + scan of the per-CTA counts; d_counters[0] receives the candidate count
static int sweep_classify(FuelMap* m, const FParams& fp, const SweepPlan& pl, cudaStream_t s) {
  FrontierState* f = m->fs;
  ENSURE(f->maskE, pl.nmask);
  ENSURE(f->maskS, pl.nmask);
  ENSURE(f->blockcnt, pl.nb);
  ENSURE(f->blockoff, pl.nb);
  if (pl.words)
    classify_words_kernel<<<pl.nb, WORD_BLOCK, 0, s>>>(m->g, fp, pl.wg, m->occ, m->flag, f->maskE.p, f->maskS.p,
                                                       f->blockcnt.p);
  else
    classify_kernel<<<pl.nb, CLS_BLOCK, 0, s>>>(m->g, fp, m->occ, m->flag, f->maskE.p, f->maskS.p, f->blockcnt.p,
                                                pl.ndom);
  FUEL_LAUNCHES(m, 1);
  if (scan_ints(m, f->blockcnt.p, f->blockoff.p, (int)pl.nb, f->d_counters + 0)) return FUELGPU_ENOMEM;
  return 0;
}

// masks + scanned offsets -> address-ordered cell list (at most `cap` cells are written)
static void sweep_compact(FuelMap* m, const FParams& fp, const SweepPlan& pl, int* cellidx, int cap, cudaStream_t s) {
  FrontierState* f = m->fs;
  if (pl.words)
    compact_words_kernel<<<pl.nb, WORD_BLOCK, 0, s>>>(m->g, fp, pl.wg, f->maskE.p, f->maskS.p, f->blockoff.p,
                                                      f->cell_addr.p, f->cell_cls.p, cellidx, cap);
  else
    compact_kernel<<<pl.nb, CLS_BLOCK, 0, s>>>(m->g, fp, f->maskE.p, f->maskS.p, f->blockoff.p, f->cell_addr.p,
                                               f->cell_cls.p, cellidx, pl.ndom, cap);
  FUEL_LAUNCHES(m, 1);
}

static size_t view_bytes(int K, int C) {
  return (size_t)K * (3 * sizeof(int) + 3 * sizeof(float)) + (size_t)C * (sizeof(ClusterMeta) + sizeof(ClusterStat)) + 64;
}

// byte offsets of the arrays of K cells / C clusters in a result buffer (16-byte aligned pieces)
struct ResultLayout {
  size_t meta, stat, addr, cl, leaf, cent, bytes;
};
static ResultLayout result_layout(int K, int C) {
  ResultLayout l;
  size_t p = 0;
  auto put = [&](size_t bytes) {
    const size_t o = p;
    p += (bytes + 15) & ~(size_t)15;
    return o;
  };
  l.meta = put(sizeof(ClusterMeta) * C);
  l.stat = put(sizeof(ClusterStat) * C);
  l.addr = put(sizeof(int) * K);
  l.cl = put(sizeof(int) * K);
  l.leaf = put(sizeof(int) * K);
  l.cent = put(sizeof(float) * 3 * K);
  l.bytes = p;
  return l;
}
static void result_view(const ResultLayout& l, const char* base, HostView* v) {
  v->meta = (const ClusterMeta*)(base + l.meta);
  v->stat = (const ClusterStat*)(base + l.stat);
  v->addr = (const int*)(base + l.addr);
  v->cl = (const int*)(base + l.cl);
  v->leaf = (const int*)(base + l.leaf);
  v->cent = (const float*)(base + l.cent);
}

// enqueue the D2H of K cells / C clusters into the pinned buffer at `base` (no sync)
static int enqueue_download(FuelMap* m, int K, int C, char* base, HostView* v) {
  FrontierState* f = m->fs;
  cudaStream_t s = m->fs->stream;
  const ResultLayout l = result_layout(K, C);
  result_view(l, base, v);
  auto get = [&](const void* dst, const void* src, size_t bytes) {
    if (bytes) cudaMemcpyAsync((void*)dst, src, bytes, cudaMemcpyDeviceToHost, s);
  };
  get(v->meta, f->meta.p, sizeof(ClusterMeta) * C);
  get(v->stat, f->stat.p, sizeof(ClusterStat) * C);
  get(v->addr, f->k_addr.p, sizeof(int) * K);
  get(v->cl, f->k_cl.p, sizeof(int) * K);
  get(v->leaf, f->k_leaf.p, sizeof(int) * K);
  get(v->cent, f->k_cent.p, sizeof(float) * 3 * K);
  FUEL_CUDA(m, cudaGetLastError());
  return 0;
}

static int frontier_build_csr(FuelMap* m, int K, int C, const HostView& hv, int32_t* n_clusters,
                              int32_t* n_cells, int32_t* n_filtered);

// ---- optional: the reference's own cell order ---------------------------------------------------------------
// expandFrontier (frontier_finder.cpp:123-164) appends cells in BFS order from the seed (the first cell of the
// cluster in scan order = its lowest address), neighbours in allNeighbors order (:848-860: x, y, z from -1 to 1),
// and splitHorizontally (:217-224) partitions a parent's cells_ keeping their relative order.  The device emits a
// cluster's cells in ascending address; membership, cluster order and flags do not depend on the order, but the fp64
// running sum of average_ (:374-385) and the float32 per-leaf sums of the VoxelGrid centroids (:757-774) do, in their
// last bits.  With FUELGPU_CELLS_BFS the host re-derives the BFS rank of every cell of a root cluster (the BFS only
// ever moves between cells of that cluster, so the fetched cell set is all it needs), re-orders the cells of its final
// clusters by it and recomputes average_ and filtered_cells_ in that order: bit-identical with the reference.
static void frontier_apply_bfs_order(FuelMap* m, const std::vector<int>& out_root) {
  FrontierState* f = m->fs;
  const Geom& g = m->g;
  const int C = (int)out_root.size();
  const int64_t sy = g.nz, sx = (int64_t)g.ny * g.nz;
  std::vector<int32_t> new_filt_off(C + 1, 0);
  std::vector<double> new_filtered;
  new_filtered.reserve(f->h_filtered.size());
  std::vector<int> tab;  // open-addressing hash: address -> local index
  for (int r0 = 0; r0 < C;) {
    int r1 = r0 + 1;
    while (r1 < C && out_root[r1] == out_root[r0]) ++r1;
    const int a0 = f->h_cell_off[r0], a1 = f->h_cell_off[r1], n = a1 - a0;
    int cap = 16;
    while (cap < 2 * n) cap <<= 1;
    tab.assign(cap, -1);
    auto slot_of = [&](int addr) { return (int)(((uint32_t)addr * 2654435761u) & (uint32_t)(cap - 1)); };
    // the seed = the first cell of the cluster the scan of the search box meets (:108-116): lowest address inside it
    int seed = -1;
    const FParams& sp = f->pend_fp;
    for (int i = 0; i < n; ++i) {
      const int addr = f->h_cell_addr[a0 + i];
      const int cx = (int)(addr / sx), cy = (int)((addr % sx) / sy), cz = (int)(addr % sy);
      const bool in_search = cx >= sp.s_lo[0] && cx <= sp.s_hi[0] && cy >= sp.s_lo[1] && cy <= sp.s_hi[1] &&
                             cz >= sp.s_lo[2] && cz <= sp.s_hi[2];
      if (in_search && (seed < 0 || addr < f->h_cell_addr[a0 + seed])) seed = i;
      int s = slot_of(addr);
      while (tab[s] >= 0) s = (s + 1) & (cap - 1);
      tab[s] = i;
    }
    auto find = [&](int addr) {
      int s = slot_of(addr);
      while (tab[s] >= 0) {
        if (f->h_cell_addr[a0 + tab[s]] == addr) return tab[s];
        s = (s + 1) & (cap - 1);
      }
      return -1;
    };
    if (seed < 0) seed = 0;  // (cannot happen: every root has its seed inside the search box)
    std::vector<int> bfs_rank(n, -1), queue;
    queue.reserve(n);
    queue.push_back(seed);
    bfs_rank[seed] = 0;
    for (size_t qh = 0; qh < queue.size(); ++qh) {
      const int addr = f->h_cell_addr[a0 + queue[qh]];
      const int x = (int)(addr / sx), y = (int)((addr % sx) / sy), z = (int)(addr % sy);
      for (int dx = -1; dx <= 1; ++dx)
        for (int dy = -1; dy <= 1; ++dy)
          for (int dz = -1; dz <= 1; ++dz) {
            if (!dx && !dy && !dz) continue;
            const int xx = x + dx, yy = y + dy, zz = z + dz;
            if (xx < 0 || yy < 0 || zz < 0 || xx >= g.nx || yy >= g.ny || zz >= g.nz) continue;
            const int j = find((int)(xx * sx + yy * sy + zz));
            if (j >= 0 && bfs_rank[j] < 0) {
              bfs_rank[j] = (int)queue.size();
              queue.push_back(j);
            }
          }
    }
    int next = (int)queue.size();
    for (int i = 0; i < n; ++i)  // (not reachable from the seed: cannot happen for a region-grown cluster)
      if (bfs_rank[i] < 0) bfs_rank[i] = next++;
    for (int r = r0; r < r1; ++r) {
      const int c0 = f->h_cell_off[r] - a0, c1 = f->h_cell_off[r + 1] - a0, cn = c1 - c0;
      std::vector<std::pair<int, int>> key(cn);
      for (int i = 0; i < cn; ++i) key[i] = std::make_pair(bfs_rank[c0 + i], f->h_cell_addr[a0 + c0 + i]);
      std::sort(key.begin(), key.end());
      // computeFrontierInfo in this order: positions = indexToPos (sdf_map.h:133-136), fp64 running sum
      std::vector<float> pf((size_t)3 * cn);
      double sum[3] = { 0, 0, 0 };
      for (int i = 0; i < cn; ++i) {
        const int addr = key[i].second;
        f->h_cell_addr[a0 + c0 + i] = addr;
        const int id[3] = { (int)(addr / sx), (int)((addr % sx) / sy), (int)(addr % sy) };
        for (int a = 0; a < 3; ++a) {
          const double pos = (id[a] + 0.5) * g.res + g.origin[a];
          sum[a] += pos;
          pf[(size_t)3 * i + a] = (float)pos;
        }
      }
      for (int a = 0; a < 3; ++a) f->h_avg[(size_t)3 * r + a] = sum[a] / (double)cn;
      // pcl::VoxelGrid (third party, restated as in DESIGN.md: leaf index from floor(p * inv_leaf) relative to the
      // cloud's minimum, centroids in ascending leaf index, points of a leaf summed in float32 in input order)
      const float inv = 1.0f / f->last_leaf;
      float minp[3] = { pf[0], pf[1], pf[2] }, maxp[3] = { pf[0], pf[1], pf[2] };
      for (int i = 1; i < cn; ++i)
        for (int a = 0; a < 3; ++a) {
          minp[a] = std::min(minp[a], pf[(size_t)3 * i + a]);
          maxp[a] = std::max(maxp[a], pf[(size_t)3 * i + a]);
        }
      int minb[3], divb[3];
      for (int a = 0; a < 3; ++a) {
        minb[a] = (int)floorf(minp[a] * inv);
        divb[a] = (int)floorf(maxp[a] * inv) - minb[a] + 1;
      }
      std::vector<std::pair<int, int>> lk(cn);
      for (int i = 0; i < cn; ++i) {
        int ijk[3];
        for (int a = 0; a < 3; ++a) ijk[a] = (int)(floorf(pf[(size_t)3 * i + a] * inv) - (float)minb[a]);
        lk[i] = std::make_pair(ijk[0] + ijk[1] * divb[0] + ijk[2] * divb[0] * divb[1], i);
      }
      std::sort(lk.begin(), lk.end());
      int nf = 0;
      for (int i = 0; i < cn;) {
        int j = i;
        float acc[3] = { 0.f, 0.f, 0.f };
        while (j < cn && lk[j].first == lk[i].first) {
          for (int a = 0; a < 3; ++a) acc[a] += pf[(size_t)3 * lk[j].second + a];
          ++j;
        }
        const float cntf = (float)(j - i);
        for (int a = 0; a < 3; ++a) new_filtered.push_back((double)(acc[a] / cntf));
        ++nf;
        i = j;
      }
      new_filt_off[r + 1] = new_filt_off[r] + nf;
    }
    r0 = r1;
  }
  f->h_filt_off.swap(new_filt_off);
  f->h_filtered.swap(new_filtered);
}

static int frontier_marshal(FuelMap* m, int K, int C, int32_t* n_clusters, int32_t* n_cells,
                            int32_t* n_filtered) {
  int rc = m->fs->h_pin.ensure(m, view_bytes(K, C));
  if (rc) return rc;
  HostView hv;
  rc = enqueue_download(m, K, C, m->fs->h_pin.p, &hv);
  if (rc) return rc;
  FUEL_CUDA(m, cudaStreamSynchronize(m->fs->stream));
  return frontier_build_csr(m, K, C, hv, n_clusters, n_cells, n_filtered);
}

static int frontier_build_csr(FuelMap* m, int K, int C, const HostView& hv, int32_t* n_clusters,
                              int32_t* n_cells, int32_t* n_filtered) {
  FrontierState* f = m->fs;
  const Geom& g = m->g;
  const int* h_addr = hv.addr;
  const int* h_cl = hv.cl;
  const int* h_leaf = hv.leaf;
  const float* h_cent = hv.cent;
  const ClusterMeta* h_meta = hv.meta;
  const ClusterStat* h_stat = hv.stat;
  // ---- marshal into CSR (ordering only; no geometry is decided here) ------
  // cluster order: (root, path) lexicographic = the reference's in-place list replacement
  std::vector<int> order(C);
  for (int c = 0; c < C; ++c) order[c] = c;
  std::sort(order.begin(), order.end(), [&](int a, int b) {
    if (h_meta[a].root != h_meta[b].root) return h_meta[a].root < h_meta[b].root;
    return h_meta[a].path < h_meta[b].path;
  });
  std::vector<int> rank(C);
  for (int i = 0; i < C; ++i) rank[order[i]] = i;

  f->h_cell_off.assign(C + 1, 0);
  f->h_filt_off.assign(C + 1, 0);
  for (int k = 0; k < K; ++k) {
    f->h_cell_off[rank[h_cl[k]] + 1]++;
    if (h_leaf[k] >= 0) f->h_filt_off[rank[h_cl[k]] + 1]++;
  }
  for (int c = 0; c < C; ++c) {
    f->h_cell_off[c + 1] += f->h_cell_off[c];
    f->h_filt_off[c + 1] += f->h_filt_off[c];
  }
  f->h_cell_addr.resize(K);
  const int NF = f->h_filt_off[C];
  std::vector<std::pair<int, int>> filt_keys(NF);  // (leaf, kept index) per slot
  {
    std::vector<int> cur(f->h_cell_off.begin(), f->h_cell_off.end() - 1);
    std::vector<int> curf(f->h_filt_off.begin(), f->h_filt_off.end() - 1);
    for (int k = 0; k < K; ++k) {  // k ascending = address ascending (stable)
      const int r = rank[h_cl[k]];
      f->h_cell_addr[cur[r]++] = h_addr[k];
      if (h_leaf[k] >= 0) filt_keys[curf[r]++] = std::make_pair(h_leaf[k], k);
    }
  }
  f->h_filtered.resize((size_t)3 * NF);
  for (int c = 0; c < C; ++c) {
    // VoxelGrid emits centroids in ascending leaf index
    std::sort(filt_keys.begin() + f->h_filt_off[c], filt_keys.begin() + f->h_filt_off[c + 1]);
    for (int i = f->h_filt_off[c]; i < f->h_filt_off[c + 1]; ++i) {
      const int k = filt_keys[i].second;
      for (int a = 0; a < 3; ++a) f->h_filtered[(size_t)3 * i + a] = (double)h_cent[(size_t)3 * k + a];
    }
  }
  f->h_avg.resize((size_t)3 * C);
  f->h_bmin.resize((size_t)3 * C);
  f->h_bmax.resize((size_t)3 * C);
  for (int c = 0; c < C; ++c) {
    const int r = rank[c];
    for (int a = 0; a < 3; ++a) {
      f->h_avg[(size_t)3 * r + a] = h_meta[c].mean[a];
      f->h_bmin[(size_t)3 * r + a] = (h_stat[c].lo[a] + 0.5) * g.res + g.origin[a];
      f->h_bmax[(size_t)3 * r + a] = (h_stat[c].hi[a] + 0.5) * g.res + g.origin[a];
    }
  }
  *n_clusters = C;
  *n_cells = K;
  *n_filtered = NF;
  if (f->cell_order == FUELGPU_CELLS_BFS) {
    std::vector<int> out_root(C);
    for (int c = 0; c < C; ++c) out_root[rank[c]] = h_meta[c].root;
    frontier_apply_bfs_order(m, out_root);
    *n_filtered = f->h_filt_off[C];
  }
  return 0;
}

// search box, sweep domain and the per-search constants (frontier_finder.cpp:94-104,152)
static int frontier_cluster_large(FuelMap* m, const FParams& fp, int n_cand, int32_t* n_clusters, int32_t* n_cells,
                                  int32_t* n_filtered);

static void frontier_make_params(FuelMap* m, const double umin[3], const double umax[3], const FuelFrontierParams* p,
                                 FParams* out) {
  FrontierState* f = m->fs;
  const Geom& g = m->g;
  const int nmax[3] = { g.nx, g.ny, g.nz };
  // search box: updated box inflated by (1,1,0.5) m, clamped to the exploration box, then
  // posToIndex (frontier_finder.cpp:94-104)
  FParams fp;
  const double infl[3] = { 1, 1, 0.5 };
  for (int k = 0; k < 3; ++k) {
    double lo = umin[k] - infl[k], hi = umax[k] + infl[k];
    lo = lo > g.box_mind[k] ? lo : g.box_mind[k];
    hi = hi < g.box_maxd[k] ? hi : g.box_maxd[k];
    int ilo = (int)floor((lo - g.origin[k]) * g.res_inv);
    int ihi = (int)floor((hi - g.origin[k]) * g.res_inv);
    // cells outside the map are never knownfree; clip (the reference indexes out of bounds
    // there, SURVEY H9)
    fp.s_lo[k] = ilo < 0 ? 0 : ilo;
    fp.s_hi[k] = ihi > nmax[k] - 1 ? nmax[k] - 1 : ihi;
    // sweep domain: exploration box [box_min, box_max] united with the search box
    int dlo = g.box_min[k] < fp.s_lo[k] ? g.box_min[k] : fp.s_lo[k];
    int dhi = g.box_max[k] > fp.s_hi[k] ? g.box_max[k] : fp.s_hi[k];
    dlo = dlo < 0 ? 0 : dlo;
    dhi = dhi > nmax[k] - 1 ? nmax[k] - 1 : dhi;
    fp.dom_lo[k] = dlo;
    fp.dom_n[k] = dhi - dlo + 1;
    if (fp.dom_n[k] <= 0) {
      fp.dom_n[k] = 0;
    }
  }
  // first z index whose centre is not below min_z: `pos[2] < 0.4 -> continue` (:152)
  {
    int zi = 0;
    while (zi < g.nz && ((zi + 0.5) * g.res + g.origin[2]) < p->min_z) ++zi;
    fp.z_min_idx = zi;
  }
  fp.cluster_min = p->cluster_min;
  fp.size_xy = p->cluster_size_xy;
  fp.leaf = (float)(g.res * p->down_sample);  // setLeafSize(float) narrowing
  f->last_leaf = fp.leaf;
  fp.leaf_inv = 1.0f / fp.leaf;
  f->pend_fp = fp;  // (search box and leaf size are also what the host-side BFS ordering needs)
  *out = fp;
}

// the result of the last collected search becomes empty (fuelgpu_frontier_fetch returns nothing)
static void frontier_clear_results(FrontierState* f) {
  f->h_cell_off.assign(1, 0);
  f->h_cell_addr.clear();
  f->h_filt_off.assign(1, 0);
  f->h_filtered.clear();
  f->h_avg.clear();
  f->h_bmin.clear();
  f->h_bmax.clear();
  f->res_blk = -1;
}

// FUELGPU_FRONTIER_HOST_CSR=1 (read by every search_begin): the small path returns its raw arrays and the host orders
// them (frontier_build_csr), as the large path does -- the reference the device-built result is tested against
static bool frontier_host_csr() {
  const char* e = getenv("FUELGPU_FRONTIER_HOST_CSR");
  return e && *e && strcmp(e, "0") != 0;
}

int frontier_search_begin_impl(FuelMap* m, const double umin[3], const double umax[3],
                               const FuelFrontierParams* p) {
  FrontierState* f = m->fs;
  const Geom& g = m->g;
  cudaStream_t s = m->fs->stream;
  FParams fp;
  frontier_make_params(m, umin, umax, p, &fp);

  // (the result of the last collected search stays readable until the next search_end)
  f->pend_active = false;
  f->pend_empty = true;

  const SweepPlan pl = sweep_plan(g, fp);
  if (pl.ndom <= 0) return 0;
  f->pend_empty = false;
  {
    const int rc = sweep_classify(m, fp, pl, s);
    if (rc) return rc;
  }
  // ---- small path: one compaction + ONE cluster launch, one result copy, one host sync --------------------------
  {
    ENSURE(f->cell_addr, SMALL_CAP); ENSURE(f->cell_cls, SMALL_CAP); ENSURE(f->parent, SMALL_CAP);
    ENSURE(f->claim, SMALL_CAP); ENSURE(f->csize, SMALL_CAP); ENSURE(f->seed, SMALL_CAP);
    ENSURE(f->is_root, SMALL_CAP); ENSURE(f->is_kept, SMALL_CAP); ENSURE(f->root_rank, SMALL_CAP);
    ENSURE(f->kept_off, SMALL_CAP); ENSURE(f->k_addr, SMALL_CAP); ENSURE(f->k_cl, SMALL_CAP);
    ENSURE(f->k_leaf, SMALL_CAP); ENSURE(f->k_cent, (size_t)3 * SMALL_CAP);
    ENSURE(f->meta, SMALL_CCAP); ENSURE(f->stat, SMALL_CCAP);
    ENSURE(f->res, RB_BYTES); ENSURE(f->asm_scr, ASM_SCR);
    // the BFS cell order re-derives the cells' order on the host from the marshalled arrays
    const bool assemble = !frontier_host_csr() && f->cell_order != FUELGPU_CELLS_BFS;
    const int blk = f->res_blk == 0 ? 1 : 0;
    ENSURE(f->h_res[blk], RB_BYTES);  // (a fixed size: allocated once, never replaced)
    sweep_compact(m, fp, pl, f->cellidx, SMALL_CAP, s);
    SmallBufs sb;
    sb.cell_addr = f->cell_addr.p; sb.parent = f->parent.p; sb.claim = f->claim.p; sb.csize = f->csize.p;
    sb.seed = f->seed.p; sb.is_root = f->is_root.p; sb.is_kept = f->is_kept.p; sb.root_rank = f->root_rank.p;
    sb.kept_off = f->kept_off.p; sb.cell_cls = f->cell_cls.p; sb.k_addr = f->k_addr.p; sb.k_cl = f->k_cl.p;
    sb.k_leaf = f->k_leaf.p; sb.k_cent = f->k_cent.p; sb.meta = f->meta.p; sb.stat = f->stat.p;
    sb.counters = f->d_counters;
    sb.res = f->res.p;
    sb.scr = f->asm_scr.p;
    sb.assemble = assemble ? 1 : 0;
    cluster_small_kernel<<<SMALL_CTAS, 1024, 0, s>>>(g, fp, m->flag, f->cellidx, sb);
    FUEL_LAUNCHES(m, 1);
    FUEL_CUDA(m, cudaMemcpyAsync(f->h_res[blk].p, f->res.p, assemble ? RB_BYTES : RB_CELL_OFF, cudaMemcpyDeviceToHost, s));
    f->pend_blk = blk;
    f->pend_fp = fp;
    f->pend_plan = pl;
    f->pend_active = true;
  }
  // classify / union / claim kernels read `occ` on the frontier stream: a later writer of `occ` on the main
  // stream (upload, inflate, fusion) must queue behind them (frontier_order_writer)
  cudaEventRecord(f->ev_out, f->stream);
  f->ev_out_valid = true;
  return 0;
}

int frontier_search_end_impl(FuelMap* m, int32_t* n_clusters, int32_t* n_cells, int32_t* n_filtered) {
  FrontierState* f = m->fs;
  const Geom& g = m->g;
  cudaStream_t s = m->fs->stream;
  *n_clusters = *n_cells = *n_filtered = 0;
  frontier_clear_results(f);
#ifdef FUEL_PROF
  m->end_prof_us[0] = 0.0;
#endif
  if (f->pend_empty || !f->pend_active) {
    f->pend_active = false;
    return 0;
  }
  f->pend_active = false;
  const FParams fp = f->pend_fp;
  const SweepPlan pl = f->pend_plan;
  int n_cand = 0;
  {
    const int* cnt = (const int*)f->h_res[f->pend_blk].p;
#ifdef FUEL_PROF
    const double t0 = prof_now_us();
#endif
    FUEL_CUDA(m, cudaStreamSynchronize(s));
#ifdef FUEL_PROF
    m->end_prof_us[0] = prof_now_us() - t0;
#endif
    n_cand = cnt[0];
    if (n_cand == 0) return 0;
    if (cnt[4] == 0) {
      const int R = cnt[1], K = cnt[2], C = cnt[5];
      if (R == 0 || K == 0) return 0;
      if (cnt[8]) {  // ordered on the device: the block is the result
        *n_clusters = C;
        *n_cells = K;
        *n_filtered = cnt[9];
        f->res_blk = f->pend_blk;
        return 0;
      }
      return frontier_marshal(m, K, C, n_clusters, n_cells, n_filtered);
    }
    // capacity exceeded (status 1: cells, 2: clusters): fall through to the multi-kernel path.
    // Flags written so far are the same ones it will write; cellidx was reset by the kernel
    // (status 2) or never touched beyond the cap (status 1: reset what compaction wrote).
    if (cnt[4] == 1) {
      reset_cellidx_kernel<<<nblk(SMALL_CAP, 256), 256, 0, s>>>(f->cell_addr.p, f->cellidx, SMALL_CAP);
      FUEL_LAUNCHES(m, 1);
    }
  }

  ENSURE(f->cell_addr, n_cand); ENSURE(f->cell_cls, n_cand); ENSURE(f->parent, n_cand);
  ENSURE(f->claim, n_cand); ENSURE(f->csize, n_cand); ENSURE(f->seed, n_cand);
  ENSURE(f->is_root, n_cand); ENSURE(f->is_kept, n_cand); ENSURE(f->root_rank, n_cand);
  ENSURE(f->kept_off, n_cand);

  sweep_compact(m, fp, pl, f->cellidx, n_cand, s);
  return frontier_cluster_large(m, fp, n_cand, n_clusters, n_cells, n_filtered);
}

// the multi-kernel clustering + split over n_cand compacted candidate cells (cell_addr / cell_cls ascending by
// address, cellidx[addr] = index already set): union-find, claims, flags, kept-cell gather, split levels, marshal.
// Nothing here waits for the device until the split levels are enqueued: the root / kept-cell / cluster counts
// stay in device memory (LevelCtl), arrays are sized by their bound n_cand.
static int frontier_cluster_large(FuelMap* m, const FParams& fp, int n_cand, int32_t* n_clusters, int32_t* n_cells,
                                  int32_t* n_filtered) {
  FrontierState* f = m->fs;
  const Geom& g = m->g;
  cudaStream_t s = m->fs->stream;
  ENSURE(f->parent, n_cand);
  ENSURE(f->claim, n_cand); ENSURE(f->csize, n_cand); ENSURE(f->seed, n_cand);
  ENSURE(f->is_root, n_cand); ENSURE(f->is_kept, n_cand); ENSURE(f->root_rank, n_cand);
  ENSURE(f->kept_off, n_cand);
  // kept cells K <= n_cand; every cluster holds at least one kept cell, so the cluster count never exceeds K
  ENSURE(f->k_addr, n_cand); ENSURE(f->k_cl, n_cand); ENSURE(f->k_leaf, n_cand); ENSURE(f->k_cent, (size_t)3 * n_cand);
  ENSURE(f->meta, (size_t)n_cand + 1024);
  ENSURE(f->stat, (size_t)n_cand + 1024);
  const unsigned cb = nblk(n_cand, 256);
  init_parent_kernel<<<cb, 256, 0, s>>>(f->parent.p, f->claim.p, f->csize.p, n_cand);
  union_kernel<<<cb, 256, 0, s>>>(g, f->cell_addr.p, f->cell_cls.p, f->cellidx, f->parent.p, n_cand);
  flatten_kernel<<<cb, 256, 0, s>>>(f->parent.p, f->cell_cls.p, n_cand);
  claim_kernel<<<cb, 256, 0, s>>>(g, fp, f->cell_addr.p, f->cell_cls.p, f->cellidx, f->parent.p, f->claim.p, n_cand);
  assign_kernel<<<cb, 256, 0, s>>>(f->cell_addr.p, f->cell_cls.p, f->parent.p, f->claim.p, f->seed.p,
                                   f->csize.p, m->flag, n_cand);
  mark_kernel<<<cb, 256, 0, s>>>(f->seed.p, f->csize.p, fp.cluster_min, f->is_root.p, f->is_kept.p, n_cand);
  FUEL_LAUNCHES(m, 6);
  if (scan_ints(m, f->is_root.p, f->root_rank.p, n_cand, f->d_counters + 1)) return FUELGPU_ENOMEM;
  if (scan_ints(m, f->is_kept.p, f->kept_off.p, n_cand, f->d_counters + 2)) return FUELGPU_ENOMEM;
  gather_kept_kernel<<<cb, 256, 0, s>>>(f->cell_addr.p, f->seed.p, f->is_kept.p, f->kept_off.p,
                                        f->root_rank.p, f->k_addr.p, f->k_cl.p, f->cellidx, n_cand);
  FUEL_LAUNCHES(m, 1);

  // ---- split levels -------------------------------------------------------------------
  LevelCtl ctl;
  ctl.R = f->d_counters + 1;
  ctl.K = f->d_counters + 2;
  ctl.n_new = f->d_counters + 3;
  ctl.c_final = f->d_counters + 5;
  ctl.ccur = f->d_counters + 6;
  ctl.cnext = f->d_counters + 7;
  // a root cluster has more than cluster_min cells; every level at most doubles the cluster count
  const int64_t r_ub = n_cand / ((fp.cluster_min > 0 ? fp.cluster_min : 0) + 1) + 1;
  init_meta_kernel<<<nblk(r_ub, 256), 256, 0, s>>>(f->meta.p, f->stat.p, ctl);
  FUEL_LAUNCHES(m, 1);
  int cnt[8] = { 0, 0, 0, 0, 0, 0, 0, 0 };
  constexpr int LEVELS_PER_BATCH = 12, MAX_LEVELS = 36;  // (a cluster stops splitting at depth 32: pca_item)
  auto c_bound = [&](int level) -> int64_t {
    const int64_t c = level < 24 ? (r_ub << level) : (int64_t)n_cand;
    return c > n_cand ? (int64_t)n_cand : c;
  };
  for (int level = 0; level < MAX_LEVELS; ++level) {
    const unsigned ccb = nblk(c_bound(level), 256);
    stat_accum_kernel<<<cb, 256, 0, s>>>(g, f->k_addr.p, f->k_cl.p, f->meta.p, f->stat.p, ctl);
    downsample_kernel<<<cb, 256, 0, s>>>(g, fp, f->k_addr.p, f->k_cl.p, f->cellidx, f->meta.p, f->stat.p,
                                         f->k_cent.p, f->k_leaf.p, ctl);
    cov_kernel<<<cb, 256, 0, s>>>(g, f->k_cl.p, f->k_leaf.p, f->k_cent.p, f->meta.p, f->stat.p, ctl);
    pca_kernel<<<ccb, 256, 0, s>>>(g, f->meta.p, f->stat.p, ctl);
    side_count_kernel<<<cb, 256, 0, s>>>(g, f->k_addr.p, f->k_cl.p, f->meta.p, f->stat.p, ctl);
    split_alloc_kernel<<<1, 1024, 0, s>>>(f->meta.p, f->stat.p, ctl);
    relabel_kernel<<<cb, 256, 0, s>>>(g, f->k_addr.p, f->k_cl.p, f->meta.p, ctl);
    next_level_kernel<<<nblk(c_bound(level + 1), 256), 256, 0, s>>>(f->meta.p, f->stat.p, ctl);
    FUEL_LAUNCHES(m, 8);
    int* t = ctl.ccur;
    ctl.ccur = ctl.cnext;
    ctl.cnext = t;
    if ((level + 1) % LEVELS_PER_BATCH == 0 || level + 1 == MAX_LEVELS) {
      FUEL_CUDA(m, cudaMemcpyAsync(cnt, f->d_counters, sizeof(int) * 8, cudaMemcpyDeviceToHost, s));
      FUEL_CUDA(m, cudaStreamSynchronize(s));
      if (cnt[3] == 0) break;
    }
  }
  reset_cellidx_kernel<<<cb, 256, 0, s>>>(f->cell_addr.p, f->cellidx, n_cand);
  FUEL_LAUNCHES(m, 1);
  FUEL_CUDA(m, cudaGetLastError());
  const int R = cnt[1], K = cnt[2], C = cnt[5];
  if (R == 0 || K == 0) return 0;
  return frontier_marshal(m, K, C, n_clusters, n_cells, n_filtered);
}


// ---- sharded sweep (SURVEY 8e row 2) --------------------------------------------------------------------
// The voxel sweep (2 B/voxel, the HBM-bound part) shards on z; the clustering is O(frontier cells) and runs on the
// union of the candidates.  A rank classifies the voxels of ITS z planes [z_lo, z_hi] (it needs the tri-state of
// those planes plus one halo plane on each side) and hands back its candidate cells; the host program gathers the
// lists of all ranks (ascending address), and every rank clusters the full list -- same kernels, same result as the
// single-GPU search, bit for bit.
__global__ void set_cellidx_kernel(const int* __restrict__ cell_addr, int* __restrict__ cellidx, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) cellidx[cell_addr[i]] = i;
}

int frontier_candidates_impl(FuelMap* m, const double umin[3], const double umax[3], const FuelFrontierParams* p, int z_lo,
                             int z_hi, int32_t* n_out) {
  FrontierState* f = m->fs;
  const Geom& g = m->g;
  cudaStream_t s = frontier_stream(m);
  FParams fp;
  frontier_make_params(m, umin, umax, p, &fp);
  *n_out = 0;
  const int dz0 = fp.dom_lo[2] > z_lo ? fp.dom_lo[2] : z_lo;
  const int dz1 = (fp.dom_lo[2] + fp.dom_n[2] - 1) < z_hi ? (fp.dom_lo[2] + fp.dom_n[2] - 1) : z_hi;
  if (dz1 < dz0) return 0;
  fp.dom_lo[2] = dz0;
  fp.dom_n[2] = dz1 - dz0 + 1;
  const SweepPlan pl = sweep_plan(g, fp);
  if (pl.ndom <= 0) return 0;
  {
    const int rc = sweep_classify(m, fp, pl, s);
    if (rc) return rc;
  }
  int n = 0;
  FUEL_CUDA(m, cudaMemcpyAsync(&n, f->d_counters, sizeof(int), cudaMemcpyDeviceToHost, s));
  FUEL_CUDA(m, cudaStreamSynchronize(s));
  if (n > 0) {
    ENSURE(f->cell_addr, n);
    ENSURE(f->cell_cls, n);
    sweep_compact(m, fp, pl, nullptr, n, s);
    FUEL_CUDA(m, cudaGetLastError());
  }
  *n_out = n;
  return 0;
}

int frontier_candidates_fetch_impl(FuelMap* m, int32_t n, int32_t* addr, uint8_t* cls) {
  FrontierState* f = m->fs;
  if (n <= 0) return 0;
  cudaStream_t s = f->stream;
  FUEL_CUDA(m, cudaMemcpyAsync(addr, f->cell_addr.p, sizeof(int) * n, cudaMemcpyDeviceToHost, s));
  FUEL_CUDA(m, cudaMemcpyAsync(cls, f->cell_cls.p, n, cudaMemcpyDeviceToHost, s));
  FUEL_CUDA(m, cudaStreamSynchronize(s));
  return 0;
}

int frontier_search_from_candidates_impl(FuelMap* m, const double umin[3], const double umax[3], const FuelFrontierParams* p,
                                         int32_t n, const int32_t* addr, const uint8_t* cls, int32_t* n_clusters,
                                         int32_t* n_cells, int32_t* n_filtered) {
  FrontierState* f = m->fs;
  cudaStream_t s = frontier_stream(m);
  FParams fp;
  frontier_make_params(m, umin, umax, p, &fp);
  frontier_clear_results(f);
  f->pend_active = false;
  f->pend_empty = true;
  *n_clusters = *n_cells = *n_filtered = 0;
  if (n <= 0) return 0;
  for (int i = 1; i < n; ++i)
    if (addr[i] <= addr[i - 1]) return fuel_fail(m, FUELGPU_EINVAL, "candidate addresses must be strictly ascending");
  if (addr[0] < 0 || (int64_t)addr[n - 1] >= m->nvox) return fuel_fail(m, FUELGPU_EINVAL, "candidate address outside the map");
  ENSURE(f->cell_addr, n);
  ENSURE(f->cell_cls, n);
  FUEL_CUDA(m, cudaMemcpyAsync(f->cell_addr.p, addr, sizeof(int) * n, cudaMemcpyHostToDevice, s));
  FUEL_CUDA(m, cudaMemcpyAsync(f->cell_cls.p, cls, n, cudaMemcpyHostToDevice, s));
  set_cellidx_kernel<<<nblk(n, 256), 256, 0, s>>>(f->cell_addr.p, f->cellidx, n);
  FUEL_LAUNCHES(m, 1);
  FUEL_CUDA(m, cudaMemcpyAsync(f->d_counters, &n, sizeof(int), cudaMemcpyHostToDevice, s));
  const int rc = frontier_cluster_large(m, fp, n, n_clusters, n_cells, n_filtered);
  cudaEventRecord(f->ev_out, f->stream);
  f->ev_out_valid = true;
  return rc;
}

int frontier_search_impl(FuelMap* m, const double umin[3], const double umax[3],
                         const FuelFrontierParams* p, int32_t* n_clusters, int32_t* n_cells,
                         int32_t* n_filtered) {
  int rc = frontier_search_begin_impl(m, umin, umax, p);
  if (rc) return rc;
  return frontier_search_end_impl(m, n_clusters, n_cells, n_filtered);
}

int frontier_fetch_impl(FuelMap* m, int32_t* cell_offsets, int32_t* cell_addr, int32_t* filt_offsets,
                        double* filtered, double* average, double* box_min, double* box_max) {
  FrontierState* f = m->fs;
  if (f->res_blk >= 0) {  // the block the small path's kernel ordered
    const char* rb = f->h_res[f->res_blk].p;
    const int* cnt = (const int*)rb;
    const int K = cnt[2], C = cnt[5], NF = cnt[9];
    const Geom& g = m->g;
    if (cell_offsets) memcpy(cell_offsets, rb + RB_CELL_OFF, sizeof(int32_t) * (C + 1));
    if (cell_addr) memcpy(cell_addr, rb + RB_ADDR, sizeof(int32_t) * K);
    if (filt_offsets) memcpy(filt_offsets, rb + RB_FILT_OFF, sizeof(int32_t) * (C + 1));
    if (filtered) memcpy(filtered, rb + RB_FILT, sizeof(double) * 3 * NF);
    if (average) memcpy(average, rb + RB_AVG, sizeof(double) * 3 * C);
    const int* box = (const int*)(rb + RB_BOX);
    for (int r = 0; r < C; ++r)
      for (int a = 0; a < 3; ++a) {  // (the expression of frontier_build_csr)
        if (box_min) box_min[3 * r + a] = (box[6 * r + a] + 0.5) * g.res + g.origin[a];
        if (box_max) box_max[3 * r + a] = (box[6 * r + 3 + a] + 0.5) * g.res + g.origin[a];
      }
    return 0;
  }
  if (cell_offsets) memcpy(cell_offsets, f->h_cell_off.data(), sizeof(int32_t) * f->h_cell_off.size());
  if (cell_addr) memcpy(cell_addr, f->h_cell_addr.data(), sizeof(int32_t) * f->h_cell_addr.size());
  if (filt_offsets) memcpy(filt_offsets, f->h_filt_off.data(), sizeof(int32_t) * f->h_filt_off.size());
  if (filtered) memcpy(filtered, f->h_filtered.data(), sizeof(double) * f->h_filtered.size());
  if (average) memcpy(average, f->h_avg.data(), sizeof(double) * f->h_avg.size());
  if (box_min) memcpy(box_min, f->h_bmin.data(), sizeof(double) * f->h_bmin.size());
  if (box_max) memcpy(box_max, f->h_bmax.data(), sizeof(double) * f->h_bmax.size());
  return 0;
}

int frontier_is_changed_impl(FuelMap* m, int32_t mcl, const int32_t* offs, const int32_t* addr,
                             uint8_t* changed, int32_t* counts) {
  if (mcl <= 0) return 0;
  const int ncell = offs[mcl];
  const size_t nci = (size_t)(ncell > 0 ? ncell : 1);
  int rc = m->fr_scr.ensure(m, sizeof(int) * ((size_t)2 * mcl + 1 + nci) + mcl + 16);
  if (rc) return rc;
  int* d_off = (int*)m->fr_scr.p;
  int* d_addr = d_off + mcl + 1;
  int* d_cnt = d_addr + nci;
  uint8_t* d_ch = (uint8_t*)(d_cnt + mcl);
  cudaStream_t s = m->fs->stream;
  FUEL_CUDA(m, cudaMemcpyAsync(d_off, offs, sizeof(int) * (mcl + 1), cudaMemcpyHostToDevice, s));
  if (ncell > 0) FUEL_CUDA(m, cudaMemcpyAsync(d_addr, addr, sizeof(int) * ncell, cudaMemcpyHostToDevice, s));
  is_changed_kernel<<<mcl, 128, 0, s>>>(m->g, m->occ, d_off, d_addr, d_ch, d_cnt, mcl);
  FUEL_LAUNCHES(m, 1);
  if (changed) FUEL_CUDA(m, cudaMemcpyAsync(changed, d_ch, mcl, cudaMemcpyDeviceToHost, s));
  if (counts) FUEL_CUDA(m, cudaMemcpyAsync(counts, d_cnt, sizeof(int) * mcl, cudaMemcpyDeviceToHost, s));
  FUEL_CUDA(m, cudaStreamSynchronize(s));
  return 0;
}

#ifdef FUEL_PROF
// debug-only (FUEL_PROF builds): %globaltimer stamps taken after every cluster.sync()
extern "C" __attribute__((visibility("default"))) int fuelgpu_debug_frontier_prof(FuelMap* m, long long* out,
                                                                                  int n) {
  cudaMemcpy(out, (long long*)(m->fs->d_counters + 8), sizeof(long long) * n, cudaMemcpyDeviceToHost);
  return 0;
}
// debug-only: host µs of the last fuelgpu_frontier_search_end, split into the wait for the frontier stream, the
// result assembly and the closing timing event
extern "C" __attribute__((visibility("default"))) int fuelgpu_debug_frontier_end_prof(FuelMap* m, double* out) {
  for (int i = 0; i < 3; ++i) out[i] = m->end_prof_us[i];
  return 0;
}
#endif
