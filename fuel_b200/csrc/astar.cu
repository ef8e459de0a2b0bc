// astar.cu -- the geometric path to the next viewpoint on sm_90a: Astar::search (path_searching/src/astar2.cpp:47-149)
// with backtrack, then FastExplorationManager::shortenPath and planExploreMotion's goal branch
// (exploration_manager/src/fast_exploration_manager.cpp:238-263, 295-325), for a batch of (start, goal) queries.
//
// One warp per search; a persistent grid pulls searches from a counter, so the scratch is sized by the warps that run
// at once, not by B.  Each loop iteration: lane 0 reads the open set's top and pops it; lanes 0..25 take the 26
// neighbours in the reference's loop order and run their map tests, check points and close-set / open-map lookups in
// parallel; lane 0 then applies the state updates (node allocation, g / f, parent, heap push) serially in loop order.
// Built with -fmad=false: every double operation rounds as the reference's does.
#include "common.cuh"
#include "heap.cuh"
#include "raycast.cuh"

#include <math.h>

#include <algorithm>

namespace {

constexpr int AS_WARPS = 4;
constexpr int AS_THREADS = 32 * AS_WARPS;
constexpr int AS_NBR = 26;

struct AsConsts {
  double res, inv_res, lambda, tie;
  int alloc, max_iter, heap_cap, w_max, path_max;
  unsigned tmask;
  // per-warp scratch: byte offsets of each array inside one warp's piece, and the piece size
  size_t off_g, off_f, off_par, off_slot, off_heap, off_path, off_tab, stride;
};

// the open set's ids and the key table entry: (x, y, z) node index, w = 2 * node id + closed, -1 when empty
struct Slot {
  int x, y, z, w;
};

__device__ __forceinline__ double norm3(double x, double y, double z) { return sqrt((x * x + y * y) + z * z); }

// getDiagHeu (astar2.cpp:192-212)
__device__ __forceinline__ double diag_heu(const AsConsts& c, const double a[3], const double b[3]) {
  double dx = fabs(a[0] - b[0]), dy = fabs(a[1] - b[1]), dz = fabs(a[2] - b[2]);
  double h = 0.0;
  const double diag = fmin(fmin(dx, dy), dz);
  dx -= diag;
  dy -= diag;
  dz -= diag;
  const double S3 = 1.7320508075688772, S2 = 1.4142135623730951;  // sqrt(3.0), sqrt(2.0)
  if (dx < 1e-4) h = S3 * diag + S2 * fmin(dy, dz) + fabs(dy - dz);
  if (dy < 1e-4) h = S3 * diag + S2 * fmin(dx, dz) + fabs(dx - dz);
  if (dz < 1e-4) h = S3 * diag + S2 * fmin(dx, dy) + fabs(dx - dy);
  return c.tie * h;
}

// Astar::posToIndex (:232-234) on the map's origin
__device__ __forceinline__ void node_index(const Geom& g, const AsConsts& c, const double p[3], int id[3]) {
#pragma unroll
  for (int k = 0; k < 3; ++k) id[k] = (int)floor((p[k] - g.origin[k]) * c.inv_res);
}

// getInflateOccupancy(pos) == 1 || getOccupancy(pos) == UNKNOWN; outside the map both read -1
__device__ __forceinline__ bool blocked(const Geom& g, const uint8_t* __restrict__ occ, const double p[3]) {
  int id[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) id[k] = (int)floor((p[k] - g.origin[k]) * g.res_inv);
  if (!idx_in_map(g, id[0], id[1], id[2])) return false;
  const uint8_t o = occ[addr_of(g, id[0], id[1], id[2])];
  return (o & 4) || (o & 3) == FUELGPU_UNKNOWN;
}

__device__ __forceinline__ unsigned key_hash(int x, int y, int z) {
  unsigned h = (unsigned)x * 73856093u ^ (unsigned)y * 19349663u ^ (unsigned)z * 83492791u;
  h ^= h >> 15;
  h *= 0x2c1b3c6du;
  h ^= h >> 12;
  return h;
}

// open_set_map_ / close_set_map_ find: -1 absent, else 2 * node id + closed
__device__ int table_find(const Slot* tab, unsigned mask, const int id[3]) {
  unsigned s = key_hash(id[0], id[1], id[2]) & mask;
  for (;;) {
    const Slot e = tab[s];
    if (e.w < 0) return -1;
    if (e.x == id[0] && e.y == id[1] && e.z == id[2]) return e.w;
    s = (s + 1) & mask;
  }
}
__device__ int table_insert(Slot* tab, unsigned mask, const int id[3], int w) {
  unsigned s = key_hash(id[0], id[1], id[2]) & mask;
  while (tab[s].w >= 0) s = (s + 1) & mask;
  tab[s] = Slot{ id[0], id[1], id[2], w };
  return (int)s;
}

struct NbrShared {  // one warp's 26 neighbour results, written in parallel and consumed by lane 0 in loop order
  double pos[AS_NBR][3];
  double g[AS_NBR], h[AS_NBR];
  int idx[AS_NBR][3];
  int found[AS_NBR];  // node id from the open map, -1 absent
  int node[AS_NBR];   // lane 0: the node this neighbour ended up on (-1 none)
  int cur;
  FuelPathInfo inf;  // lane 0: the result of the current search
};

// kRaw: the search of ViewNode::searchPath (active_perception/src/graph_node.cpp:48-57) over the pairs whose straight
// line is blocked.  The queries are list[0 .. *n_list) of the pair arrays, a count the line test leaves on the device,
// and each writes getPath() with its Astar::pathLength (astar2.cpp:169-175) into info.length: no shortenPath, branch
// or tour.
template <bool kRaw>
__global__ void __launch_bounds__(AS_THREADS)
astar_kernel(Geom g, const uint8_t* __restrict__ occ, AsConsts c, int B, const double* __restrict__ start,
             const double* __restrict__ goal, uint8_t* __restrict__ scratch, int* __restrict__ counter,
             FuelPathInfo* __restrict__ info_out, double* __restrict__ path_out, int32_t* __restrict__ nwp_out,
             double* __restrict__ wp_out, const int* __restrict__ n_list, const int* __restrict__ list) {
  __shared__ NbrShared sh_all[AS_WARPS];
  const int lane = threadIdx.x & 31, wl = threadIdx.x >> 5;
  NbrShared& sh = sh_all[wl];
  uint8_t* base = scratch + (size_t)(blockIdx.x * AS_WARPS + wl) * c.stride;
  double* pos = (double*)base;
  double* gs = (double*)(base + c.off_g);
  double* fs = (double*)(base + c.off_f);
  int* par = (int*)(base + c.off_par);
  int* slot = (int*)(base + c.off_slot);
  int* heap = (int*)(base + c.off_heap);
  double* ps = (double*)(base + c.off_path);
  Slot* tab = (Slot*)(base + c.off_tab);

  // neighbour k of the loop dx, dy, dz (each -res, -res + res, -res + res + res), the centre skipped
  const int kk = lane < 13 ? lane : lane + 1;
  const int sgn[3] = { kk / 9, (kk / 3) % 3, kk % 3 };
  double step[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    double d = -c.res;
    for (int i = 0; i < sgn[a]; ++i) d += c.res;
    step[a] = d;
  }
  const double step_norm = norm3(step[0], step[1], step[2]);

  for (;;) {
    int b = 0;
    if (lane == 0) b = atomicAdd(counter, 1);
    b = __shfl_sync(0xffffffffu, b, 0);
    if (b >= (kRaw ? *n_list : B)) return;
    if (kRaw) b = list[b];
    const double sp[3] = { start[3 * b], start[3 * b + 1], start[3 * b + 2] };
    const double ep[3] = { goal[3 * b], goal[3 * b + 1], goal[3 * b + 2] };
    FuelPathInfo& inf = sh.inf;
    if (lane == 0) {
      memset(&inf, 0, sizeof(inf));
      inf.status = FUELGPU_ASTAR_NO_PATH;
    }
    bool finite = true;
#pragma unroll
    for (int k = 0; k < 3; ++k) finite = finite && isfinite(sp[k]) && isfinite(ep[k]);
    int end_node = -1, use = 0, n_ins = 0;
    if (!finite) {
      if (lane == 0) inf.reason = FUELGPU_ASTAR_BAD_INPUT;
    } else {
      int end_idx[3];
      node_index(g, c, ep, end_idx);
      int heap_len = 0, iter = 0, loops = 0;
      if (lane == 0) {
        pos[0] = sp[0], pos[1] = sp[1], pos[2] = sp[2];
        par[0] = -1;
        gs[0] = 0.0;
        fs[0] = c.lambda * diag_heu(c, sp, ep);
        heap[0] = 0;
        int id[3];
        node_index(g, c, sp, id);
        slot[0] = table_insert(tab, c.tmask, id, 0);
      }
      heap_len = 1, use = 1, n_ins = 1;
      if (lane == 0) inf.reason = FUELGPU_ASTAR_OPEN_EMPTY;
      __syncwarp();
      for (;;) {
        // lane 0: goal test on top(), the iteration cap, pop, close.  action 0 = expand, 1 = stop
        int action = 0, cur = 0;
        if (lane == 0) {
          if (heap_len == 0) {
            action = 1;
          } else {
            cur = heap[0];
            const double cp[3] = { pos[3 * cur], pos[3 * cur + 1], pos[3 * cur + 2] };
            int ci[3];
            node_index(g, c, cp, ci);
            if (abs(ci[0] - end_idx[0]) <= 1 && abs(ci[1] - end_idx[1]) <= 1 && abs(ci[2] - end_idx[2]) <= 1) {
              inf.status = FUELGPU_ASTAR_REACH_END;
              inf.reason = FUELGPU_ASTAR_FOUND;
              end_node = cur;
              action = 1;
            } else if (++loops > c.max_iter) {
              inf.reason = FUELGPU_ASTAR_ITER_CAP;
              inf.early_terminate_cost = gs[cur] + diag_heu(c, cp, ep);
              action = 1;
            } else {
              heap_pop(heap, heap_len, fs);
              --heap_len;
              tab[slot[cur]].w = 2 * cur + 1;
              ++iter;
              sh.cur = cur;
            }
          }
        }
        action = __shfl_sync(0xffffffffu, action, 0);
        if (action) break;
        __syncwarp();
        cur = sh.cur;
        const double cp[3] = { pos[3 * cur], pos[3 * cur + 1], pos[3 * cur + 2] };
        const double cg = gs[cur];
        bool ok = false;
        if (lane < AS_NBR) {
          double np[3] = { cp[0] + step[0], cp[1] + step[1], cp[2] + step[2] };
          ok = step_norm >= 1e-3;
          for (int k = 0; k < 3; ++k)
            if (np[k] <= g.box_mind[k] || np[k] >= g.box_maxd[k]) ok = false;
          if (ok && blocked(g, occ, np)) ok = false;
          if (ok) {  // the check points l = 0.1, 0.2, ... < |step| along the normalized step
            double dir[3] = { np[0] - cp[0], np[1] - cp[1], np[2] - cp[2] };
            const double len = norm3(dir[0], dir[1], dir[2]);
            const double z = (dir[0] * dir[0] + dir[1] * dir[1]) + dir[2] * dir[2];
            if (z > 0.0) {
              const double n = sqrt(z);
              dir[0] = dir[0] / n, dir[1] = dir[1] / n, dir[2] = dir[2] / n;
            }
            for (double l = 0.1; l < len; l += 0.1) {
              const double ck[3] = { cp[0] + l * dir[0], cp[1] + l * dir[1], cp[2] + l * dir[2] };
              if (blocked(g, occ, ck)) {
                ok = false;
                break;
              }
            }
          }
          int id[3];
          node_index(g, c, np, id);
          int found = -1;
          if (ok) {
            const int w = table_find(tab, c.tmask, id);
            if (w >= 0 && (w & 1)) ok = false;  // close set
            found = w >= 0 ? (w >> 1) : -1;
          }
          sh.pos[lane][0] = np[0], sh.pos[lane][1] = np[1], sh.pos[lane][2] = np[2];
          sh.idx[lane][0] = id[0], sh.idx[lane][1] = id[1], sh.idx[lane][2] = id[2];
          sh.found[lane] = found;
          sh.g[lane] = step_norm + cg;
          sh.h[lane] = ok ? diag_heu(c, np, ep) : 0.0;
        }
        const unsigned okm = __ballot_sync(0xffffffffu, ok);
        __syncwarp();
        if (lane == 0) {
          unsigned rest = okm;
          while (rest) {
            const int k = __ffs(rest) - 1;
            rest &= rest - 1;
            int node = sh.found[k];
            if (node < 0)  // an earlier neighbour of this iteration with the same index (floor rounding) made it
              for (int j = 0; j < k; ++j)
                if (((okm >> j) & 1) && sh.node[j] >= 0 && sh.idx[j][0] == sh.idx[k][0] && sh.idx[j][1] == sh.idx[k][1] &&
                    sh.idx[j][2] == sh.idx[k][2])
                  node = sh.node[j];
            const double tg = sh.g[k];
            int nb;
            bool fresh = false;
            if (node < 0) {
              nb = use++;
              if (use == c.alloc) {
                inf.reason = FUELGPU_ASTAR_POOL;
                sh.node[k] = -1;
                action = 1;
                break;
              }
              pos[3 * nb] = sh.pos[k][0], pos[3 * nb + 1] = sh.pos[k][1], pos[3 * nb + 2] = sh.pos[k][2];
              fresh = true;
            } else if (tg < gs[node]) {
              nb = node;
            } else {
              sh.node[k] = node;
              continue;
            }
            sh.node[k] = nb;
            par[nb] = cur;
            gs[nb] = tg;
            fs[nb] = tg + c.lambda * sh.h[k];
            if (heap_len == c.heap_cap) {
              inf.reason = FUELGPU_ASTAR_HEAP_FULL;
              action = 1;
              break;
            }
            heap_sift_up(heap, fs, heap_len++, nb);
            if (fresh) {
              slot[nb] = table_insert(tab, c.tmask, sh.idx[k], 2 * nb);
              ++n_ins;
            }
          }
        }
        action = __shfl_sync(0xffffffffu, action, 0);
        __syncwarp();
        if (action) break;
      }
      if (lane == 0) inf.iter_num = iter;
    }
    if (lane == 0) inf.use_node_num = use;
    n_ins = __shfl_sync(0xffffffffu, n_ins, 0);
    end_node = __shfl_sync(0xffffffffu, end_node, 0);

    // getPath(): start ... end node, goal (backtrack, :177-186); then shortenPath and the branch on lane 0
    int n_path = 0, nt = 0;
    if (lane == 0 && end_node >= 0) {
      int cnt = 0;
      for (int n = end_node; n >= 0; n = par[n]) ++cnt;
      n_path = cnt + 1;
      ps[3 * cnt] = ep[0], ps[3 * cnt + 1] = ep[1], ps[3 * cnt + 2] = ep[2];
      int i = cnt - 1;
      for (int n = end_node; n >= 0; n = par[n], --i)
        ps[3 * i] = pos[3 * n], ps[3 * i + 1] = pos[3 * n + 1], ps[3 * i + 2] = pos[3 * n + 2];
      inf.n_path = n_path;
    }
    n_path = __shfl_sync(0xffffffffu, n_path, 0);
    __syncwarp();
    if (path_out) {  // getPath(), its first path_max rows
      const int ncopy = min(n_path, c.path_max);
      double* dst = path_out + (size_t)b * c.path_max * 3;
      for (int i = lane; i < c.path_max * 3; i += 32) dst[i] = i < 3 * ncopy ? ps[i] : 0.0;
    }
    __syncwarp();
    if (kRaw) {
      if (lane == 0) {
        if (end_node >= 0) {
          double len = 0.0;  // Astar::pathLength(getPath())
          for (int k = 0; k + 1 < n_path; ++k)
            len += norm3(ps[3 * k + 3] - ps[3 * k], ps[3 * k + 4] - ps[3 * k + 1], ps[3 * k + 5] - ps[3 * k + 2]);
          inf.length = len;
        }
        info_out[b] = inf;
      }
      for (int i = lane; i < n_ins; i += 32) tab[slot[i]].w = -1;
      __syncwarp();
      continue;
    }
    if (lane == 0 && end_node >= 0) {
      // shortenPath (:295-325), in place: the short tour never outgrows the path read so far
      const double last[3] = { ps[3 * (n_path - 1)], ps[3 * (n_path - 1) + 1], ps[3 * (n_path - 1) + 2] };
      int m = 1;
      for (int k = 1; k < n_path - 1; ++k) {
        const double* q = ps + 3 * k;
        const double* t = ps + 3 * (m - 1);
        bool keep;
        if (norm3(q[0] - t[0], q[1] - t[1], q[2] - t[2]) > 3.0)
          keep = true;
        else
          keep = !ray_is_clear(g, occ, t, ps + 3 * (k + 1));
        if (keep) {
          const double v[3] = { q[0], q[1], q[2] };
          ps[3 * m] = v[0], ps[3 * m + 1] = v[1], ps[3 * m + 2] = v[2];
          ++m;
        }
      }
      {
        const double* t = ps + 3 * (m - 1);
        if (norm3(last[0] - t[0], last[1] - t[1], last[2] - t[2]) > 1e-3) {
          ps[3 * m] = last[0], ps[3 * m + 1] = last[1], ps[3 * m + 2] = last[2];
          ++m;
        }
      }
      if (m == 2) {  // at least three points
        for (int a = 0; a < 3; ++a) {
          const double p0 = ps[a], p1 = ps[3 + a];
          ps[6 + a] = p1;
          ps[3 + a] = 0.5 * (p0 + p1);
        }
        m = 3;
      }
      double len = 0.0;  // Astar::pathLength
      if (m >= 2)
        for (int k = 0; k + 1 < m; ++k)
          len += norm3(ps[3 * k + 3] - ps[3 * k], ps[3 * k + 4] - ps[3 * k + 1], ps[3 * k + 5] - ps[3 * k + 2]);
      inf.length = len;
      nt = m;
      if (len < 1.5) {
        inf.branch = FUELGPU_ASTAR_CLOSE;
      } else if (len > 5.0) {
        inf.branch = FUELGPU_ASTAR_FAR;
        double len2 = 0.0;
        int t = 1;
        for (int k = 1; k < m && len2 < 5.0; ++k) {
          len2 += norm3(ps[3 * k] - ps[3 * t - 3], ps[3 * k + 1] - ps[3 * t - 2], ps[3 * k + 2] - ps[3 * t - 1]);
          ++t;
        }
        nt = t;
      } else {
        inf.branch = FUELGPU_ASTAR_MID;
      }
      if (inf.branch == FUELGPU_ASTAR_FAR) {
        inf.next_goal[0] = ps[3 * nt - 3], inf.next_goal[1] = ps[3 * nt - 2], inf.next_goal[2] = ps[3 * nt - 1];
      } else {
        inf.next_goal[0] = ep[0], inf.next_goal[1] = ep[1], inf.next_goal[2] = ep[2];
      }
      inf.n_wp = nt;
      inf.tour_status = nt < 3 ? FUELGPU_ASTAR_DEGENERATE
                               : ((nt > FUELGPU_MAX_WAYPTS || nt > c.w_max) ? FUELGPU_ASTAR_TOO_LONG : 0);
    }
    if (lane == 0) {
      info_out[b] = inf;
      nwp_out[b] = (end_node >= 0 && inf.tour_status == 0) ? nt : 0;
    }
    nt = __shfl_sync(0xffffffffu, nt, 0);
    __syncwarp();
    const int ncopy = min(nt, c.w_max);
    for (int i = lane; i < c.w_max * 3; i += 32) wp_out[(size_t)b * c.w_max * 3 + i] = i < 3 * ncopy ? ps[i] : 0.0;
    // clear the table slots this search touched
    for (int i = lane; i < n_ins; i += 32) tab[slot[i]].w = -1;
    __syncwarp();
  }
}

}  // namespace

// Scratch of one warp, in 256-byte pieces: positions 24 A, g and f 8 A each, parent and table slot 4 A each, the open
// set 4 * 2A, the path 24 (A + 1), the key table 16 T (T the least power of two >= 2A, at least 64).
static void astar_layout(int A, AsConsts* c) {
  auto al = [](size_t b) { return (b + 255) & ~(size_t)255; };
  size_t T = 64;
  while (T < 2 * (size_t)A) T <<= 1;
  c->tmask = (unsigned)(T - 1);
  c->heap_cap = 2 * A;
  size_t o = al(24 * (size_t)A);
  c->off_g = o, o += al(8 * (size_t)A);
  c->off_f = o, o += al(8 * (size_t)A);
  c->off_par = o, o += al(4 * (size_t)A);
  c->off_slot = o, o += al(4 * (size_t)A);
  c->off_heap = o, o += al(4 * (size_t)c->heap_cap);
  c->off_path = o, o += al(24 * ((size_t)A + 1));
  c->off_tab = o, o += al(16 * T);
  c->stride = o;
}

constexpr size_t AS_BUDGET = (size_t)4 << 30;  // bytes of search scratch the warps running at once may use

// One launch of astar_kernel<raw> over a pool of `alloc` nodes per search.
static int astar_launch(FuelMap* m, bool raw, int B, const int* n_list, const int* list, const double* start_dev,
                        const double* goal_dev, const FuelAstarParams* p, int alloc, FuelPathInfo* info_dev, int path_max,
                        double* path_dev, int w_max, int32_t* nwp_dev, double* wp_dev) {
  if (B == 0) return 0;
  AsConsts c;
  memset(&c, 0, sizeof(c));
  c.res = p->resolution;
  c.inv_res = 1.0 / p->resolution;  // Astar::setResolution / init (:28, :44)
  c.lambda = p->lambda_heu;
  c.tie = 1.0 + 1.0 / 1000;  // tie_breaker_ (:23)
  c.alloc = alloc;
  c.max_iter = p->max_iter;
  c.w_max = w_max;
  c.path_max = path_dev ? path_max : 0;
  astar_layout(alloc, &c);
  size_t W = (size_t)B;
  W = std::min(W, (size_t)m->sm_count * 32);
  W = std::min(W, std::max((size_t)1, AS_BUDGET / c.stride));
  const size_t blocks = (W + AS_WARPS - 1) / AS_WARPS, warps = blocks * AS_WARPS;
  bool fresh = false;
  const int rc = m->as_buf.ensure(m, 256 + warps * c.stride, &fresh);
  if (rc) return rc;
  uint8_t* scr = m->as_buf.p + 256;
  // every key table starts empty (all bits set); a search clears the slots it used before it ends, so only a new
  // block, a new layout or warps not used before need the fill
  if (fresh || m->as_stride != c.stride) {
    FUEL_CUDA(m, cudaMemsetAsync(scr, 0xff, warps * c.stride, m->stream));
    m->as_stride = c.stride;
    m->as_warps = warps;
  } else if (warps > m->as_warps) {
    FUEL_CUDA(m, cudaMemsetAsync(scr + m->as_warps * c.stride, 0xff, (warps - m->as_warps) * c.stride, m->stream));
    m->as_warps = warps;
  }
  int* counter = (int*)m->as_buf.p;
  FUEL_CUDA(m, cudaMemsetAsync(counter, 0, sizeof(int), m->stream));
  if (raw)
    astar_kernel<true><<<(unsigned)blocks, AS_THREADS, 0, m->stream>>>(m->g, m->occ, c, B, start_dev, goal_dev, scr,
                                                                       counter, info_dev, path_dev, nullptr, nullptr,
                                                                       n_list, list);
  else
    astar_kernel<false><<<(unsigned)blocks, AS_THREADS, 0, m->stream>>>(m->g, m->occ, c, B, start_dev, goal_dev, scr,
                                                                        counter, info_dev, path_dev, nwp_dev, wp_dev,
                                                                        nullptr, nullptr);
  FUEL_LAUNCHES(m, 1);
  FUEL_CUDA(m, cudaGetLastError());
  return 0;
}

int astar_impl(FuelMap* m, int B, const double* start_dev, const double* goal_dev, const FuelAstarParams* p,
               FuelPathInfo* info_dev, int path_max, double* path_dev, int w_max, int32_t* nwp_dev, double* wp_dev) {
  return astar_launch(m, false, B, nullptr, nullptr, start_dev, goal_dev, p, p->allocate_num, info_dev, path_max,
                      path_dev, w_max, nwp_dev, wp_dev);
}

int astar_raw_impl(FuelMap* m, int P, const int* n_list_dev, const int* list_dev, const double* p1_dev,
                   const double* p2_dev, const FuelAstarParams* p, FuelPathInfo* info_dev, int path_max,
                   double* path_dev) {
  // A search expands at most max_iter nodes and each expansion allocates and pushes at most 26, so it never holds more
  // than 1 + 26 * max_iter nodes or open-set entries: a pool of min(allocate_num, 26 * max_iter + 2) ends every search
  // where allocate_num does, and keeps the per-warp scratch small at the reference's allocate_num of 1 000 000.
  const int alloc = (int)std::min<long long>(p->allocate_num, 26LL * p->max_iter + 2);
  return astar_launch(m, true, P, n_list_dev, list_dev, p1_dev, p2_dev, p, alloc, info_dev, path_max, path_dev, 0,
                      nullptr, nullptr);
}
