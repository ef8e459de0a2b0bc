// kino_astar.cu -- the mid-range goal's path on sm_90a: FastPlannerManager::kinodynamicReplan's search
// (plan_manage/src/planner_manager.cpp:131-164): the close-goal refusal, KinodynamicAstar::reset / search(start, vel,
// acc, goal, 0, init) with the retry at init = false (path_searching/src/kinodynamic_astar.cpp:15-263, 484-501),
// computeShotTraj (:331-394) and getSamples (:543-634) at ts = ctrl_pt_dist / max_vel, for a batch of queries.
//
// One warp per search; a persistent grid pulls searches from a counter, so the scratch is sized by the warps that run
// at once, not by B.  Each expansion: lane 0 reads the open set's top, tests the horizon and the goal tolerance and
// pops it; the lanes take the expansion's candidates (125 inputs x 1 duration, or 1 x 20 in the init expansion) in the
// reference's (i, j) order and compute each one's state, box, close-set, velocity, same-voxel and safety tests and its g
// and f in parallel; lane 0 then replays, in that order, everything that touches the pool, the key table and the open
// set: the prune against the nodes this expansion made, allocation, push, insert and the open-node update.  The close
// set cannot change inside an expansion, so the parallel tests read what the serial loop would.
// The open set is libstdc++'s heap over node ids compared through each node's current f (heap.cuh): the reference
// assigns f_score to nodes inside the heap (:198-205, :241-250) and never re-heaps.
// The powers of the search come from host tables (0.5 * pow(tau, 2) with the host's pow, in the reference's loops);
// the heuristic's cbrt and the three-root branch go through kino_math.cuh.  Built with -fmad=false.
#include "common.cuh"
#include "heap.cuh"
#include "kino_math.cuh"

#include <math.h>

#include <algorithm>
#include <vector>

namespace {

constexpr int KS_WARPS = 4;
constexpr int KS_THREADS = 32 * KS_WARPS;
constexpr int KS_MAX_ACC = 8, KS_MAX_INIT = 32, KS_MAX_CHECK = 16;
constexpr int KS_MAX_CAND = KS_MAX_ACC * KS_MAX_ACC * KS_MAX_ACC;
constexpr int KS_K = FUELGPU_MAX_PTS - 2;
enum { KS_REACH_HORIZON = 1, KS_REACH_END = 2, KS_NO_PATH = 3, KS_NEAR_END = 4 };

struct KinoConsts {
  double max_vel, w_time, horizon, lambda, inv_res, ts0;
  double size[3];
  int alloc, check_num, optimistic, tol, n_acc, n_init, node_max;
  unsigned tmask;
  double acc[KS_MAX_ACC];
  // the init durations and the one other duration: `for (tau = max_tau; tau <= max_tau; tau += max_tau)` (:120) runs once
  double tau_init[KS_MAX_INIT], tau_norm;
  // 0.5 * pow(t, 2): [0] t = tau, [k] t = tau * k / check_num
  double h_init[KS_MAX_INIT][KS_MAX_CHECK + 1], h_norm[KS_MAX_CHECK + 1];
  size_t off_in, off_dur, off_g, off_f, off_par, off_idx, off_closed, off_heap, off_slot, off_tab, off_cs, off_cgf,
      off_cidx, off_cint, off_pts, stride;
};

struct Slot {
  int x, y, z, w;  // w = node id, -1 empty
};

__device__ __forceinline__ double dot3(const double* a, const double* b) { return (a[0] * b[0] + a[1] * b[1]) + a[2] * b[2]; }

// stateTransit (:657-668): phi_ * state0 over its six columns in order, plus (0.5 * pow(tau, 2)) * um and tau * um
__device__ void transit(const double* x0, double* x1, const double* um, double tau, double half_t2) {
#pragma unroll
  for (int i = 0; i < 6; ++i) {
    double s = 0.0;
#pragma unroll
    for (int j = 0; j < 6; ++j) {
      const double phi = i == j ? 1.0 : (i < 3 && j == i + 3 ? tau : 0.0);
      s = j == 0 ? phi * x0[0] : s + phi * x0[j];
    }
    x1[i] = s + (i < 3 ? half_t2 * um[i] : tau * um[i - 3]);
  }
}

// cubic(a, b, c, d).front() (:396-423)
__device__ double cubic_front(double a, double b, double c, double d) {
  const double a2 = b / a, a1 = c / a, a0 = d / a;
  const double Q = (3 * a1 - a2 * a2) / 9;
  const double R = (9 * a1 * a2 - 27 * a0 - 2 * a2 * a2 * a2) / 54;
  const double D = Q * Q * Q + R * R;
  if (D > 0) {
    const double S = km_cbrt(R + sqrt(D));
    const double T = km_cbrt(R - sqrt(D));
    return -a2 / 3 + (S + T);
  } else if (D == 0) {
    const double S = km_cbrt(R);
    return -a2 / 3 + S + S;
  }
  const double theta = km_acos_cr(R / sqrt(-Q * Q * Q));
  return 2 * sqrt(-Q) * km_cos_cr(theta / 3) - a2 / 3;
}

// estimateHeuristic (:296-329) with quartic (:425-458)
__device__ double heuristic(const KinoConsts& c, const double* x1, const double* x2, double* optimal_time) {
  const double dp[3] = { x2[0] - x1[0], x2[1] - x1[1], x2[2] - x1[2] };
  const double* v0 = x1 + 3;
  const double* v1 = x2 + 3;
  const double vs[3] = { v0[0] + v1[0], v0[1] + v1[1], v0[2] + v1[2] };
  const double c1 = -36 * dot3(dp, dp);
  const double c2 = 24 * dot3(vs, dp);
  const double c3 = -4 * (dot3(v0, v0) + dot3(v0, v1) + dot3(v1, v1));
  const double c4 = 0;
  double ts[5];
  int n = 0;
  {
    const double a = c.w_time, a3 = c4 / a, a2 = c3 / a, a1 = c2 / a, a0 = c1 / a;
    const double y1 = cubic_front(1, -a2, a1 * a3 - 4 * a0, 4 * a2 * a0 - a1 * a1 - a3 * a3 * a0);
    const double r = a3 * a3 / 4 - a2 + y1;
    if (!(r < 0)) {
      const double R = sqrt(r);
      double D, E;
      if (R != 0) {
        D = sqrt(0.75 * a3 * a3 - R * R - 2 * a2 + 0.25 * (4 * a3 * a2 - 8 * a1 - a3 * a3 * a3) / R);
        E = sqrt(0.75 * a3 * a3 - R * R - 2 * a2 - 0.25 * (4 * a3 * a2 - 8 * a1 - a3 * a3 * a3) / R);
      } else {
        D = sqrt(0.75 * a3 * a3 - 2 * a2 + 2 * sqrt(y1 * y1 - 4 * a0));
        E = sqrt(0.75 * a3 * a3 - 2 * a2 - 2 * sqrt(y1 * y1 - 4 * a0));
      }
      if (!isnan(D)) {
        ts[n++] = -a3 / 4 + R / 2 + D / 2;
        ts[n++] = -a3 / 4 + R / 2 - D / 2;
      }
      if (!isnan(E)) {
        ts[n++] = -a3 / 4 - R / 2 + E / 2;
        ts[n++] = -a3 / 4 - R / 2 - E / 2;
      }
    }
  }
  const double v_max = c.max_vel * 0.5;
  double inf = 0.0;
  for (int i = 0; i < 3; ++i) inf = fmax(inf, fabs(x1[i] - x2[i]));
  const double t_bar = inf / v_max;
  ts[n++] = t_bar;
  double cost = 100000000, t_d = t_bar;
  for (int i = 0; i < n; ++i) {
    const double t = ts[i];
    if (t < t_bar) continue;
    const double cc = -c1 / (3 * t * t * t) - c2 / (2 * t * t) - c3 / t + c.w_time * t;
    if (cc < cost) cost = cc, t_d = t;
  }
  *optimal_time = t_d;
  return 1.0 * (1 + (1.0 + 1.0 / 10000)) * cost;
}

__device__ __forceinline__ bool in_box(const Geom& g, const double* p) {
  for (int i = 0; i < 3; ++i)
    if (p[i] <= g.box_mind[i] || p[i] >= g.box_maxd[i]) return false;
  return true;
}
// the map's voxel of p (SDFMap::posToIndex); false outside the map
__device__ __forceinline__ bool map_voxel(const Geom& g, const double* p, int64_t* a) {
  int id[3];
  for (int k = 0; k < 3; ++k) id[k] = (int)floor((p[k] - g.origin[k]) * g.res_inv);
  if (id[0] < 0 || id[1] < 0 || id[2] < 0 || id[0] > g.nx - 1 || id[1] > g.ny - 1 || id[2] > g.nz - 1) return false;
  *a = addr_of(g, id[0], id[1], id[2]);
  return true;
}
// the safety test of one sample (:172-180)
__device__ __forceinline__ bool unsafe(const Geom& g, const uint8_t* __restrict__ occ, const KinoConsts& c, const double* p) {
  int64_t a;
  const bool in = map_voxel(g, p, &a);
  const uint8_t o = in ? occ[a] : 0;
  if ((in && (o & 4)) || !in_box(g, p)) return true;
  return !c.optimistic && in && (o & 3) == FUELGPU_UNKNOWN;
}

__device__ __forceinline__ unsigned key_hash(const int* id) {
  unsigned h = (unsigned)id[0] * 73856093u ^ (unsigned)id[1] * 19349663u ^ (unsigned)id[2] * 83492791u;
  h ^= h >> 15;
  h *= 0x2c1b3c6du;
  h ^= h >> 12;
  return h;
}
__device__ int tab_find(const Slot* tab, unsigned mask, const int* id) {
  for (unsigned s = key_hash(id) & mask;; s = (s + 1) & mask) {
    const Slot e = tab[s];
    if (e.w < 0) return -1;
    if (e.x == id[0] && e.y == id[1] && e.z == id[2]) return e.w;
  }
}
__device__ int tab_insert(Slot* tab, unsigned mask, const int* id, int w) {
  unsigned s = key_hash(id) & mask;
  while (tab[s].w >= 0) s = (s + 1) & mask;
  tab[s] = Slot{ id[0], id[1], id[2], w };
  return (int)s;
}

struct Pool {  // one warp's search state in its scratch piece
  double *state, *input, *dur, *g, *f;
  int *par, *idx, *heap, *slot;
  uint8_t* closed;
  Slot* tab;
  double *cs, *cgf;  // candidates: state [NC][6], (g, f) [NC][2]
  int *cidx, *cint;  // candidates: index [NC][3], (ok, found, first, node) [NC][4]
  double* pts;       // getSamples' points, in the order it makes them
};

struct WarpShared {
  int cur, action, heap_len, use, iter, reason, shot, end_node;
  double coef[3][4], t_shot, end_vel[3];
};

// computeShotTraj (:331-394), lane 0
__device__ void shot_traj(const Geom& g, const uint8_t* __restrict__ occ, const KinoConsts& c, WarpShared& sh,
                          const double* s1, const double* s2, double t_d) {
  double dp[3], v0[3], dv[3], coef[3][4];
  for (int i = 0; i < 3; ++i) {
    dp[i] = s2[i] - s1[i];
    v0[i] = s1[3 + i];
    dv[i] = s2[3 + i] - v0[i];
    sh.end_vel[i] = s2[3 + i];
  }
  for (int i = 0; i < 3; ++i) {
    const double a = 1.0 / 6.0 * (-12.0 / (t_d * t_d * t_d) * (dp[i] - v0[i] * t_d) + 6 / (t_d * t_d) * dv[i]);
    const double b = 0.5 * (6.0 / (t_d * t_d) * (dp[i] - v0[i] * t_d) - 2 / t_d * dv[i]);
    coef[i][0] = s1[i], coef[i][1] = v0[i], coef[i][2] = b, coef[i][3] = a;
  }
  const double t_delta = t_d / 10;
  for (double time = t_delta; time <= t_d; time += t_delta) {
    const double t[4] = { 1.0, time, time * time, km_cube(time) };
    double coord[3];
    for (int i = 0; i < 3; ++i)
      coord[i] = ((coef[i][0] * t[0] + coef[i][1] * t[1]) + coef[i][2] * t[2]) + coef[i][3] * t[3];
    for (int i = 0; i < 3; ++i)
      if (coord[i] < g.origin[i] || coord[i] >= c.size[i]) return;  // map_size_3d_, not origin + size (getRegion)
    int64_t a;
    if (map_voxel(g, coord, &a) && (occ[a] & 4)) return;
  }
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 4; ++j) sh.coef[i][j] = coef[i][j];
  sh.t_shot = t_d;
  sh.shot = 1;
}

// KinodynamicAstar::search(start, vel, acc, goal, 0, init) on one warp; returns the status on every lane
__device__ int search(const Geom& g, const uint8_t* __restrict__ occ, const KinoConsts& c, const Pool& P,
                      WarpShared& sh, const double* sp, const double* sv, const double* sa, const double* ep, bool init) {
  const int lane = threadIdx.x & 31;
  const double end_state[6] = { ep[0], ep[1], ep[2], 0.0, 0.0, 0.0 };
  int end_index[3];
  for (int k = 0; k < 3; ++k) end_index[k] = (int)floor((ep[k] - g.origin[k]) * c.inv_res);
  double ttg;
  if (lane == 0) {
    for (int i = 0; i < 3; ++i) P.state[i] = sp[i], P.state[3 + i] = sv[i], P.input[i] = 0.0;
    P.par[0] = -1;
    for (int k = 0; k < 3; ++k) P.idx[k] = (int)floor((sp[k] - g.origin[k]) * c.inv_res);
    P.g[0] = 0.0;
    P.dur[0] = 0.0;
    P.f[0] = c.lambda * heuristic(c, P.state, end_state, &ttg);
    P.closed[0] = 0;
    P.heap[0] = 0;
    P.slot[0] = tab_insert(P.tab, c.tmask, P.idx, 0);
    sh.heap_len = 1, sh.use = 1, sh.iter = 0, sh.shot = 0, sh.end_node = -1;
  }
  bool init_search = init;
  int status = 0;
  for (;;) {
    if (lane == 0) {
      sh.action = 0;
      if (sh.heap_len == 0) {
        sh.reason = FUELGPU_KINO_OPEN_EMPTY;
        sh.action = KS_NO_PATH;
      } else {
        const int cur = P.heap[0];
        const double* cs = P.state + 6 * cur;
        const double d[3] = { cs[0] - sp[0], cs[1] - sp[1], cs[2] - sp[2] };
        const bool reach_horizon = sqrt(dot3(d, d)) >= c.horizon;
        const int* ci = P.idx + 3 * cur;
        const bool near_end = abs(ci[0] - end_index[0]) <= c.tol && abs(ci[1] - end_index[1]) <= c.tol &&
                              abs(ci[2] - end_index[2]) <= c.tol;
        if (reach_horizon || near_end) {
          sh.end_node = cur;
          if (near_end) {
            heuristic(c, cs, end_state, &ttg);
            shot_traj(g, occ, c, sh, cs, end_state, ttg);
          }
        }
        sh.reason = FUELGPU_KINO_FOUND;
        if (reach_horizon) {
          sh.action = sh.shot ? KS_REACH_END : KS_REACH_HORIZON;
        } else if (near_end) {
          if (sh.shot) {
            sh.action = KS_REACH_END;
          } else if (P.par[cur] >= 0) {
            sh.action = KS_NEAR_END;
          } else {
            sh.reason = FUELGPU_KINO_START_NEAR_END;
            sh.action = KS_NO_PATH;
          }
        } else {
          heap_pop(P.heap, sh.heap_len, P.f);
          --sh.heap_len;
          P.closed[cur] = 1;
          sh.iter += 1;
          sh.cur = cur;
        }
      }
    }
    __syncwarp();
    status = sh.action;
    const int cur = sh.cur;
    __syncwarp();
    if (status) break;
    double cur_state[6];
    for (int i = 0; i < 6; ++i) cur_state[i] = P.state[6 * cur + i];
    const int ci[3] = { P.idx[3 * cur], P.idx[3 * cur + 1], P.idx[3 * cur + 2] };
    const double cur_g = P.g[cur];
    const int n_acc = c.n_acc;
    const int n_dur = init_search ? c.n_init : 1;
    const int n_cand = init_search ? n_dur : n_acc * n_acc * n_acc;
    const double* taus = init_search ? c.tau_init : &c.tau_norm;
    for (int k = lane; k < n_cand; k += 32) {
      const int i = k / n_dur, j = k % n_dur;
      double um[3];
      if (init_search)
        um[0] = sa[0], um[1] = sa[1], um[2] = sa[2];
      else
        um[0] = c.acc[i / (n_acc * n_acc)], um[1] = c.acc[(i / n_acc) % n_acc], um[2] = c.acc[i % n_acc];
      const double tau = taus[j];
      const double* H = init_search ? c.h_init[j] : c.h_norm;
      double ps[6];
      transit(cur_state, ps, um, tau, H[0]);
      int pid[3];
      for (int a = 0; a < 3; ++a) pid[a] = (int)floor((ps[a] - g.origin[a]) * c.inv_res);
      bool ok = in_box(g, ps);
      int found = -1;
      if (ok) {
        found = tab_find(P.tab, c.tmask, pid);
        if (found >= 0 && P.closed[found]) ok = false;
      }
      if (ok && (fabs(ps[3]) > c.max_vel || fabs(ps[4]) > c.max_vel || fabs(ps[5]) > c.max_vel)) ok = false;
      if (ok && pid[0] == ci[0] && pid[1] == ci[1] && pid[2] == ci[2]) ok = false;
      if (ok)
        for (int q = 1; q <= c.check_num; ++q) {
          const double dt = tau * (double)q / (double)c.check_num;
          double xt[6];
          transit(cur_state, xt, um, dt, H[q]);
          if (unsafe(g, occ, c, xt)) {
            ok = false;
            break;
          }
        }
      if (ok) {
        const double tg = (dot3(um, um) + c.w_time) * tau + cur_g;
        double t2g;
        const double tf = tg + c.lambda * heuristic(c, ps, end_state, &t2g);
        for (int a = 0; a < 6; ++a) P.cs[6 * k + a] = ps[a];
        P.cgf[2 * k] = tg, P.cgf[2 * k + 1] = tf;
      }
      P.cidx[3 * k] = pid[0], P.cidx[3 * k + 1] = pid[1], P.cidx[3 * k + 2] = pid[2];
      P.cint[4 * k] = ok, P.cint[4 * k + 1] = found;
    }
    __syncwarp();
    // the first passing candidate of each new voxel makes its node; later ones in that voxel are pruned against it
    for (int k = lane; k < n_cand; k += 32) {
      int first = k;
      if (P.cint[4 * k] && P.cint[4 * k + 1] < 0)
        for (int q = 0; q < k; ++q)
          if (P.cint[4 * q] && P.cidx[3 * q] == P.cidx[3 * k] && P.cidx[3 * q + 1] == P.cidx[3 * k + 1] &&
              P.cidx[3 * q + 2] == P.cidx[3 * k + 2]) {
            first = q;
            break;
          }
      P.cint[4 * k + 2] = first;
    }
    __syncwarp();
    if (lane == 0) {
      for (int k = 0; k < n_cand; ++k) {
        if (!P.cint[4 * k]) continue;
        const int i = k / n_dur, j = k % n_dur;
        double um[3];
        if (init_search)
          um[0] = sa[0], um[1] = sa[1], um[2] = sa[2];
        else
          um[0] = c.acc[i / (n_acc * n_acc)], um[1] = c.acc[(i / n_acc) % n_acc], um[2] = c.acc[i % n_acc];
        const double tau = taus[j];
        const double tg = P.cgf[2 * k], tf = P.cgf[2 * k + 1];
        const int found = P.cint[4 * k + 1], first = P.cint[4 * k + 2];
        int e = -1;
        if (found >= 0) {
          if (tg < P.g[found]) e = found, P.par[found] = cur;  // the open-node update (:240-250)
        } else if (first != k) {
          e = P.cint[4 * first + 3];  // the prune (:192-208)
          if (!(tf < P.f[e])) e = -1;
        } else {
          e = sh.use;
          for (int a = 0; a < 3; ++a) P.idx[3 * e + a] = P.cidx[3 * k + a];
          P.par[e] = cur;
          P.closed[e] = 0;
        }
        if (e >= 0) {
          for (int a = 0; a < 6; ++a) P.state[6 * e + a] = P.cs[6 * k + a];
          for (int a = 0; a < 3; ++a) P.input[3 * e + a] = um[a];
          P.dur[e] = tau, P.g[e] = tg, P.f[e] = tf;
        }
        if (found < 0 && first == k) {
          heap_sift_up(P.heap, P.f, sh.heap_len++, e);
          P.slot[e] = tab_insert(P.tab, c.tmask, P.idx + 3 * e, e);
          P.cint[4 * k + 3] = e;
          sh.use += 1;
          if (sh.use == c.alloc) {
            sh.reason = FUELGPU_KINO_POOL;
            sh.action = KS_NO_PATH;
            break;
          }
        }
      }
    }
    init_search = false;
    __syncwarp();
    status = sh.action;
    __syncwarp();
    if (status) break;
  }
  return status;
}

__device__ void reset(const Pool& P, WarpShared& sh) {
  const int lane = threadIdx.x & 31;
  __syncwarp();
  for (int i = lane; i < sh.use; i += 32) P.tab[P.slot[i]].w = -1;
  __syncwarp();
}

__global__ void __launch_bounds__(KS_THREADS)
kino_kernel(Geom g, const uint8_t* __restrict__ occ, const __grid_constant__ KinoConsts c, int B, const double* __restrict__ start,
            const double* __restrict__ vel, const double* __restrict__ acc, const double* __restrict__ goal,
            const FuelPathInfo* __restrict__ gate, uint8_t* __restrict__ scratch, int* __restrict__ counter,
            FuelKinoInfo* __restrict__ info_out, double* __restrict__ points, double* __restrict__ derivs,
            double* __restrict__ dt_out, double* __restrict__ nodes_out, double* __restrict__ shot_out) {
  __shared__ WarpShared sh_all[KS_WARPS];
  const int lane = threadIdx.x & 31, wl = threadIdx.x >> 5;
  WarpShared& sh = sh_all[wl];
  uint8_t* base = scratch + (size_t)(blockIdx.x * KS_WARPS + wl) * c.stride;
  Pool P;
  P.state = (double*)base;
  P.input = (double*)(base + c.off_in);
  P.dur = (double*)(base + c.off_dur);
  P.g = (double*)(base + c.off_g);
  P.f = (double*)(base + c.off_f);
  P.par = (int*)(base + c.off_par);
  P.idx = (int*)(base + c.off_idx);
  P.closed = base + c.off_closed;
  P.heap = (int*)(base + c.off_heap);
  P.slot = (int*)(base + c.off_slot);
  P.tab = (Slot*)(base + c.off_tab);
  P.cs = (double*)(base + c.off_cs);
  P.cgf = (double*)(base + c.off_cgf);
  P.cidx = (int*)(base + c.off_cidx);
  P.cint = (int*)(base + c.off_cint);
  P.pts = (double*)(base + c.off_pts);

  for (;;) {
    int b = 0;
    if (lane == 0) b = atomicAdd(counter, 1);
    b = __shfl_sync(0xffffffffu, b, 0);
    if (b >= B) return;
    const double sp[3] = { start[3 * b], start[3 * b + 1], start[3 * b + 2] };
    const double sv[3] = { vel[3 * b], vel[3 * b + 1], vel[3 * b + 2] };
    const double sa[3] = { acc[3 * b], acc[3 * b + 1], acc[3 * b + 2] };
    const double ep[3] = { goal[3 * b], goal[3 * b + 1], goal[3 * b + 2] };
    FuelKinoInfo inf;
    memset(&inf, 0, sizeof(inf));
    inf.traj_status = FUELGPU_KINO_NO_TRAJ;
    bool finite = true;
    for (int k = 0; k < 3; ++k) finite = finite && isfinite(sp[k]) && isfinite(sv[k]) && isfinite(sa[k]) && isfinite(ep[k]);
    const double d[3] = { sp[0] - ep[0], sp[1] - ep[1], sp[2] - ep[2] };
    int status = 0;
    if (gate && gate[b].branch != FUELGPU_ASTAR_MID) {
      inf.status = FUELGPU_KINO_SKIPPED;
    } else if (!finite) {
      inf.status = FUELGPU_KINO_BAD_INPUT;
    } else if (sqrt(dot3(d, d)) < 1e-2) {  // "Close goal" (:131-134)
      inf.status = FUELGPU_KINO_NO_PATH;
      inf.reason = FUELGPU_KINO_CLOSE_GOAL;
    } else {
      status = search(g, occ, c, P, sh, sp, sv, sa, ep, true);
      if (status == KS_NO_PATH) {
        reset(P, sh);
        inf.retried = 1;
        status = search(g, occ, c, P, sh, sp, sv, sa, ep, false);
      }
      inf.status = status;
      inf.reason = sh.reason;
      inf.iter_num = sh.iter;
      inf.use_node_num = sh.use;
    }
    double* pts_b = points + (size_t)b * KS_K * 3;
    double* der_b = derivs + (size_t)b * 12;
    int n_pts_written = 0;
    if (lane == 0 && status && status != KS_NO_PATH) {
      // getSamples (:543-634)
      const int back = sh.end_node;
      inf.shot = sh.shot;
      inf.t_shot = sh.shot ? sh.t_shot : 0.0;
      double T_sum = 0.0;
      if (sh.shot) T_sum += sh.t_shot;
      int node = back, cnt = 1;
      while (P.par[node] >= 0) {
        T_sum += P.dur[node];
        node = P.par[node];
        ++cnt;
      }
      inf.n_nodes = cnt;
      double end_vel[3], end_acc[3], t;
      if (sh.shot) {
        t = sh.t_shot;
        for (int i = 0; i < 3; ++i) end_vel[i] = sh.end_vel[i], end_acc[i] = 2 * sh.coef[i][2] + 6 * sh.coef[i][3] * sh.t_shot;
      } else {  // node has walked to the root: end_vel is the root's velocity
        t = P.dur[back];
        for (int i = 0; i < 3; ++i) end_vel[i] = P.state[6 * node + 3 + i], end_acc[i] = P.input[3 * back + i];
      }
      int seg_num = (int)floor(T_sum / c.ts0);
      seg_num = max(8, seg_num);
      const double ts = T_sum / (double)seg_num;
      inf.seg_num = seg_num;
      inf.T_sum = T_sum;
      bool sample_shot = sh.shot;
      node = back;
      int n = 0;
      bool too_long = false;
      for (double ti = T_sum; ti > -1e-5; ti -= ts) {
        if (n == KS_K) {
          too_long = true;
          break;
        }
        if (sample_shot) {
          const double tm[4] = { 1.0, t, t * t, km_cube(t) };
          for (int i = 0; i < 3; ++i)
            P.pts[3 * n + i] = ((sh.coef[i][0] * tm[0] + sh.coef[i][1] * tm[1]) + sh.coef[i][2] * tm[2]) + sh.coef[i][3] * tm[3];
          ++n;
          t -= ts;
          if (t < -1e-5) {
            sample_shot = false;
            if (P.par[node] >= 0) t += P.dur[node];
          }
        } else {
          double xt[6];
          transit(P.state + 6 * P.par[node], xt, P.input + 3 * node, t, 0.5 * (t * t));
          for (int i = 0; i < 3; ++i) P.pts[3 * n + i] = xt[i];
          ++n;
          t -= ts;
          if (t < -1e-5 && P.par[P.par[node]] >= 0) {
            node = P.par[node];
            t += P.dur[node];
          }
        }
      }
      if (too_long) {
        inf.traj_status = FUELGPU_KINO_TOO_LONG;
      } else {
        inf.traj_status = 0;
        inf.n_pts = n + 2;
        n_pts_written = n;
        for (int i = 0; i < 3; ++i) {
          der_b[i] = sv[i];
          der_b[3 + i] = end_vel[i];
          der_b[6 + i] = P.par[back] < 0 ? 2 * sh.coef[i][2] : P.input[3 * node + i];
          der_b[9 + i] = end_acc[i];
        }
        dt_out[b] = ts;
      }
    }
    n_pts_written = __shfl_sync(0xffffffffu, n_pts_written, 0);
    if (lane == 0) {
      if (inf.traj_status != 0) {
        dt_out[b] = __longlong_as_double(0x7ff8000000000000LL);
        for (int i = 0; i < 12; ++i) der_b[i] = 0.0;
      }
      info_out[b] = inf;
    }
    __syncwarp();
    for (int i = lane; i < KS_K * 3; i += 32) {  // the points reversed, zero past K
      const int r = i / 3;
      pts_b[i] = r < n_pts_written ? P.pts[3 * (n_pts_written - 1 - r) + i % 3] : 0.0;
    }
    const int n_nodes = __shfl_sync(0xffffffffu, inf.n_nodes, 0);
    if (nodes_out) {  // the path root .. end: state, input, duration, g, f
      double* o = nodes_out + (size_t)b * c.node_max * 12;
      for (int i = lane; i < c.node_max * 12; i += 32) o[i] = 0.0;
      __syncwarp();
      if (lane == 0 && n_nodes > 0) {
        int i = n_nodes - 1;
        for (int nd = sh.end_node; nd >= 0; nd = P.par[nd], --i) {
          if (i >= c.node_max) continue;
          double* r = o + 12 * (size_t)i;
          for (int a = 0; a < 6; ++a) r[a] = P.state[6 * nd + a];
          for (int a = 0; a < 3; ++a) r[6 + a] = P.input[3 * nd + a];
          r[9] = P.dur[nd], r[10] = P.g[nd], r[11] = P.f[nd];
        }
      }
    }
    if (shot_out && lane < 12) {
      const int sh_ok = __shfl_sync(0x00000fffu, (int)(inf.shot), 0);
      shot_out[(size_t)b * 12 + lane] = sh_ok ? sh.coef[lane / 4][lane % 4] : 0.0;
    }
    // clear the key-table slots this search used
    if (status) reset(P, sh);
    __syncwarp();
  }
}

}  // namespace

// Scratch of one warp, in 256-byte pieces: per node A: state 48, input 24, duration, g, f 8 each, parent 4, index 12,
// closed 1, open set 4, table slot 4; the key table 16 T (T the least power of two >= 2 A, at least 64); per candidate
// (KS_MAX_CAND): state 48, g and f 16, index 12, flags 16; the samples 24 (FUELGPU_MAX_PTS - 2).
static void kino_layout(int A, KinoConsts* c) {
  auto al = [](size_t b) { return (b + 255) & ~(size_t)255; };
  size_t T = 64;
  while (T < 2 * (size_t)A) T <<= 1;
  c->tmask = (unsigned)(T - 1);
  const size_t a = (size_t)A, nc = KS_MAX_CAND;
  size_t o = al(48 * a);
  c->off_in = o, o += al(24 * a);
  c->off_dur = o, o += al(8 * a);
  c->off_g = o, o += al(8 * a);
  c->off_f = o, o += al(8 * a);
  c->off_par = o, o += al(4 * a);
  c->off_idx = o, o += al(12 * a);
  c->off_closed = o, o += al(a);
  c->off_heap = o, o += al(4 * a);
  c->off_slot = o, o += al(4 * a);
  c->off_tab = o, o += al(16 * T);
  c->off_cs = o, o += al(48 * nc);
  c->off_cgf = o, o += al(16 * nc);
  c->off_cidx = o, o += al(12 * nc);
  c->off_cint = o, o += al(16 * nc);
  c->off_pts = o, o += al(24 * (size_t)KS_K);
  c->stride = o;
}

constexpr size_t KS_BUDGET = (size_t)4 << 30;  // bytes of search scratch the warps running at once may use

// the duration and input lists of the reference's loops (:107-122) and their 0.5 * pow(t, 2) tables, with the host's
// pow; false when a list outgrows the tables
static bool kino_tables(const FuelKinoParams* p, KinoConsts* c) {
  std::vector<double> v;
  for (double tau = 1 / 20.0 * p->init_max_tau; tau <= p->init_max_tau + 1e-3; tau += 1 / 20.0 * p->init_max_tau) {
    if (v.size() == KS_MAX_INIT) return false;
    v.push_back(tau);
  }
  c->n_init = (int)v.size();
  for (int j = 0; j < c->n_init; ++j) c->tau_init[j] = v[j];
  c->tau_norm = 1 / 1.0 * p->max_tau;
  v.clear();
  for (double a = -p->max_acc; a <= p->max_acc + 1e-3; a += p->max_acc * (1 / 2.0)) {
    if (v.size() == KS_MAX_ACC) return false;
    v.push_back(a);
  }
  c->n_acc = (int)v.size();
  for (int j = 0; j < c->n_acc; ++j) c->acc[j] = v[j];
  auto fill = [&](const double* taus, int n, double (*h)[KS_MAX_CHECK + 1]) {
    for (int j = 0; j < n; ++j) {
      h[j][0] = 0.5 * pow(taus[j], 2);
      for (int k = 1; k <= p->check_num; ++k) {
        const double dt = taus[j] * double(k) / double(p->check_num);
        h[j][k] = 0.5 * pow(dt, 2);
      }
    }
  };
  fill(c->tau_init, c->n_init, c->h_init);
  fill(&c->tau_norm, 1, &c->h_norm);
  return c->n_init > 0 && c->n_acc > 0;
}

int kino_check_params(FuelMap* m, const FuelKinoParams* p) {
  if (!p) return fuel_fail(m, FUELGPU_EINVAL, "null params");
  auto fp = [](double x) { return x > 0.0 && x <= 1.7976931348623157e308; };
  if (!fp(p->max_tau) || !fp(p->init_max_tau) || !fp(p->max_acc) || !fp(p->w_time) || !fp(p->horizon) ||
      !fp(p->ctrl_pt_dist) || !fp(p->manager_max_vel) || !fp(p->max_vel + p->vel_margin) || !isfinite(p->max_vel) ||
      !isfinite(p->vel_margin))
    return fuel_fail(m, FUELGPU_EINVAL, "max_tau, init_max_tau, max_acc, w_time, horizon, ctrl_pt_dist, manager_max_vel "
                                        "and max_vel + vel_margin must be finite and positive");
  if (!(p->resolution >= 1e-6 && p->resolution <= 1e6)) return fuel_fail(m, FUELGPU_EINVAL, "resolution outside [1e-6, 1e6]");
  if (!isfinite(p->lambda_heu)) return fuel_fail(m, FUELGPU_EINVAL, "lambda_heu must be finite");
  if (p->allocate_num < 2 || p->allocate_num > (1 << 26)) return fuel_fail(m, FUELGPU_EINVAL, "allocate_num outside 2..2^26");
  if (p->check_num < 1 || p->check_num > KS_MAX_CHECK) return fuel_fail(m, FUELGPU_EINVAL, "check_num outside 1..16");
  KinoConsts* c = new KinoConsts();
  const bool ok = kino_tables(p, c);
  delete c;
  if (!ok)
    return fuel_fail(m, FUELGPU_EINVAL, "more than 32 init durations or 8 acceleration steps per axis");
  return 0;
}

int kino_search_impl(FuelMap* m, int B, const double* start, const double* vel, const double* acc, const double* goal,
                     const FuelPathInfo* gate, const FuelKinoParams* p, FuelKinoInfo* info, double* points,
                     double* derivs, double* dt, int node_max, double* nodes, double* shot) {
  if (B == 0) return 0;
  KinoConsts c;
  memset(&c, 0, sizeof(c));
  kino_tables(p, &c);
  c.max_vel = p->max_vel + p->vel_margin;  // setParam (:280-282)
  c.w_time = p->w_time;
  c.horizon = p->horizon;
  c.lambda = p->lambda_heu;
  c.inv_res = 1.0 / p->resolution;
  c.tol = (int)ceil(1 / p->resolution);
  c.ts0 = p->ctrl_pt_dist / p->manager_max_vel;  // kinodynamicReplan (:162)
  for (int i = 0; i < 3; ++i)
    c.size[i] = m->desc.map_size[i] > 0.0 ? m->desc.map_size[i] : m->desc.n[i] * m->desc.resolution;
  c.alloc = p->allocate_num;
  c.check_num = p->check_num;
  c.optimistic = p->optimistic != 0;
  c.node_max = nodes ? node_max : 0;
  kino_layout(c.alloc, &c);
  size_t W = (size_t)B;
  W = std::min(W, (size_t)m->sm_count * 32);
  W = std::min(W, std::max((size_t)1, KS_BUDGET / c.stride));
  const size_t blocks = (W + KS_WARPS - 1) / KS_WARPS, warps = blocks * KS_WARPS;
  bool fresh = false;
  const int rc = m->ks_buf.ensure(m, 256 + warps * c.stride, &fresh);
  if (rc) return rc;
  uint8_t* scr = m->ks_buf.p + 256;
  // every key table starts empty (all bits set); a search clears the slots it used before it ends, so only a new
  // block, a new layout or warps not used before need the fill, and only of their key tables
  const size_t tab_bytes = 16 * ((size_t)c.tmask + 1);
  if (fresh || m->ks_stride != c.stride) {
    FUEL_CUDA(m, cudaMemset2DAsync(scr + c.off_tab, c.stride, 0xff, tab_bytes, warps, m->stream));
    m->ks_stride = c.stride;
    m->ks_warps = warps;
  } else if (warps > m->ks_warps) {
    FUEL_CUDA(m, cudaMemset2DAsync(scr + m->ks_warps * c.stride + c.off_tab, c.stride, 0xff, tab_bytes,
                                   warps - m->ks_warps, m->stream));
    m->ks_warps = warps;
  }
  int* counter = (int*)m->ks_buf.p;
  FUEL_CUDA(m, cudaMemsetAsync(counter, 0, sizeof(int), m->stream));
  kino_kernel<<<(unsigned)blocks, KS_THREADS, 0, m->stream>>>(m->g, m->occ, c, B, start, vel, acc, goal, gate, scr,
                                                               counter, info, points, derivs, dt, nodes, shot);
  FUEL_LAUNCHES(m, 1);
  FUEL_CUDA(m, cudaGetLastError());
  return 0;
}
