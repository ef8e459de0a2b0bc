/* CPU restatement of FastPlannerManager::kinodynamicReplan's search (plan_manage/src/planner_manager.cpp:131-164):
 * the close-goal refusal, KinodynamicAstar::reset / search(start, vel, acc, goal, 0, init) with the retry at init = false
 * (path_searching/src/kinodynamic_astar.cpp:15-263, 484-501), retrievePath, estimateHeuristic / cubic / quartic
 * (:296-329, :396-458), computeShotTraj (:331-394) and getSamples (:543-634) at ts = ctrl_pt_dist / max_vel, over the
 * occupancy byte the device reads (bits 0-1 tri-state, bit 2 inflate).
 * The open set is libstdc++'s std::priority_queue (push_heap / pop_heap) over node ids compared through each node's
 * current f_score: the reference assigns f_score to nodes inside the heap and never re-heaps.  expanded_nodes_ is an
 * open-addressing table keyed by the node index (insert never overwrites; the search only inserts new keys).
 * Vector sums run left to right ((x*x + y*y) + z*z), phi_ * state0 over its six columns in order.
 * ORC_KINO_GLIBC calls libm as the reference does; ORC_KINO_DEVICE is the device's arithmetic: the search's powers are
 * the same libm pow values, pow(t, 2) and pow(t, 3) outside the search are correctly rounded, and the D < 0 branch of
 * cubic() takes acos and cos correctly rounded (binary128, rounded to double).
 * TEST INFRASTRUCTURE ONLY (the GPU tests compare the device with ORC_KINO_DEVICE, tests/test_oracle_kino.py compares the
 * two modes). */
#include "fuel_oracle_kino.h"

#include <math.h>
#include <quadmath.h>
#include <stdlib.h>
#include <string.h>

#define MAX_PTS 64 /* FUELGPU_MAX_PTS */
enum { REACH_HORIZON = 1, REACH_END = 2, NO_PATH = 3, NEAR_END = 4 };
enum { R_FOUND = 0, R_OPEN_EMPTY = 1, R_POOL = 2, R_START_NEAR_END = 3, R_CLOSE_GOAL = 4 };

typedef struct {
  int x, y, z, w; /* w = node id, -1 empty */
} Slot;

typedef struct {
  const OrcAstarMap* m;
  const OrcKinoParams* p;
  int math;
  double size[3], max_vel, inv_res;
  int tol, A;
  double *state, *input, *dur, *g, *f;
  int *par, *idx, *heap, *slot;
  char* closed;
  Slot* tab;
  unsigned mask;
  int heap_len, use, iter;
  int shot;
  double coef[3][4], t_shot, end_vel[3], start_vel[3], start_acc[3];
  int end_node;
} K;

static double dot3(const double a[3], const double b[3]) { return (a[0] * b[0] + a[1] * b[1]) + a[2] * b[2]; }

static double pow2(const K* k, double t) { return k->math == ORC_KINO_DEVICE ? t * t : pow(t, 2); }
static double pow3(const K* k, double t) {
  return k->math == ORC_KINO_DEVICE ? (double)((__float128)t * t * t) : pow(t, 3);
}

/* stateTransit (:657-668): phi_ * state0 + integral, integral = (0.5 * pow(tau, 2)) * um, tau * um */
static void transit(const double x0[6], double x1[6], const double um[3], double tau, double half_t2) {
  for (int i = 0; i < 6; ++i) {
    double s = 0.0;
    for (int j = 0; j < 6; ++j) {
      const double phi = i == j ? 1.0 : (i < 3 && j == i + 3 ? tau : 0.0);
      s = j == 0 ? phi * x0[0] : s + phi * x0[j];
    }
    x1[i] = s + (i < 3 ? half_t2 * um[i] : tau * um[i - 3]);
  }
}

static long long three_root_count; /* calls that took cubic()'s D < 0 branch (orc_kino_three_root_count) */

long long orc_kino_three_root_count(int32_t reset) {
  const long long n = three_root_count;
  if (reset) three_root_count = 0;
  return n;
}

static double cubic_front(const K* k, double a, double b, double c, double d) {
  const double a2 = b / a, a1 = c / a, a0 = d / a;
  const double Q = (3 * a1 - a2 * a2) / 9;
  const double R = (9 * a1 * a2 - 27 * a0 - 2 * a2 * a2 * a2) / 54;
  const double D = Q * Q * Q + R * R;
  if (D > 0) {
    const double S = cbrt(R + sqrt(D));
    const double T = cbrt(R - sqrt(D));
    return -a2 / 3 + (S + T);
  } else if (D == 0) {
    const double S = cbrt(R);
    return -a2 / 3 + S + S;
  }
  const double arg = R / sqrt(-Q * Q * Q);
  ++three_root_count;
  if (k->math == ORC_KINO_DEVICE) {
    const double theta = (double)acosq((__float128)arg);
    return 2 * sqrt(-Q) * (double)cosq((__float128)(theta / 3)) - a2 / 3;
  }
  const double theta = acos(arg);
  return 2 * sqrt(-Q) * cos(theta / 3) - a2 / 3;
}

/* quartic (:425-458); returns the root count */
static int quartic(const K* k, double a, double b, double c, double d, double e, double ts[4]) {
  const double a3 = b / a, a2 = c / a, a1 = d / a, a0 = e / a;
  const double y1 = cubic_front(k, 1, -a2, a1 * a3 - 4 * a0, 4 * a2 * a0 - a1 * a1 - a3 * a3 * a0);
  const double r = a3 * a3 / 4 - a2 + y1;
  if (r < 0) return 0;
  const double R = sqrt(r);
  double D, E;
  if (R != 0) {
    D = sqrt(0.75 * a3 * a3 - R * R - 2 * a2 + 0.25 * (4 * a3 * a2 - 8 * a1 - a3 * a3 * a3) / R);
    E = sqrt(0.75 * a3 * a3 - R * R - 2 * a2 - 0.25 * (4 * a3 * a2 - 8 * a1 - a3 * a3 * a3) / R);
  } else {
    D = sqrt(0.75 * a3 * a3 - 2 * a2 + 2 * sqrt(y1 * y1 - 4 * a0));
    E = sqrt(0.75 * a3 * a3 - 2 * a2 - 2 * sqrt(y1 * y1 - 4 * a0));
  }
  int n = 0;
  if (!isnan(D)) {
    ts[n++] = -a3 / 4 + R / 2 + D / 2;
    ts[n++] = -a3 / 4 + R / 2 - D / 2;
  }
  if (!isnan(E)) {
    ts[n++] = -a3 / 4 - R / 2 + E / 2;
    ts[n++] = -a3 / 4 - R / 2 - E / 2;
  }
  return n;
}

/* estimateHeuristic (:296-329) */
static double heuristic(const K* k, const double x1[6], const double x2[6], double* optimal_time) {
  const double dp[3] = { x2[0] - x1[0], x2[1] - x1[1], x2[2] - x1[2] };
  const double* v0 = x1 + 3;
  const double* v1 = x2 + 3;
  const double vs[3] = { v0[0] + v1[0], v0[1] + v1[1], v0[2] + v1[2] };
  const double w = k->p->w_time;
  const double c1 = -36 * dot3(dp, dp);
  const double c2 = 24 * dot3(vs, dp);
  const double c3 = -4 * (dot3(v0, v0) + dot3(v0, v1) + dot3(v1, v1));
  const double c4 = 0;
  double ts[5];
  int n = quartic(k, w, c4, c3, c2, c1, ts);
  const double v_max = k->max_vel * 0.5;
  double inf = 0.0;
  for (int i = 0; i < 3; ++i) inf = fmax(inf, fabs(x1[i] - x2[i]));
  const double t_bar = inf / v_max;
  ts[n++] = t_bar;
  double cost = 100000000, t_d = t_bar;
  for (int i = 0; i < n; ++i) {
    const double t = ts[i];
    if (t < t_bar) continue;
    const double cc = -c1 / (3 * t * t * t) - c2 / (2 * t * t) - c3 / t + w * t;
    if (cc < cost) cost = cc, t_d = t;
  }
  *optimal_time = t_d;
  return 1.0 * (1 + (1.0 + 1.0 / 10000)) * cost;
}

static void pos_index(const K* k, const double p[3], int id[3]) {
  for (int i = 0; i < 3; ++i) id[i] = (int)floor((p[i] - k->m->origin[i]) * k->inv_res);
}
static int map_index(const OrcAstarMap* m, const double p[3], int id[3]) {
  for (int i = 0; i < 3; ++i) id[i] = (int)floor((p[i] - m->origin[i]) * m->res_inv);
  for (int i = 0; i < 3; ++i)
    if (id[i] < 0 || id[i] > m->n[i] - 1) return 0;
  return 1;
}
static uint8_t occ_at(const OrcAstarMap* m, const int id[3]) {
  return m->occ[((int64_t)id[0] * m->n[1] + id[1]) * m->n[2] + id[2]];
}
static int in_box(const OrcAstarMap* m, const double p[3]) {
  for (int i = 0; i < 3; ++i)
    if (p[i] <= m->box_mind[i] || p[i] >= m->box_maxd[i]) return 0;
  return 1;
}
/* the safety test of one sample (:172-180): inflate bit, out of box, UNKNOWN unless optimistic */
static int unsafe(const K* k, const double p[3]) {
  int id[3];
  const int in = map_index(k->m, p, id);
  if ((in && (occ_at(k->m, id) & 4)) || !in_box(k->m, p)) return 1;
  return !k->p->optimistic && in && (occ_at(k->m, id) & 3) == 0;
}

static unsigned key_hash(const int id[3]) {
  unsigned h = (unsigned)id[0] * 73856093u ^ (unsigned)id[1] * 19349663u ^ (unsigned)id[2] * 83492791u;
  h ^= h >> 15;
  h *= 0x2c1b3c6du;
  h ^= h >> 12;
  return h;
}
static int tab_find(const K* k, const int id[3]) {
  for (unsigned s = key_hash(id) & k->mask;; s = (s + 1) & k->mask) {
    if (k->tab[s].w < 0) return -1;
    if (k->tab[s].x == id[0] && k->tab[s].y == id[1] && k->tab[s].z == id[2]) return k->tab[s].w;
  }
}
static int tab_insert(K* k, const int id[3], int w) {
  unsigned s = key_hash(id) & k->mask;
  while (k->tab[s].w >= 0) s = (s + 1) & k->mask;
  k->tab[s].x = id[0], k->tab[s].y = id[1], k->tab[s].z = id[2], k->tab[s].w = w;
  return (int)s;
}

/* libstdc++ push_heap / pop_heap with NodeComparator (node1->f_score > node2->f_score) */
static void sift_up(K* k, int hole, int v) {
  int parent = (hole - 1) / 2;
  while (hole > 0 && k->f[k->heap[parent]] > k->f[v]) {
    k->heap[hole] = k->heap[parent];
    hole = parent;
    parent = (hole - 1) / 2;
  }
  k->heap[hole] = v;
}
static void heap_push(K* k, int v) { sift_up(k, k->heap_len++, v); }
static void heap_pop(K* k) {
  const int len = k->heap_len--;
  if (len <= 1) return;
  const int n = len - 1, v = k->heap[n];
  k->heap[n] = k->heap[0];
  int hole = 0, child = 0;
  while (child < (n - 1) / 2) {
    child = 2 * (child + 1);
    if (k->f[k->heap[child]] > k->f[k->heap[child - 1]]) child--;
    k->heap[hole] = k->heap[child];
    hole = child;
  }
  if ((n & 1) == 0 && child == (n - 2) / 2) {
    child = 2 * (child + 1);
    k->heap[hole] = k->heap[child - 1];
    hole = child - 1;
  }
  sift_up(k, hole, v);
}

/* computeShotTraj (:331-394) */
static void shot_traj(K* k, const double s1[6], const double s2[6], double t_d) {
  double dp[3], v0[3], v1[3], dv[3], coef[3][4];
  for (int i = 0; i < 3; ++i) {
    dp[i] = s2[i] - s1[i];
    v0[i] = s1[3 + i];
    v1[i] = s2[3 + i];
    dv[i] = v1[i] - v0[i];
    k->end_vel[i] = v1[i];
  }
  for (int i = 0; i < 3; ++i) {
    const double a = 1.0 / 6.0 * (-12.0 / (t_d * t_d * t_d) * (dp[i] - v0[i] * t_d) + 6 / (t_d * t_d) * dv[i]);
    const double b = 0.5 * (6.0 / (t_d * t_d) * (dp[i] - v0[i] * t_d) - 2 / t_d * dv[i]);
    coef[i][0] = s1[i], coef[i][1] = v0[i], coef[i][2] = b, coef[i][3] = a;
  }
  const double t_delta = t_d / 10;
  for (double time = t_delta; time <= t_d; time += t_delta) {
    const double t[4] = { 1.0, time, pow2(k, time), pow3(k, time) };
    double coord[3];
    for (int i = 0; i < 3; ++i)
      coord[i] = ((coef[i][0] * t[0] + coef[i][1] * t[1]) + coef[i][2] * t[2]) + coef[i][3] * t[3];
    for (int i = 0; i < 3; ++i)
      if (coord[i] < k->m->origin[i] || coord[i] >= k->size[i]) return;
    int id[3];
    if (map_index(k->m, coord, id) && (occ_at(k->m, id) & 4)) return;
  }
  memcpy(k->coef, coef, sizeof(coef));
  k->t_shot = t_d;
  k->shot = 1;
}

/* the duration list of one expansion (:107-122) */
static int durations(const K* k, int init, double* taus) {
  int n = 0;
  if (init) {
    const double step = 1 / 20.0 * k->p->init_max_tau;
    for (double tau = step; tau <= k->p->init_max_tau + 1e-3; tau += step) taus[n++] = tau;
  } else {
    const double step = 1 / 1.0 * k->p->max_tau;
    for (double tau = step; tau <= k->p->max_tau; tau += step) taus[n++] = tau;
  }
  return n;
}
static int acc_values(const K* k, double* v) {
  int n = 0;
  for (double a = -k->p->max_acc; a <= k->p->max_acc + 1e-3; a += k->p->max_acc * (1 / 2.0)) v[n++] = a;
  return n;
}

static void reset(K* k) {
  for (int i = 0; i < k->use; ++i) k->tab[k->slot[i]].w = -1;
  k->use = k->iter = k->heap_len = 0;
  k->shot = 0;
  k->end_node = -1;
}

/* KinodynamicAstar::search(start, vel, acc, goal, 0, init) (:15-263); *reason gets why it ended */
static int search(K* k, const double sp[3], const double sv[3], const double sa[3], const double ep[3], int init,
                  int* reason) {
  const OrcKinoParams* p = k->p;
  memcpy(k->start_vel, sv, sizeof(double) * 3);
  memcpy(k->start_acc, sa, sizeof(double) * 3);
  for (int i = 0; i < 3; ++i) k->state[i] = sp[i], k->state[3 + i] = sv[i];
  k->par[0] = -1;
  pos_index(k, sp, k->idx);
  k->g[0] = 0.0;
  k->input[0] = k->input[1] = k->input[2] = 0.0;
  k->dur[0] = 0.0;
  const double end_state[6] = { ep[0], ep[1], ep[2], 0.0, 0.0, 0.0 };
  int end_index[3];
  pos_index(k, ep, end_index);
  double ttg;
  k->f[0] = p->lambda_heu * heuristic(k, k->state, end_state, &ttg);
  k->closed[0] = 0;
  heap_push(k, 0);
  k->use = 1;
  k->slot[0] = tab_insert(k, k->idx, 0);
  int init_search = init;
  double taus[64], accs[16];  /* the callers keep the counts within 32 and 8 */
  const int n_acc = acc_values(k, accs);
  int tmp[512];
  while (k->heap_len > 0) {
    const int cur = k->heap[0];
    const double* cs = k->state + 6 * cur;
    const double d[3] = { cs[0] - sp[0], cs[1] - sp[1], cs[2] - sp[2] };
    const int reach_horizon = sqrt(dot3(d, d)) >= p->horizon;
    const int* ci = k->idx + 3 * cur;
    const int near_end = abs(ci[0] - end_index[0]) <= k->tol && abs(ci[1] - end_index[1]) <= k->tol &&
                         abs(ci[2] - end_index[2]) <= k->tol;
    if (reach_horizon || near_end) {
      k->end_node = cur;
      if (near_end) {
        heuristic(k, cs, end_state, &ttg);
        shot_traj(k, cs, end_state, ttg);
      }
    }
    *reason = R_FOUND;
    if (reach_horizon) return k->shot ? REACH_END : REACH_HORIZON;
    if (near_end) {
      if (k->shot) return REACH_END;
      if (k->par[cur] >= 0) return NEAR_END;
      *reason = R_START_NEAR_END;
      return NO_PATH;
    }
    heap_pop(k);
    k->closed[cur] = 1;
    k->iter += 1;

    double cur_state[6];
    memcpy(cur_state, cs, sizeof(cur_state));
    const double cur_g = k->g[cur];
    const int n_in = init_search ? 1 : n_acc * n_acc * n_acc;
    const int n_dur = durations(k, init_search, taus);
    const int was_init = init_search;
    init_search = 0;
    int n_tmp = 0;
    for (int i = 0; i < n_in; ++i)
      for (int j = 0; j < n_dur; ++j) {
        double um[3];
        if (was_init)
          memcpy(um, k->start_acc, sizeof(um));
        else
          um[0] = accs[i / (n_acc * n_acc)], um[1] = accs[(i / n_acc) % n_acc], um[2] = accs[i % n_acc];
        const double tau = taus[j];
        double ps[6];
        transit(cur_state, ps, um, tau, 0.5 * pow(tau, 2));
        if (!in_box(k->m, ps)) continue;
        int pid[3];
        pos_index(k, ps, pid);
        int pro = tab_find(k, pid);
        if (pro >= 0 && k->closed[pro]) continue;
        if (fabs(ps[3]) > k->max_vel || fabs(ps[4]) > k->max_vel || fabs(ps[5]) > k->max_vel) continue;
        if (pid[0] == ci[0] && pid[1] == ci[1] && pid[2] == ci[2]) continue;
        int occ = 0;
        for (int c = 1; c <= p->check_num; ++c) {
          const double dt = tau * (double)c / (double)p->check_num;
          double xt[6];
          transit(cur_state, xt, um, dt, 0.5 * pow(dt, 2));
          if (unsafe(k, xt)) {
            occ = 1;
            break;
          }
        }
        if (occ) continue;
        const double tg = (dot3(um, um) + p->w_time) * tau + cur_g;
        const double tf = tg + p->lambda_heu * heuristic(k, ps, end_state, &ttg);
        int prune = 0;
        for (int t = 0; t < n_tmp; ++t) {
          const int e = tmp[t];
          if (pid[0] == k->idx[3 * e] && pid[1] == k->idx[3 * e + 1] && pid[2] == k->idx[3 * e + 2]) {
            prune = 1;
            if (tf < k->f[e]) {
              k->f[e] = tf, k->g[e] = tg;
              memcpy(k->state + 6 * e, ps, sizeof(ps));
              memcpy(k->input + 3 * e, um, sizeof(um));
              k->dur[e] = tau;
            }
            break;
          }
        }
        if (prune) continue;
        if (pro < 0) {
          pro = k->use;
          memcpy(k->idx + 3 * pro, pid, sizeof(pid));
          memcpy(k->state + 6 * pro, ps, sizeof(ps));
          k->f[pro] = tf, k->g[pro] = tg;
          memcpy(k->input + 3 * pro, um, sizeof(um));
          k->dur[pro] = tau;
          k->par[pro] = cur;
          k->closed[pro] = 0;
          heap_push(k, pro);
          k->slot[pro] = tab_insert(k, pid, pro);
          tmp[n_tmp++] = pro;
          k->use += 1;
          if (k->use == k->A) {
            *reason = R_POOL;
            return NO_PATH;
          }
        } else if (tg < k->g[pro]) {
          memcpy(k->state + 6 * pro, ps, sizeof(ps));
          k->f[pro] = tf, k->g[pro] = tg;
          memcpy(k->input + 3 * pro, um, sizeof(um));
          k->dur[pro] = tau;
          k->par[pro] = cur;
        }
      }
  }
  *reason = R_OPEN_EMPTY;
  return NO_PATH;
}

/* getSamples (:543-634); returns K, the sample count, or -1 when more than MAX_PTS - 2 */
static int samples(K* k, double* ts_io, double* points, double* derivs, int* seg_out, double* tsum_out) {
  const int back = k->end_node;
  double T_sum = 0.0;
  if (k->shot) T_sum += k->t_shot;
  int node = back;
  while (k->par[node] >= 0) {
    T_sum += k->dur[node];
    node = k->par[node];
  }
  double end_vel[3], end_acc[3], t;
  if (k->shot) {
    t = k->t_shot;
    for (int i = 0; i < 3; ++i) end_vel[i] = k->end_vel[i], end_acc[i] = 2 * k->coef[i][2] + 6 * k->coef[i][3] * k->t_shot;
  } else {
    t = k->dur[back];
    for (int i = 0; i < 3; ++i) end_vel[i] = k->state[6 * node + 3 + i], end_acc[i] = k->input[3 * back + i];
  }
  int seg_num = (int)floor(T_sum / *ts_io);
  seg_num = seg_num > 8 ? seg_num : 8;
  const double ts = T_sum / (double)seg_num;
  *ts_io = ts;
  *seg_out = seg_num;
  *tsum_out = T_sum;
  int sample_shot = k->shot;
  node = back;
  int n = 0;
  double pts[MAX_PTS - 2][3];
  for (double ti = T_sum; ti > -1e-5; ti -= ts) {
    if (n == MAX_PTS - 2) return -1;
    if (sample_shot) {
      const double tm[4] = { 1.0, t, pow2(k, t), pow3(k, t) };
      for (int i = 0; i < 3; ++i)
        pts[n][i] = ((k->coef[i][0] * tm[0] + k->coef[i][1] * tm[1]) + k->coef[i][2] * tm[2]) + k->coef[i][3] * tm[3];
      ++n;
      t -= ts;
      if (t < -1e-5) {
        sample_shot = 0;
        if (k->par[node] >= 0) t += k->dur[node];
      }
    } else {
      double xt[6];
      transit(k->state + 6 * k->par[node], xt, k->input + 3 * node, t, 0.5 * pow2(k, t));
      memcpy(pts[n++], xt, sizeof(double) * 3);
      t -= ts;
      if (t < -1e-5 && k->par[k->par[node]] >= 0) {
        node = k->par[node];
        t += k->dur[node];
      }
    }
  }
  for (int i = 0; i < n; ++i) memcpy(points + 3 * i, pts[n - 1 - i], sizeof(double) * 3);
  double start_acc[3];
  for (int i = 0; i < 3; ++i) start_acc[i] = k->par[back] < 0 ? 2 * k->coef[i][2] : k->input[3 * node + i];
  memcpy(derivs, k->start_vel, sizeof(double) * 3);
  memcpy(derivs + 3, end_vel, sizeof(double) * 3);
  memcpy(derivs + 6, start_acc, sizeof(double) * 3);
  memcpy(derivs + 9, end_acc, sizeof(double) * 3);
  return n;
}

int orc_kino_replan(const OrcAstarMap* m, const double map_size[3], const OrcKinoParams* p, int32_t math,
                    const double start[3], const double vel[3], const double acc[3], const double goal[3],
                    OrcKinoInfo* info, double* points, double* derivs, double* dt, int32_t node_max, double* nodes,
                    double* shot) {
  memset(info, 0, sizeof(*info));
  memset(points, 0, sizeof(double) * (MAX_PTS - 2) * 3);
  memset(derivs, 0, sizeof(double) * 12);
  if (nodes) memset(nodes, 0, sizeof(double) * 12 * (size_t)node_max);
  if (shot) memset(shot, 0, sizeof(double) * 12);
  *dt = NAN;
  info->traj_status = 2;
  const double d[3] = { start[0] - goal[0], start[1] - goal[1], start[2] - goal[2] };
  if (sqrt(dot3(d, d)) < 1e-2) {
    info->status = NO_PATH;
    info->reason = R_CLOSE_GOAL;
    return 0;
  }
  K k;
  memset(&k, 0, sizeof(k));
  k.m = m, k.p = p, k.math = math, k.A = p->allocate_num;
  for (int i = 0; i < 3; ++i) k.size[i] = map_size[i];
  k.max_vel = p->max_vel + p->vel_margin;
  k.inv_res = 1.0 / p->resolution;
  k.tol = (int)ceil(1 / p->resolution);
  size_t T = 64;
  while (T < 2 * (size_t)k.A) T <<= 1;
  k.mask = (unsigned)(T - 1);
  const size_t A = (size_t)k.A;
  k.state = malloc(sizeof(double) * 6 * A), k.input = malloc(sizeof(double) * 3 * A);
  k.dur = malloc(sizeof(double) * A), k.g = malloc(sizeof(double) * A), k.f = malloc(sizeof(double) * A);
  k.par = malloc(sizeof(int) * A), k.idx = malloc(sizeof(int) * 3 * A), k.heap = malloc(sizeof(int) * A);
  k.slot = malloc(sizeof(int) * A), k.closed = malloc(A), k.tab = malloc(sizeof(Slot) * T);
  int rc = -1;
  if (!k.state || !k.input || !k.dur || !k.g || !k.f || !k.par || !k.idx || !k.heap || !k.slot || !k.closed || !k.tab)
    goto out;
  for (size_t s = 0; s < T; ++s) k.tab[s].w = -1;
  rc = 0;
  int reason;
  reset(&k);
  int status = search(&k, start, vel, acc, goal, 1, &reason);
  if (status == NO_PATH) {
    info->retried = 1;
    reset(&k);
    status = search(&k, start, vel, acc, goal, 0, &reason);
  }
  info->status = status, info->reason = reason;
  info->iter_num = k.iter, info->use_node_num = k.use;
  if (status == NO_PATH) goto out;
  info->shot = k.shot;
  info->t_shot = k.shot ? k.t_shot : 0.0;
  int cnt = 0;
  for (int n = k.end_node; n >= 0; n = k.par[n]) ++cnt;
  info->n_nodes = cnt;
  if (nodes) {
    int i = cnt - 1;
    for (int n = k.end_node; n >= 0; n = k.par[n], --i) {
      if (i >= node_max) continue;
      double* o = nodes + 12 * (size_t)i;
      memcpy(o, k.state + 6 * n, sizeof(double) * 6);
      memcpy(o + 6, k.input + 3 * n, sizeof(double) * 3);
      o[9] = k.dur[n], o[10] = k.g[n], o[11] = k.f[n];
    }
  }
  if (shot && k.shot) memcpy(shot, k.coef, sizeof(k.coef));
  double ts = p->ctrl_pt_dist / p->manager_max_vel;
  const int n = samples(&k, &ts, points, derivs, &info->seg_num, &info->T_sum);
  if (n < 0) {
    info->traj_status = 1;
    memset(points, 0, sizeof(double) * (MAX_PTS - 2) * 3);
    memset(derivs, 0, sizeof(double) * 12);
    goto out;
  }
  info->traj_status = 0;
  info->n_pts = n + 2;
  *dt = ts;
out:
  free(k.state), free(k.input), free(k.dur), free(k.g), free(k.f), free(k.par), free(k.idx), free(k.heap);
  free(k.slot), free(k.closed), free(k.tab);
  return rc;
}
