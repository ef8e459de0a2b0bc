/* fuel_oracle_traj.c -- CPU restatement of NonUniformBspline (bspline/src/non_uniform_bspline.cpp) for uniform cubic
 * splines, of FastPlannerManager::checkTrajCollision (plan_manage/src/planner_manager.cpp:96-118) and of selectBestTraj
 * (:476-482).  TEST INFRASTRUCTURE ONLY (see fuel_oracle.h).  Sequential fp64, no FMA contraction, in the reference's
 * order: what the device check (fuel_b200/csrc/traj_check.cu) must equal bit for bit.  Declared in fuel_oracle_traj.h. */
#include <math.h>
#include <stdlib.h>

#include "fuel_oracle_traj.h"

#define ORC_TRAJ_MAX_PTS 64
#define ORC_CHECK_MAX_SAMPLES (1 << 20) /* FUELGPU_CHECK_MAX_SAMPLES */

typedef struct {
  int p, nc;                         /* p_, control_points_.rows() */
  double c[ORC_TRAJ_MAX_PTS][3];     /* control_points_ */
  double u[ORC_TRAJ_MAX_PTS + 4];    /* u_, m_ + 1 = nc + p + 1 knots */
} Spline;

/* setUniformBspline (:16-32) */
static void set_uniform(Spline* s, const double* ctrl, int n, double dt) {
  s->p = 3;
  s->nc = n;
  for (int i = 0; i < n; ++i)
    for (int j = 0; j < 3; ++j) s->c[i][j] = ctrl[3 * i + j];
  const int m = n + 3;
  for (int i = 0; i <= m; ++i) s->u[i] = i <= 3 ? (double)(-3 + i) * dt : s->u[i - 1] + dt;
}

/* getDerivativeControlPoints + getDerivative (:77-86, :97-106): degree p-1, knots u_[1..m-1] */
static void derivative(const Spline* s, Spline* d) {
  const int p = s->p;
  d->p = p - 1;
  d->nc = s->nc - 1;
  for (int i = 0; i < d->nc; ++i)
    for (int j = 0; j < 3; ++j) d->c[i][j] = (p * (s->c[i + 1][j] - s->c[i][j])) / (s->u[i + p + 1] - s->u[i + 1]);
  const int nk = s->nc + p + 1;  /* u_.rows() */
  for (int i = 0; i < nk - 2; ++i) d->u[i] = s->u[i + 1];
}

static inline double std_max(double a, double b) { return a < b ? b : a; }
static inline double std_min(double a, double b) { return b < a ? b : a; }

/* evaluateDeBoor (:51-71) / evaluateDeBoorT (:73-75) */
static void eval_t(const Spline* s, double t, double out[3]) {
  const int p = s->p, m = s->nc + p;
  const double ub = std_min(std_max(s->u[p], t + s->u[p]), s->u[m - p]);
  int k = p;
  while (s->u[k + 1] < ub) ++k;
  double d[4][3];
  for (int i = 0; i <= p; ++i)
    for (int j = 0; j < 3; ++j) d[i][j] = s->c[k - p + i][j];
  for (int r = 1; r <= p; ++r)
    for (int i = p; i >= r; --i) {
      const double alpha = (ub - s->u[i + k - p]) / (s->u[i + 1 + k - r] - s->u[i + k - p]);
      for (int j = 0; j < 3; ++j) d[i][j] = (1 - alpha) * d[i - 1][j] + alpha * d[i][j];
    }
  for (int j = 0; j < 3; ++j) out[j] = d[p][j];
}

static void load(Spline* s, int b, int n, int nvar, const double* x, const double* dt) {
  const double* xb = x + (size_t)b * nvar;
  set_uniform(s, xb, n, nvar == 3 * n + 1 ? xb[3 * n] : dt[b]);
}

void orc_bspline_evaluate(int32_t B, int32_t n_pts, int32_t nvar, const double* x, const double* dt, int32_t n_t,
                          const double* t, int32_t deriv, double* out) {
  Spline s[3];
  for (int b = 0; b < B; ++b) {
    load(&s[0], b, n_pts, nvar, x, dt);
    for (int k = 1; k <= deriv; ++k) derivative(&s[k - 1], &s[k]);
    for (int q = 0; q < n_t; ++q) {
      const size_t o = (size_t)b * n_t + q;
      eval_t(&s[deriv], t[o], out + 3 * o);
    }
  }
}

/* SDFMap::getInflateOccupancy(pos) (sdf_map.h:217-226) with posToIndex (:127-130) and isInMap(idx) (:163-169) */
static int inflate_occupancy(const OrcGrid* g, const int8_t* inflate, const double pos[3]) {
  int32_t id[3];
  orc_pos_to_index(g, pos, id);
  for (int i = 0; i < 3; ++i)
    if (id[i] < 0 || id[i] > g->n[i] - 1) return -1;
  return inflate[(int64_t)id[0] * g->n[1] * g->n[2] + (int64_t)id[1] * g->n[2] + id[2]];
}

static double norm3(const double a[3], const double b[3]) {
  const double d0 = a[0] - b[0], d1 = a[1] - b[1], d2 = a[2] - b[2];
  return sqrt(d0 * d0 + d1 * d1 + d2 * d2);
}

void orc_bspline_check(const OrcGrid* g, const int8_t* inflate, int32_t B, int32_t n_pts, int32_t nvar, const double* x,
                       const double* dt, const OrcTrajCheckParams* prm, OrcTrajReport* rep, int32_t best[2]) {
  for (int b = 0; b < B; ++b) {
    Spline s = { 0 }, d1, d2, d3;
    load(&s, b, n_pts, nvar, x, dt);
    const int p = s.p;
    OrcTrajReport r = { 0 };
    /* getTimeSum (:267-269) */
    r.duration = s.u[s.nc] - s.u[p]; /* u_(m_ - p_) with m_ = nc + p_ */
    /* getJerk (:283-298) */
    derivative(&s, &d1);
    derivative(&d1, &d2);
    derivative(&d2, &d3);
    double jerk = 0.0;
    for (int i = 0; i < d3.nc; ++i)
      for (int j = 0; j < 3; ++j) jerk += (d3.u[i + 1] - d3.u[i]) * d3.c[i][j] * d3.c[i][j];
    r.jerk = jerk;
    /* checkRatio (:135-160) and checkFeasibility (:443-487) */
    double max_vel = -1.0, max_acc = -1.0;
    int fea = 1;
    for (int i = 0; i < s.nc - 1; ++i) {
      double vel[3];
      for (int j = 0; j < 3; ++j) vel[j] = (p * (s.c[i + 1][j] - s.c[i][j])) / (s.u[i + p + 1] - s.u[i + 1]);
      if (fabs(vel[0]) > prm->max_vel + 1e-4 || fabs(vel[1]) > prm->max_vel + 1e-4 || fabs(vel[2]) > prm->max_vel + 1e-4)
        fea = 0;
      for (int j = 0; j < 3; ++j) max_vel = std_max(max_vel, fabs(vel[j]));
    }
    for (int i = 0; i < s.nc - 2; ++i) {
      double acc[3];
      for (int j = 0; j < 3; ++j)
        acc[j] = (p * (p - 1) * ((s.c[i + 2][j] - s.c[i + 1][j]) / (s.u[i + p + 2] - s.u[i + 2]) -
                                 (s.c[i + 1][j] - s.c[i][j]) / (s.u[i + p + 1] - s.u[i + 1]))) /
                 (s.u[i + p + 1] - s.u[i + 2]);
      if (fabs(acc[0]) > prm->max_acc + 1e-4 || fabs(acc[1]) > prm->max_acc + 1e-4 || fabs(acc[2]) > prm->max_acc + 1e-4)
        fea = 0;
      for (int j = 0; j < 3; ++j) max_acc = std_max(max_acc, fabs(acc[j]));
    }
    r.ratio = std_max(max_vel / prm->max_vel, sqrt(fabs(max_acc) / prm->max_acc));
    r.feasible = fea;
    /* checkTrajCollision (planner_manager.cpp:96-118) */
    const double t_now = prm->t_now;
    double cur[3], fut[3];
    eval_t(&s, t_now, cur);
    double radius = 0.0, fut_t = 0.02;
    r.safe = 1;
    r.distance = -1.0;
    while (radius < 6.0 && t_now + fut_t < r.duration && r.n_checked < ORC_CHECK_MAX_SAMPLES) {
      eval_t(&s, t_now + fut_t, fut);
      ++r.n_checked;
      if (inflate_occupancy(g, inflate, fut) == 1) {
        r.distance = radius;
        r.safe = 0;
        break;
      }
      radius = norm3(fut, cur);
      fut_t += 0.02;
    }
    rep[b] = r;
  }
  /* selectBestTraj (planner_manager.cpp:476-482) */
  best[0] = best[1] = -1;
  for (int b = 0; b < B; ++b) {
    const double j = rep[b].jerk;
    if (isnan(j)) continue;
    if (best[0] < 0 || j < rep[best[0]].jerk) best[0] = b;
    if (rep[b].safe && rep[b].feasible && (best[1] < 0 || j < rep[best[1]].jerk)) best[1] = b;
  }
}
