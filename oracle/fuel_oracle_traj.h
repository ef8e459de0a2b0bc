/*
 * fuel_oracle_traj.h -- CPU restatement of NonUniformBspline (bspline/src/non_uniform_bspline.cpp) for uniform cubic
 * splines, FastPlannerManager::checkTrajCollision and selectBestTraj (plan_manage/src/planner_manager.cpp:96-118,
 * 476-482): fuel_oracle_traj.c, built into libfuel_oracle_traj.so by traj.mk.
 *
 * TEST INFRASTRUCTURE ONLY (see fuel_oracle.h).  Pinned bit for bit against the reference's own
 * non_uniform_bspline.cpp, compiled unmodified into _ref/libfuel_ref_traj.so (traj.mk, ref_traj_wrap.cpp), by
 * tests/test_oracle_traj.py.  parameterizeToBspline (a third-party QR) is compiled there but neither called nor restated.
 *
 * Splines come in the solver's layout: x [B][nvar], control point i of trajectory b at x[b][3i..3i+2];
 * nvar == 3n+1 -> dt = x[b][3n] (dt == NULL), nvar == 3n -> dt[b].
 */
#ifndef FUEL_ORACLE_TRAJ_H
#define FUEL_ORACLE_TRAJ_H

#include "fuel_oracle.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct {
  double max_vel, max_acc; /* setPhysicalLimits (:129-133) */
  double t_now;            /* checkTrajCollision's t_now (planner_manager.cpp:97) */
} OrcTrajCheckParams;
typedef struct {
  double duration, jerk, ratio, distance; /* getTimeSum, getJerk, checkRatio, checkTrajCollision's distance (-1: safe) */
  int32_t safe, feasible, n_checked, reserved;
} OrcTrajReport;
/* evaluateDeBoorT (:73-75) of the spline (deriv 0) or of getDerivative() applied deriv times (:97-106), at
 * t [B][n_t]; out [B][n_t][3] */
void orc_bspline_evaluate(int32_t B, int32_t n_pts, int32_t nvar, const double* x, const double* dt, int32_t n_t,
                          const double* t, int32_t deriv, double* out);
/* getTimeSum, getJerk, checkRatio, checkFeasibility and checkTrajCollision on the inflate buffer (char {0,1}) per
 * trajectory; best[0] = selectBestTraj (least jerk, lowest index on ties, NaN never), best[1] = the same among
 * safe && feasible (-1: none) */
void orc_bspline_check(const OrcGrid* g, const int8_t* inflate, int32_t B, int32_t n_pts, int32_t nvar, const double* x,
                       const double* dt, const OrcTrajCheckParams* p, OrcTrajReport* rep, int32_t best[2]);

#ifdef __cplusplus
}
#endif
#endif
