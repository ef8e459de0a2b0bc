/*
 * fuel_oracle_param.h -- CPU restatement of NonUniformBspline::parameterizeToBspline (bspline/src/non_uniform_bspline.cpp
 * :178-265, degree 3), of getBoundaryStates(2, 0) (:108-123) and of the pt_dist_ BsplineOptimizer::optimize() freezes
 * (bspline_optimizer.cpp:136-140): fuel_oracle_param.c, built into libfuel_oracle_param.so by param.mk on top of
 * libfuel_oracle_traj.so (evaluateDeBoorT) and libfuel_oracle.so (orc_pt_dist).
 *
 * TEST INFRASTRUCTURE ONLY (see fuel_oracle.h).  Pinned against the reference's own non_uniform_bspline.cpp, compiled
 * unmodified into _ref/libfuel_ref_param.so (param.mk, ref_param_wrap.cpp), by tests/test_oracle_traj_param.py: the
 * system A, b and the boundary states bit for bit.  The solve, colPivHouseholderQr().solve(), is a third-party algorithm
 * (Eigen): it is restated below and stays "parity unpinned"; the reference is compiled against a stand-in that returns
 * this restatement (ref_standin_param/Eigen/Eigen), and the tests check it against exact rational least squares.
 *
 * Splines come in the solver's layout: x [B][nvar], control point i of trajectory b at x[b][3i..3i+2];
 * nvar == 3n+1 -> dt = x[b][3n] (dt == NULL), nvar == 3n -> dt[b].
 */
#ifndef FUEL_ORACLE_PARAM_H
#define FUEL_ORACLE_PARAM_H

#include "fuel_oracle.h"

#ifdef __cplusplus
extern "C" {
#endif

/* parameterizeToBspline's system, bit for bit: A [K+4][K+2] row-major, b [3][K+4] (one right-hand side per axis), from
 * points [K][3] and derivs [4][3] (start vel, end vel, start acc, end acc). */
void orc_bspline_param_system(int32_t K, double ts, const double* points, const double* derivs, double* A, double* b);
/* Its solve, "parity unpinned": a dense fp64 column-pivoted Householder least-squares solve, restated from the published
 * description of the algorithm Eigen's ColPivHouseholderQR names.  A [rows][cols] row-major, b [nrhs][rows] ->
 * x [nrhs][cols]; returns the numerical rank (-1: rows < cols or more than 128 columns). */
int32_t orc_lstsq_colpiv_qr(int32_t rows, int32_t cols, const double* A, int32_t nrhs, const double* b, double* x);
/* getBoundaryStates(2, 0) of setUniformBspline(ctrl, 3, dt) for B splines in the solver's layout:
 * start [B][3][3] (pos, vel, acc at t = 0), end [B][3] (position at getTimeSum()) */
void orc_bspline_boundary_states(int32_t B, int32_t n_pts, int32_t nvar, const double* x, const double* dt, double* start,
                                 double* end);
/* B trajectories of K = n_pts - 2 samples: points [B][K][3], derivs [B][4][3], dt [B], time_lb [B] or NULL (-1) ->
 * x [B][nvar] (control points; dt in the last column when nvar == 3 n_pts + 1) and tc [B]: pt_dist (orc_pt_dist),
 * knot_span = dt, start = the boundary states' start, end[0] = their end, n_end = 1, time_lb, view_idx = -1, the rest 0 */
void orc_bspline_parameterize(int32_t B, int32_t n_pts, int32_t nvar, const double* points, const double* derivs,
                              const double* dt, const double* time_lb, double* x, OrcTrajConst* tc);

#ifdef __cplusplus
}
#endif
#endif
