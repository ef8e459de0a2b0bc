/*
 * fuel_oracle_poly.h -- CPU restatement of PolynomialTraj::waypointsTraj (poly_traj/src/polynomial_traj.cpp:5-175), of
 * PolynomialTraj's evaluate / getTotalTime / getSamplePoints / getLength (poly_traj/include/poly_traj/polynomial_traj.h
 * :83-124) and of FastPlannerManager::planExploreTraj's lines 270-297 (plan_manage/src/planner_manager.cpp):
 * fuel_oracle_poly.c, built into libfuel_oracle_poly.so by poly.mk.
 *
 * TEST INFRASTRUCTURE ONLY (see fuel_oracle.h).  Pinned against the reference's own polynomial_traj.cpp, compiled
 * unmodified into _ref/libfuel_ref_poly.so (poly.mk, ref_poly_wrap.cpp), by tests/test_oracle_poly.py: A, Q, Ct, the
 * derivative vectors, the coefficients, getTotalTime, getLength and the sampling, bit for bit.  The three inverses the
 * reference takes (Eigen's inverse() of a dynamic matrix, a partial-pivot LU) are third-party: orc_lu_inverse restates
 * that algorithm, stays "parity unpinned", and is what the reference is compiled against (ref_standin_poly/Eigen/Eigen);
 * the tests check the coefficients against an exact rational minimizer instead.
 *
 * Matrices are row-major.  Coefficients: coeffs [S][3][6], segment k, axis j, cx[i] multiplies t^i.
 */
#ifndef FUEL_ORACLE_POLY_H
#define FUEL_ORACLE_POLY_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* inverse of the n x n matrix M by an LU factorization with partial pivoting (the largest |entry| of the column, the
 * first on ties), then one forward / back substitution per column of the identity.  Returns 0, -1 if a pivot is 0. */
int32_t orc_lu_inverse(int32_t n, const double* M, double* Minv);
/* Dense matrix product in the naive order: C[i][j] = sum over k, left to right, of A[i][k] * B[k][j]. */
void orc_matmul(int32_t n, int32_t m, int32_t p, const double* A, const double* B, double* C);
/* waypointsTraj for S = W - 1 >= 2 segments: waypts [W][3], start_vel, end_vel, start_acc, end_acc [3], times [S] ->
 * coeffs [S][3][6].  A [6S][6S], Q [6S][6S], Ct [6S][4S+2], D [3][6S] (Dx, Dy, Dz as built, before the solve) are
 * written when not NULL.  Returns 0, -1 when S < 2 (the reference writes Ct out of bounds at S = 1) or an inverse
 * fails. */
int32_t orc_poly_waypoints(int32_t S, const double* waypts, const double* start_vel, const double* end_vel,
                           const double* start_acc, const double* end_acc, const double* times, double* coeffs,
                           double* A, double* Q, double* Ct, double* D);
/* PolynomialTraj::evaluate(t, k) of S segments -> out [3] */
void orc_poly_evaluate(int32_t S, const double* coeffs, const double* times, double t, int32_t k, double* out);
/* getTotalTime */
double orc_poly_total_time(int32_t S, const double* times);
/* getLength (its getSamplePoints at eval_t = 0, += 0.01 while eval_t < total_t); *n_samples = their number */
double orc_poly_length(int32_t S, const double* coeffs, const double* times, int32_t* n_samples);
/* planExploreTraj :270-297 for one tour: times |p[i+1] - p[i]| / (max_vel * 0.5) (norm ((dx*dx + dy*dy) + dz*dz)),
 * waypointsTraj with zero end states, duration, length, seg_num = max(min_seg_num, (int)(length / ctrl_pt_dist)),
 * dt = duration / seg_num, the samples at ts = 0, += dt while ts <= duration + 1e-4 (at most max_k written to
 * points [max_k][3]), and derivs [4][3] = evaluate(0, 1), evaluate(duration, 1), evaluate(0, 2), evaluate(duration, 2).
 * times_out [S] and coeffs [S][3][6] may be NULL.  out_d = {duration, length, dt}, out_i = {seg_num, K}.  Returns as
 * orc_poly_waypoints. */
int32_t orc_explore_samples(int32_t W, const double* waypts, const double* cur_vel, const double* cur_acc, double max_vel,
                            double ctrl_pt_dist, int32_t min_seg_num, int32_t max_k, double* times_out, double* coeffs,
                            double* points, double* derivs, double* out_d, int32_t* out_i);

#ifdef __cplusplus
}
#endif
#endif
