// Drives the reference's own PolynomialTraj (poly_traj/src/polynomial_traj.cpp:5-175 and the class in
// poly_traj/include/poly_traj/polynomial_traj.h, compiled unmodified from /root/reference against
// oracle/ref_standin_poly by oracle/poly.mk) so tests can compare the oracle with the real code.  The Eigen stand-in
// records the matrices waypointsTraj builds and inverts them with the oracle's orc_lu_inverse (Eigen's LU is
// third-party: "parity unpinned").  ref_poly_explore restates planExploreTraj's lines 270-297
// (plan_manage/src/planner_manager.cpp, which cannot be compiled here) over that compiled PolynomialTraj.
// TEST INFRASTRUCTURE ONLY; part of oracle/_ref/libfuel_ref_poly.so, built with hidden visibility: REF_API exports.
#include <stdint.h>

#include <algorithm>
#include <iostream>
#define private public  // the coefficients a Polynomial stores, and PolynomialTraj's times_
#include <poly_traj/polynomial_traj.h>
#undef private

#define REF_API __attribute__((visibility("default")))

using fast_planner::PolynomialTraj;

static void make_traj(int32_t S, const double* waypts, const double* sv, const double* ev, const double* sa,
                      const double* ea, const double* times, PolynomialTraj& traj) {
  Eigen::MatrixXd pos(S + 1, 3);
  for (int i = 0; i <= S; ++i)
    for (int j = 0; j < 3; ++j) pos(i, j) = waypts[3 * i + j];
  Eigen::VectorXd t(S);
  for (int i = 0; i < S; ++i) t(i) = times[i];
  Eigen::Vector3d v0(sv[0], sv[1], sv[2]), v1(ev[0], ev[1], ev[2]), a0(sa[0], sa[1], sa[2]), a1(ea[0], ea[1], ea[2]);
  PolynomialTraj::waypointsTraj(pos, v0, v1, a0, a1, t, traj);
}

static void read_coeffs(PolynomialTraj& traj, double* coeffs) {
  for (size_t k = 0; k < traj.segments_.size(); ++k)
    for (int i = 0; i < 6; ++i) {
      coeffs[(k * 3 + 0) * 6 + i] = traj.segments_[k].cx_[i];
      coeffs[(k * 3 + 1) * 6 + i] = traj.segments_[k].cy_[i];
      coeffs[(k * 3 + 2) * 6 + i] = traj.segments_[k].cz_[i];
    }
}

extern "C" {

// waypointsTraj for S >= 2 segments -> coeffs [S][3][6]; A, Q [6S][6S], Ct [6S][4S+2], D [3][6S] as it built them
REF_API void ref_poly_waypoints(int32_t S, const double* waypts, const double* sv, const double* ev, const double* sa,
                                const double* ea, const double* times, double* coeffs, double* A, double* Q, double* Ct,
                                double* D) {
  Eigen::PolyCapture& cap = Eigen::poly_capture();
  cap = Eigen::PolyCapture();
  PolynomialTraj traj;
  make_traj(S, waypts, sv, ev, sa, ea, times, traj);
  read_coeffs(traj, coeffs);
  const int nd = 6 * S;
  for (const Eigen::MatrixXd& m : cap.inv_args)  // A: A(1, 0) = 1; its transpose, inverted first, has A(0, 1) = 1
    if (m.rows() == nd && m(1, 0) == 1.0) std::copy(m.d.begin(), m.d.end(), A);
  std::copy(cap.mm_rhs[1].d.begin(), cap.mm_rhs[1].d.end(), Q);   // (C * A^-T) * Q
  std::copy(cap.mm_rhs[3].d.begin(), cap.mm_rhs[3].d.end(), Ct);  // (((C * A^-T) * Q) * A^-1) * Ct
  for (int a = 0; a < 3; ++a) std::copy(cap.mv_rhs[a].v.begin(), cap.mv_rhs[a].v.end(), D + a * nd);  // C * Dx, ...
}

// getTotalTime, getLength and evaluate(t[i], k) of waypointsTraj's result: out [n_t][3]
REF_API void ref_poly_query(int32_t S, const double* waypts, const double* sv, const double* ev, const double* sa,
                            const double* ea, const double* times, int32_t n_t, const double* t, int32_t k, double* out,
                            double* total_time, double* length) {
  PolynomialTraj traj;
  make_traj(S, waypts, sv, ev, sa, ea, times, traj);
  *total_time = traj.getTotalTime();
  *length = traj.getLength();
  for (int i = 0; i < n_t; ++i) {
    Eigen::Vector3d p = traj.evaluate(t[i], k);
    for (int j = 0; j < 3; ++j) out[3 * i + j] = p[j];
  }
}

// planExploreTraj :270-297 for one tour of W waypoints: times_out [W-1], points [max_k][3], derivs [4][3],
// out_d = {duration, length, dt}, out_i = {seg_num, K}
REF_API void ref_poly_explore(int32_t W, const double* tour, const double* cur_vel, const double* cur_acc, double max_vel,
                              double ctrl_pt_dist, int32_t min_seg_num, int32_t max_k, double* times_out, double* points,
                              double* derivs, double* out_d, int32_t* out_i) {
  const int pt_num = W;
  Eigen::MatrixXd pos(pt_num, 3);
  for (int i = 0; i < pt_num; ++i)
    for (int j = 0; j < 3; ++j) pos(i, j) = tour[3 * i + j];
  Eigen::Vector3d zero(0, 0, 0), cv(cur_vel[0], cur_vel[1], cur_vel[2]), ca(cur_acc[0], cur_acc[1], cur_acc[2]);
  Eigen::VectorXd times(pt_num - 1);
  for (int i = 0; i < pt_num - 1; ++i) {
    Eigen::Vector3d d(pos(i + 1, 0) - pos(i, 0), pos(i + 1, 1) - pos(i, 1), pos(i + 1, 2) - pos(i, 2));
    times(i) = d.norm() / (max_vel * 0.5);
  }
  PolynomialTraj init_traj;
  PolynomialTraj::waypointsTraj(pos, cv, zero, ca, zero, times, init_traj);
  std::vector<Eigen::Vector3d> pts, boundary_deri;
  double duration = init_traj.getTotalTime();
  int seg_num = init_traj.getLength() / ctrl_pt_dist;
  seg_num = std::max((int)min_seg_num, seg_num);
  double dt = duration / double(seg_num);
  for (double ts = 0.0; ts <= duration + 1e-4; ts += dt) pts.push_back(init_traj.evaluate(ts, 0));
  boundary_deri.push_back(init_traj.evaluate(0.0, 1));
  boundary_deri.push_back(init_traj.evaluate(duration, 1));
  boundary_deri.push_back(init_traj.evaluate(0.0, 2));
  boundary_deri.push_back(init_traj.evaluate(duration, 2));
  for (int i = 0; i < pt_num - 1; ++i) times_out[i] = times(i);
  for (int i = 0; i < (int)pts.size() && i < max_k; ++i)
    for (int j = 0; j < 3; ++j) points[3 * i + j] = pts[i][j];
  for (int i = 0; i < 4; ++i)
    for (int j = 0; j < 3; ++j) derivs[3 * i + j] = boundary_deri[i][j];
  out_d[0] = duration, out_d[1] = init_traj.length_, out_d[2] = dt;
  out_i[0] = seg_num, out_i[1] = (int32_t)pts.size();
}

}  // extern "C"
