// Drives the reference's own NonUniformBspline::parameterizeToBspline and getBoundaryStates
// (bspline/src/non_uniform_bspline.cpp:108-123, 178-265, compiled unmodified from /root/reference against
// oracle/ref_standin_param + oracle/ref_standin_traj + oracle/ref_standin by oracle/param.mk) so tests can compare the
// oracle's parameterization with the real code.  The Eigen stand-in records the system parameterizeToBspline builds and
// solves it with the oracle's orc_lstsq_colpiv_qr (Eigen's QR is third-party: "parity unpinned").
// TEST INFRASTRUCTURE ONLY; part of oracle/_ref/libfuel_ref_param.so, built with hidden visibility: REF_API exports.
#include <bspline/non_uniform_bspline.h>
#include <stdint.h>

#define REF_API __attribute__((visibility("default")))

using fast_planner::NonUniformBspline;

static NonUniformBspline make_traj(int32_t n, const double* ctrl, double dt) {
  Eigen::MatrixXd pts(n, 3);
  for (int i = 0; i < n; ++i)
    for (int j = 0; j < 3; ++j) pts(i, j) = ctrl[3 * i + j];
  NonUniformBspline traj;
  traj.setUniformBspline(pts, 3, dt);  // bspline_degree_ = 3 in every launch file
  return traj;
}

extern "C" {

// NonUniformBspline::parameterizeToBspline(ts, point_set, start_end_derivative, 3, ctrl_pts) (:178-265): points [K][3],
// derivs [4][3] (start vel, end vel, start acc, end acc) -> ctrl [K+2][3], and the A [K+4][K+2] and b [3][K+4] it built,
// as the Eigen stand-in recorded them (its solve is the oracle's orc_lstsq_colpiv_qr).  Returns the number of solves.
REF_API int32_t ref_param_parameterize(double ts, int32_t K, const double* points, const double* derivs, double* ctrl,
                                      double* A, double* b) {
  std::vector<Eigen::Vector3d> point_set, start_end_derivative;
  for (int i = 0; i < K; ++i) point_set.push_back(Eigen::Vector3d(points[3 * i], points[3 * i + 1], points[3 * i + 2]));
  for (int i = 0; i < 4; ++i)
    start_end_derivative.push_back(Eigen::Vector3d(derivs[3 * i], derivs[3 * i + 1], derivs[3 * i + 2]));
  Eigen::ParamCapture& cap = Eigen::param_capture();
  cap = Eigen::ParamCapture();
  Eigen::MatrixXd ctrl_pts;
  NonUniformBspline::parameterizeToBspline(ts, point_set, start_end_derivative, 3, ctrl_pts);
  for (int i = 0; i < ctrl_pts.rows(); ++i)
    for (int j = 0; j < 3; ++j) ctrl[3 * i + j] = ctrl_pts(i, j);
  for (size_t i = 0; i < cap.A.size(); ++i) A[i] = cap.A[i];
  for (int j = 0; j < 3 && j < cap.n_b; ++j)
    for (size_t i = 0; i < cap.b[j].size(); ++i) b[j * cap.b[j].size() + i] = cap.b[j][i];
  return cap.n_b;
}

// getBoundaryStates(2, 0, start, end) (:108-123) of setUniformBspline(ctrl, 3, dt): start [3][3], end [3]
REF_API void ref_param_boundary_states(int32_t n, const double* ctrl, double dt, double* start, double* end) {
  NonUniformBspline traj = make_traj(n, ctrl, dt);
  std::vector<Eigen::Vector3d> s, e;
  traj.getBoundaryStates(2, 0, s, e);
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) start[3 * i + j] = s[i](j);
  for (int j = 0; j < 3; ++j) end[j] = e[0](j);
}

}  // extern "C"
