// Drives the reference's own NonUniformBspline (bspline/src/non_uniform_bspline.cpp, compiled unmodified from
// /root/reference against oracle/ref_standin_traj + oracle/ref_standin by oracle/traj.mk) so tests can compare the
// oracle's trajectory checks with the real code:
// evaluateDeBoorT, getDerivative, getTimeSum, getJerk, setPhysicalLimits, checkFeasibility, checkRatio.
// FastPlannerManager::checkTrajCollision (plan_manage/src/planner_manager.cpp:96-118) lives in a file that needs the
// whole planner to compile; its 20-line loop is restated below over the reference's own evaluateDeBoorT and
// SDFMap::getInflateOccupancy, with t_now passed in instead of read from ros::Time.
// The SDFMap is the one oracle/_ref/libfuel_ref.so creates (oracle.RefSDFMap); only its inline accessors are used here.
// TEST INFRASTRUCTURE ONLY; part of oracle/_ref/libfuel_ref_traj.so, built with hidden visibility: REF_API exports.
#include <bspline/non_uniform_bspline.h>
#include <plan_env/sdf_map.h>
#include <stdint.h>

#define REF_API __attribute__((visibility("default")))

using fast_planner::NonUniformBspline;
using fast_planner::SDFMap;

static NonUniformBspline make_traj(int32_t n, const double* ctrl, double dt) {
  Eigen::MatrixXd pts(n, 3);
  for (int i = 0; i < n; ++i)
    for (int j = 0; j < 3; ++j) pts(i, j) = ctrl[3 * i + j];
  NonUniformBspline traj;
  traj.setUniformBspline(pts, 3, dt);  // bspline_degree_ = 3 in every launch file
  return traj;
}

extern "C" {

// evaluateDeBoorT of the spline after `deriv` getDerivative() calls: ctrl [n][3], t [n_t] -> out [n_t][3]
REF_API void ref_traj_evaluate(int32_t n, const double* ctrl, double dt, int32_t deriv, int32_t n_t, const double* t,
                               double* out) {
  NonUniformBspline traj = make_traj(n, ctrl, dt);
  for (int k = 0; k < deriv; ++k) traj = traj.getDerivative();
  for (int q = 0; q < n_t; ++q) {
    Eigen::VectorXd v = traj.evaluateDeBoorT(t[q]);
    for (int j = 0; j < 3; ++j) out[3 * q + j] = v(j);
  }
}

// out = { getTimeSum, getJerk, checkRatio }, *feasible = checkFeasibility(false), after setPhysicalLimits
REF_API void ref_traj_stats(int32_t n, const double* ctrl, double dt, double max_vel, double max_acc, double out[3],
                            int32_t* feasible) {
  NonUniformBspline traj = make_traj(n, ctrl, dt);
  traj.setPhysicalLimits(max_vel, max_acc);
  out[0] = traj.getTimeSum();
  out[1] = traj.getJerk();
  out[2] = traj.checkRatio();
  *feasible = traj.checkFeasibility(false) ? 1 : 0;
}

// checkTrajCollision (planner_manager.cpp:96-118): returns its verdict, writes `distance` only when it does, and counts
// the samples evaluated.  local_data_.duration_ = position_traj_.getTimeSum() (:523).
REF_API int32_t ref_traj_check_collision(void* sdf_map_handle, int32_t n, const double* ctrl, double dt, double t_now,
                                         double* distance, int32_t* n_checked) {
  SDFMap* sdf_map_ = (SDFMap*)sdf_map_handle;
  NonUniformBspline position_traj_ = make_traj(n, ctrl, dt);
  const double duration_ = position_traj_.getTimeSum();
  *n_checked = 0;

  Eigen::Vector3d cur_pt = position_traj_.evaluateDeBoorT(t_now);
  double radius = 0.0;
  Eigen::Vector3d fut_pt;
  double fut_t = 0.02;

  while (radius < 6.0 && t_now + fut_t < duration_) {
    fut_pt = position_traj_.evaluateDeBoorT(t_now + fut_t);
    ++*n_checked;
    if (sdf_map_->getInflateOccupancy(fut_pt) == 1) {
      *distance = radius;
      return 0;
    }
    radius = (fut_pt - cur_pt).norm();
    fut_t += 0.02;
  }
  return 1;
}

// selectBestTraj (planner_manager.cpp:476-482) over getJerk: the index std::sort puts first
REF_API int32_t ref_traj_select_best(int32_t B, int32_t n, const double* ctrl, const double* dt) {
  std::vector<std::pair<NonUniformBspline, int>> trajs;
  for (int b = 0; b < B; ++b) trajs.emplace_back(make_traj(n, ctrl + (size_t)b * n * 3, dt[b]), b);
  std::sort(trajs.begin(), trajs.end(), [](std::pair<NonUniformBspline, int>& tj1, std::pair<NonUniformBspline, int>& tj2) {
    return tj1.first.getJerk() < tj2.first.getJerk();
  });
  return B > 0 ? trajs[0].second : -1;
}

}  // extern "C"
