// Restates FastPlannerManager::planYaw's lines 695-745 (plan_manage/src/planner_manager.cpp, the kinodynamic replan's
// yaw; a file that needs the whole planner to compile) and calcNextYaw (:867-885) over the reference's own
// NonUniformBspline (setUniformBspline, getTimeSum, evaluateDeBoorT, getDerivative; bspline/src/non_uniform_bspline.cpp
// compiled unmodified against oracle/ref_standin_traj + oracle/ref_standin by oracle/plan_yaw.mk), and records what
// BsplineOptimizer::optimize() then receives: seg_num, dt_yaw, the waypoints and their indices, the end velocity and yaw,
// the (seg_num + 3) x 1 initial guess and the pt_dist_ it freezes from it (bspline_optimizer.cpp:136-140).  Two
// liberties, both stated where they are taken: |pd| is summed (dx*dx + dy*dy) + dz*dz (Eigen's order is unpinned), and
// states2pts * v is summed left to right per row.
// TEST INFRASTRUCTURE ONLY; part of oracle/_ref/libfuel_ref_plan_yaw.so, built with hidden visibility: REF_API exports.
#include <bspline/non_uniform_bspline.h>
#include <math.h>
#include <stdint.h>

#include <algorithm>
#include <vector>

#define REF_API __attribute__((visibility("default")))

using fast_planner::NonUniformBspline;

static void calcNextYaw(const double& last_yaw, double& yaw) {
  double round_last = last_yaw;
  while (round_last < -M_PI) round_last += 2 * M_PI;
  while (round_last > M_PI) round_last -= 2 * M_PI;
  double diff = yaw - round_last;
  if (fabs(diff) <= M_PI) {
    yaw = last_yaw + diff;
  } else if (diff > M_PI) {
    yaw = last_yaw + diff - 2 * M_PI;
  } else if (diff < -M_PI) {
    yaw = last_yaw + diff + 2 * M_PI;
  }
}

extern "C" {

// ctrl [n][3] at knot span dt is the position trajectory; start_yaw [3] used as given (|start_yaw[0]| <= 1000 keeps
// calcNextYaw's loops short).  od = {duration, dt_yaw, atan2 of the end velocity, end yaw after calcNextYaw, pt_dist_,
// end velocity x, y, z}; oi = {seg_num, waypoint count}; wp [max_seg], widx [max_seg], guess [max_seg + 3].  Returns 0;
// -1 where the reference would read waypts.back() of an empty vector; -2 where seg_num > max_seg (nothing written).
REF_API int32_t ref_plan_yaw(int32_t n, const double* ctrl, double dt, const double* start_yaw, int32_t max_seg,
                             double* od, int32_t* oi, double* wp, int32_t* widx, double* guess) {
  Eigen::MatrixXd pts(n, 3);
  for (int i = 0; i < n; ++i)
    for (int j = 0; j < 3; ++j) pts(i, j) = ctrl[3 * i + j];
  NonUniformBspline pos;
  pos.setUniformBspline(pts, 3, dt);
  NonUniformBspline velocity_traj_ = pos.getDerivative();  // updateTrajInfo (:518-526)
  const double duration = pos.getTimeSum();

  double dt_yaw = 0.3;
  const double q = duration / dt_yaw;
  if (!(q <= max_seg)) return -2;  // (int) of a larger quotient may be undefined; the caller's buffers end here
  int seg_num = ceil(q);
  dt_yaw = duration / seg_num;

  const double forward_t = 2.0;
  double last_yaw = start_yaw[0];
  std::vector<double> waypts;
  std::vector<int> waypt_idx;
  for (int i = 0; i < seg_num; ++i) {
    double tc = i * dt_yaw;
    Eigen::VectorXd pc = pos.evaluateDeBoorT(tc);
    double tf = std::min(duration, tc + forward_t);
    Eigen::VectorXd pf = pos.evaluateDeBoorT(tf);
    const double dx = pf(0) - pc(0), dy = pf(1) - pc(1), dz = pf(2) - pc(2);
    double waypt;
    if (sqrt((dx * dx + dy * dy) + dz * dz) > 1e-6) {
      waypt = atan2(dy, dx);
      calcNextYaw(last_yaw, waypt);
    } else if (waypts.empty()) {
      return -1;
    } else {
      waypt = waypts.back();
    }
    last_yaw = waypt;
    waypts.push_back(waypt);
    waypt_idx.push_back(i);
  }

  std::vector<double> yaw(seg_num + 3, 0.0);
  const double states2pts[3][3] = {{1.0, -dt_yaw, (1 / 3.0) * dt_yaw * dt_yaw},
                                   {1.0, 0.0, -(1 / 6.0) * dt_yaw * dt_yaw},
                                   {1.0, dt_yaw, (1 / 3.0) * dt_yaw * dt_yaw}};
  for (int r = 0; r < 3; ++r)
    yaw[r] = (states2pts[r][0] * start_yaw[0] + states2pts[r][1] * start_yaw[1]) + states2pts[r][2] * start_yaw[2];
  Eigen::VectorXd end_v = velocity_traj_.evaluateDeBoorT(duration - 0.1);
  const double end_raw = atan2(end_v(1), end_v(0));
  double end_yaw = end_raw;
  calcNextYaw(last_yaw, end_yaw);
  for (int r = 0; r < 3; ++r)  // written after the start block: for seg_num 1 and 2 the blocks overlap
    yaw[seg_num + r] = (states2pts[r][0] * end_yaw + states2pts[r][1] * 0.0) + states2pts[r][2] * 0.0;

  double pt_dist_ = 0.0;  // optimize() on the (seg_num + 3) x 1 matrix: row differences of one column
  for (int i = 0; i < seg_num + 2; ++i) {
    const double d = yaw[i + 1] - yaw[i];
    pt_dist_ += sqrt(d * d);
  }
  pt_dist_ /= double(seg_num + 3);

  od[0] = duration;
  od[1] = dt_yaw;
  od[2] = end_raw;
  od[3] = end_yaw;
  od[4] = pt_dist_;
  for (int j = 0; j < 3; ++j) od[5 + j] = end_v(j);
  oi[0] = seg_num;
  oi[1] = (int32_t)waypts.size();
  for (size_t k = 0; k < waypts.size(); ++k) wp[k] = waypts[k], widx[k] = waypt_idx[k];
  for (int i = 0; i < seg_num + 3; ++i) guess[i] = yaw[i];
  return 0;
}

}  // extern "C"
