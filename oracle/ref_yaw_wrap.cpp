// Restates FastPlannerManager::planYawExplore's lines 776-824 (plan_manage/src/planner_manager.cpp, a file that needs
// the whole planner to compile) and calcNextYaw (:867-885) over the reference's own NonUniformBspline (setUniformBspline,
// getTimeSum, evaluateDeBoorT; bspline/src/non_uniform_bspline.cpp compiled unmodified from /root/reference against
// oracle/ref_standin_traj + oracle/ref_standin by oracle/yaw.mk), and records what BsplineOptimizer::optimize() then
// receives: dt_yaw, relax_num, the waypoints and waypt_idx, the initial guess, and the pt_dist_ it freezes from that
// guess (bspline_optimizer.cpp:136-140).  Two liberties, both stated where they are taken: |pd| is summed
// (dx*dx + dy*dy) + dz*dz (Eigen's order is unpinned), and states2pts * v is summed left to right per row.
// TEST INFRASTRUCTURE ONLY; part of oracle/_ref/libfuel_ref_yaw.so, built with hidden visibility: REF_API exports.
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

// ctrl [n][3] at knot span dt is the position trajectory; start_yaw [3]; the caller keeps |start_yaw[0]| <= 1000 and
// relax_time / dt_yaw < 2^31 (where the reference is undefined).
// od = {dt_yaw, end yaw after calcNextYaw, pt_dist_, start_yaw3d[0] wrapped}; oi = {relax_num, waypoint count};
// wp [11], widx [11], guess [15].  Returns 0, or -1 where the reference would read waypts.back() of an empty vector.
REF_API int32_t ref_yaw_explore(int32_t n, const double* ctrl, double dt, const double* start_yaw, double end_yaw,
                                int32_t lookfwd, double relax_time, double* od, int32_t* oi, double* wp, int32_t* widx,
                                double* guess) {
  Eigen::MatrixXd pts(n, 3);
  for (int i = 0; i < n; ++i)
    for (int j = 0; j < 3; ++j) pts(i, j) = ctrl[3 * i + j];
  NonUniformBspline position_traj_;
  position_traj_.setUniformBspline(pts, 3, dt);
  const double duration_ = position_traj_.getTimeSum();  // updateTrajInfo (:518-526)

  const int seg_num = 12;
  double dt_yaw = duration_ / seg_num;
  double start_yaw3d[3] = {start_yaw[0], start_yaw[1], start_yaw[2]};
  while (start_yaw3d[0] < -M_PI) start_yaw3d[0] += 2 * M_PI;
  while (start_yaw3d[0] > M_PI) start_yaw3d[0] -= 2 * M_PI;
  double last_yaw = start_yaw3d[0];

  std::vector<double> yaw(seg_num + 3, 0.0);
  const double states2pts[3][3] = {{1.0, -dt_yaw, (1 / 3.0) * dt_yaw * dt_yaw},
                                   {1.0, 0.0, -(1 / 6.0) * dt_yaw * dt_yaw},
                                   {1.0, dt_yaw, (1 / 3.0) * dt_yaw * dt_yaw}};
  for (int r = 0; r < 3; ++r)
    yaw[r] = (states2pts[r][0] * start_yaw3d[0] + states2pts[r][1] * start_yaw3d[1]) + states2pts[r][2] * start_yaw3d[2];

  std::vector<double> waypts;
  std::vector<int> waypt_idx;
  int relax_num = -1;
  if (lookfwd) {
    const double forward_t = 2.0;
    relax_num = relax_time / dt_yaw;
    for (int i = 1; i < seg_num - relax_num; ++i) {
      double tc = i * dt_yaw;
      Eigen::VectorXd pc = position_traj_.evaluateDeBoorT(tc);
      double tf = std::min(duration_, tc + forward_t);
      Eigen::VectorXd pf = position_traj_.evaluateDeBoorT(tf);
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
  }
  double end_yaw3d = end_yaw;
  calcNextYaw(last_yaw, end_yaw3d);
  for (int r = 0; r < 3; ++r)
    yaw[seg_num + r] = (states2pts[r][0] * end_yaw3d + states2pts[r][1] * 0.0) + states2pts[r][2] * 0.0;

  double pt_dist_ = 0.0;  // optimize() on the (seg_num + 3) x 1 matrix: row differences of one column
  for (int i = 0; i < seg_num + 2; ++i) {
    const double d = yaw[i + 1] - yaw[i];
    pt_dist_ += sqrt(d * d);
  }
  pt_dist_ /= double(seg_num + 3);

  od[0] = dt_yaw;
  od[1] = end_yaw3d;
  od[2] = pt_dist_;
  od[3] = start_yaw3d[0];
  oi[0] = relax_num;
  oi[1] = (int32_t)waypts.size();
  for (size_t k = 0; k < waypts.size(); ++k) wp[k] = waypts[k], widx[k] = waypt_idx[k];
  for (int i = 0; i < seg_num + 3; ++i) guess[i] = yaw[i];
  return 0;
}

}  // extern "C"
