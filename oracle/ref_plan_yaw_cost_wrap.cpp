// Drives the reference's own BsplineOptimizer (bspline_opt/src/bspline_optimizer.cpp, compiled unmodified into
// oracle/_ref/libfuel_ref.so by oracle/Makefile) with a one-column control-point matrix the way planYaw calls it
// (plan_manage/src/planner_manager.cpp:747-760): setWaypoints, setBoundaryStates with the start yaw as given and three
// end states, then optimize(yaw, dt_yaw, SMOOTHNESS | WAYPOINTS | START | END, 1, 1).  The NLopt stand-in
// (ref_standin/nlopt.hpp) evaluates costFunction -> combineCost with dim_ == 1 at the initial guess and at the probe
// points.  Compiled with the same stand-ins and default visibility, and linked against _ref/libfuel_ref.so, so the
// optimizer and the stand-in's recorder are that library's.
// TEST INFRASTRUCTURE ONLY; part of oracle/_ref/libfuel_ref_plan_yaw.so.
#include <bspline_opt/bspline_optimizer.h>
#include <nlopt.hpp>
#include <stdint.h>
#include <string.h>

using namespace fast_planner;

extern "C" {

void* ref_opt_create(void* sdf_map_handle, int32_t n, const char** keys, const double* values);  // ref_bspline_wrap.cpp
void ref_opt_destroy(void* h);

// n = seg_num + 3 control points: guess [n], start = start_yaw (yaw, yawdot, yawddot), end_yaw after calcNextYaw (its
// rate and acceleration 0), waypoints wp [n_wp] at widx; probes [n_probe][n] -> f [1 + n_probe], grad [1 + n_probe][n].
// Returns 0, or -1 if the objective was not evaluated 1 + n_probe times.
int32_t ref_plan_yaw_cost(void* sdf_map_handle, int32_t n_keys, const char** keys, const double* values, int32_t n,
                          const double* guess, double dt_yaw, const double* start, double end_yaw, int32_t n_wp,
                          const double* wp, const int32_t* widx, int32_t n_probe, const double* probes, double* f,
                          double* grad) {
  BsplineOptimizer* o = (BsplineOptimizer*)ref_opt_create(sdf_map_handle, n_keys, keys, values);
  std::vector<Eigen::Vector3d> waypts;
  for (int i = 0; i < n_wp; ++i) waypts.emplace_back(wp[i], 0, 0);
  o->setWaypoints(waypts, std::vector<int>(widx, widx + n_wp));
  std::vector<Eigen::Vector3d> st = {Eigen::Vector3d(start[0], 0, 0), Eigen::Vector3d(start[1], 0, 0),
                                     Eigen::Vector3d(start[2], 0, 0)};
  std::vector<Eigen::Vector3d> en = {Eigen::Vector3d(end_yaw, 0, 0), Eigen::Vector3d(0, 0, 0),
                                     Eigen::Vector3d(0, 0, 0)};
  o->setBoundaryStates(st, en);
  Eigen::MatrixXd yaw(n, 1);
  for (int i = 0; i < n; ++i) yaw(i, 0) = guess[i];
  nlopt::Recorder& r = nlopt::recorder();
  r.probes.clear();
  for (int p = 0; p < n_probe; ++p) r.probes.emplace_back(probes + (size_t)p * n, probes + (size_t)(p + 1) * n);
  double dt = dt_yaw;
  const int cost_func = BsplineOptimizer::SMOOTHNESS | BsplineOptimizer::WAYPOINTS | BsplineOptimizer::START |
                        BsplineOptimizer::END;
  o->optimize(yaw, dt, cost_func, 1, 1);
  int32_t rc = (int)r.f.size() == 1 + n_probe ? 0 : -1;
  for (int p = 0; rc == 0 && p <= n_probe; ++p) {
    f[p] = r.f[p];
    memcpy(grad + (size_t)p * n, r.grad[p].data(), sizeof(double) * n);
  }
  ref_opt_destroy(o);
  return rc;
}

}  // extern "C"
