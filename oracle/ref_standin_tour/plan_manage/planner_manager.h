// Stand-in for plan_manage/planner_manager.h: the members of FastPlannerManager that fast_exploration_manager.cpp
// touches.  The four methods are declared here and stubbed in oracle/ref_tour_wrap.cpp; refineLocalTour never calls
// them.  TEST INFRASTRUCTURE ONLY.
#pragma once
#include <memory>
#include <vector>

#include <Eigen/Eigen>
#include <path_searching/astar2.h>
#include <plan_env/edt_environment.h>
#include <ros/ros.h>

namespace fast_planner {
struct StandinTraj {
  double getTimeSum() const { return 0.0; }
};
struct StandinLocalData {
  StandinTraj position_traj_;
};
class FastPlannerManager {
public:
  void initPlanModules(ros::NodeHandle& nh);
  void planExploreTraj(const std::vector<Eigen::Vector3d>& tour, const Eigen::Vector3d& cur_vel,
                       const Eigen::Vector3d& cur_acc, const double& time_lb = -1);
  bool kinodynamicReplan(const Eigen::Vector3d& start_pt, const Eigen::Vector3d& start_vel,
                         const Eigen::Vector3d& start_acc, const Eigen::Vector3d& end_pt,
                         const Eigen::Vector3d& end_vel, const double& time_lb = -1);
  void planYawExplore(const Eigen::Vector3d& start_yaw, const double& end_yaw, bool lookfwd,
                      const double& relax_time);
  EDTEnvironment::Ptr edt_environment_;
  std::unique_ptr<Astar> path_finder_;
  StandinLocalData local_data_;
};
}  // namespace fast_planner
