// Drives the reference's own FastExplorationManager::findGlobalTour (exploration_manager/src/
// fast_exploration_manager.cpp:327-427), compiled unmodified into oracle/_ref/libfuel_ref_gtour.so (oracle/gtour.mk)
// with frontier_finder.cpp, graph_node.cpp, perception_utils.cpp, astar2.cpp and the real LKH (utils/lkh_tsp_solver:
// its src/*.c and lkh_interface.cpp), over the SDFMap and RayCaster of oracle/_ref/libfuel_ref.so.  findGlobalTour
// writes the TSPLIB file, runs LKH, parses its tour and calls getPathForTour, all as the reference does; ViewNode's
// statics are set as FastExplorationManager::initialize sets them (:55-69) and single.par holds its four lines
// (:76-80).  TEST INFRASTRUCTURE ONLY.
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <unistd.h>

#include <fstream>
#include <list>
#include <memory>
#include <string>
#include <vector>

#include <plan_env/edt_environment.h>
#include <plan_env/raycast.h>
#include <plan_env/sdf_map.h>
#include <plan_manage/planner_manager.h>
// findGlobalTour and the frontier list are private: this translation unit -- the test wrapper, not the reference
// sources -- calls and installs them
#define private public
#include <path_searching/astar2.h>
#include <active_perception/frontier_finder.h>
#include <exploration_manager/fast_exploration_manager.h>
#undef private
#include <active_perception/graph_node.h>
#include <exploration_manager/expl_data.h>

using namespace fast_planner;
using Eigen::Vector3d;

#define API extern "C" __attribute__((visibility("default")))

// what fast_exploration_manager.cpp links against beyond findGlobalTour: never called here
namespace fast_planner {
void FastPlannerManager::initPlanModules(ros::NodeHandle&) {}
void FastPlannerManager::planExploreTraj(const std::vector<Vector3d>&, const Vector3d&, const Vector3d&,
                                         const double&) {}
bool FastPlannerManager::kinodynamicReplan(const Vector3d&, const Vector3d&, const Vector3d&, const Vector3d&,
                                           const Vector3d&, const double&) {
  return false;
}
void FastPlannerManager::planYawExplore(const Vector3d&, const double&, bool, const double&) {}
}  // namespace fast_planner

namespace {
EDTEnvironment::Ptr g_env;
FastExplorationManager* g_mgr = nullptr;
std::string g_dir;
Vector3d v3(const double* p) { return Vector3d(p[0], p[1], p[2]); }
}  // namespace

// ViewNode's statics (astar/* parameters, max_search_time on the tick clock), a FrontierFinder, and ep_->tsp_dir_ =
// a fresh temporary directory holding single.par
API int32_t ref_gtour_setup(void* sdf_map_handle, double vm, double yd, double w_dir, double lambda,
                            int32_t allocate_num, double max_search_time) {
  g_env.reset(new EDTEnvironment);
  g_env->sdf_map_ = std::shared_ptr<SDFMap>((SDFMap*)sdf_map_handle, [](SDFMap*) {});
  ros::NodeHandle nh;
  nh.values["astar/resolution_astar"] = 0.4;
  nh.values["astar/lambda_heu"] = lambda;
  nh.values["astar/max_search_time"] = max_search_time;
  nh.values["astar/allocate_num"] = allocate_num;
  ViewNode::vm_ = vm;
  ViewNode::yd_ = yd;
  ViewNode::w_dir_ = w_dir;
  ViewNode::astar_.reset(new Astar);
  ViewNode::astar_->init(nh, g_env);
  Vector3d origin, size;
  g_env->sdf_map_->getRegion(origin, size);
  ViewNode::caster_.reset(new RayCaster);
  ViewNode::caster_->setParams(g_env->sdf_map_->getResolution(), origin);
  ViewNode::map_ = g_env->sdf_map_;
  g_mgr = new FastExplorationManager;
  g_mgr->ed_.reset(new ExplorationData);
  g_mgr->ep_.reset(new ExplorationParam);
  g_mgr->frontier_finder_.reset(new FrontierFinder(g_env, nh));
  char tmpl[] = "/tmp/fuel_ref_gtour_XXXXXX";
  if (!mkdtemp(tmpl)) return -1;
  g_dir = tmpl;
  g_mgr->ep_->tsp_dir_ = g_dir;
  std::ofstream par_file(g_mgr->ep_->tsp_dir_ + "/single.par");  // :76-80
  par_file << "PROBLEM_FILE = " << g_mgr->ep_->tsp_dir_ << "/single.tsp\n";
  par_file << "GAIN23 = NO\n";
  par_file << "OUTPUT_TOUR_FILE =" << g_mgr->ep_->tsp_dir_ << "/single.txt\n";
  par_file << "RUNS = 1\n";
  return 0;
}

API void ref_gtour_teardown() {
  delete g_mgr;  // ViewNode::astar_.reset(), caster_.reset(), map_.reset()
  g_mgr = nullptr;
  g_env.reset();
  for (const char* f : { "/single.par", "/single.tsp", "/single.txt" }) remove((g_dir + f).c_str());
  rmdir(g_dir.c_str());
}

// The frontier list: n clusters, each with one viewpoint (vp_pos, vp_yaw), its costs_ row (costs [n][n]) and its
// paths_ (paths_n [n][n] points each, the points in order in paths); all costed already (first_new_ftr_ = end).
// Then findGlobalTour(cur_pos, cur_vel, cur_yaw) -> indices [n] (returns their count), ed_->global_tour_ (its first
// tour_max rows, *n_tour of them), and getFullCostMatrix's matrix [(n + 1)^2] for the same state.
API int32_t ref_gtour_find(int32_t n, const double* vp_pos, const double* vp_yaw, const double* costs,
                           const int32_t* paths_n, const double* paths, const double cur_pos[3],
                           const double cur_vel[3], const double cur_yaw[3], int32_t* indices, int32_t tour_max,
                           int32_t* n_tour, double* tour, double* mat) {
  FrontierFinder& ff = *g_mgr->frontier_finder_;
  ff.frontiers_.clear();
  ff.removed_ids_.clear();
  for (int i = 0, k = 0; i < n; ++i) {
    Frontier f;
    f.id_ = i;
    Viewpoint v;
    v.pos_ = v3(vp_pos + 3 * i);
    v.yaw_ = vp_yaw[i];
    v.visib_num_ = 1;
    f.viewpoints_.push_back(v);
    for (int j = 0; j < n; ++j) {
      f.costs_.push_back(costs[i * n + j]);
      std::vector<Vector3d> p;
      for (int q = 0; q < paths_n[i * n + j]; ++q, ++k) p.push_back(v3(paths + 3 * k));
      f.paths_.push_back(p);
    }
    ff.frontiers_.push_back(f);
  }
  ff.first_new_ftr_ = ff.frontiers_.end();
  g_mgr->ed_->global_tour_.clear();
  std::vector<int> ids;
  g_mgr->findGlobalTour(v3(cur_pos), v3(cur_vel), v3(cur_yaw), ids);
  for (size_t i = 0; i < ids.size() && i < (size_t)n; ++i) indices[i] = ids[i];
  const auto& t = g_mgr->ed_->global_tour_;
  *n_tour = (int32_t)t.size();
  for (int i = 0; i < tour_max && i < (int)t.size(); ++i)
    for (int c = 0; c < 3; ++c) tour[3 * i + c] = t[i](c);
  Eigen::MatrixXd m;
  ff.getFullCostMatrix(v3(cur_pos), v3(cur_vel), v3(cur_yaw), m);
  for (int i = 0; i <= n; ++i)
    for (int j = 0; j <= n; ++j) mat[i * (n + 1) + j] = m(i, j);
  return (int32_t)ids.size();
}

// getPathForTour over the installed list for the given indices (the rows of the tour, as above)
API void ref_gtour_path(const double cur_pos[3], int32_t n, const int32_t* ids, int32_t tour_max, int32_t* n_tour,
                        double* tour) {
  std::vector<Vector3d> t;
  g_mgr->frontier_finder_->getPathForTour(v3(cur_pos), std::vector<int>(ids, ids + n), t);
  *n_tour = (int32_t)t.size();
  for (int i = 0; i < tour_max && i < (int)t.size(); ++i)
    for (int c = 0; c < 3; ++c) tour[3 * i + c] = t[i](c);
}
