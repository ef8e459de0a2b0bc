// Drives the reference's own FastExplorationManager::refineLocalTour (exploration_manager/src/
// fast_exploration_manager.cpp:429-503) and FrontierFinder::getViewpointsInfo / getTopViewpointsInfo
// (active_perception/src/frontier_finder.cpp:425-484), compiled unmodified with graph_node.cpp, perception_utils.cpp and
// astar2.cpp into oracle/_ref/libfuel_ref_tour.so (oracle/tour.mk), over the SDFMap and RayCaster of
// oracle/_ref/libfuel_ref.so.  ViewNode's statics are set as FastExplorationManager::initialize sets them (:55-69).
// The refined-id selection (:139-147) and the one-viewpoint pick (:202-214) sit inside planExploreMotion, which needs
// the whole planner; they are restated here, line for line, over the compiled ViewNode::computeCost.
// TEST INFRASTRUCTURE ONLY.
#include <stdint.h>
#include <string.h>

#include <algorithm>
#include <list>
#include <memory>
#include <vector>

#include <plan_env/edt_environment.h>
#include <plan_env/raycast.h>
#include <plan_env/sdf_map.h>
#include <plan_manage/planner_manager.h>
// refineLocalTour, the frontier list and min_candidate_dist_ are private: this translation unit -- the test wrapper,
// not the reference sources -- calls and installs them
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

// what fast_exploration_manager.cpp links against beyond the local tour: never called here
int solveTSPLKH(const char*) { return -1; }
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
// its constructor does nothing and refineLocalTour reads only ViewNode's statics and ed_; its destructor resets the
// statics (:30-34), so it lives from setup to teardown
FastExplorationManager* g_mgr = nullptr;
Vector3d v3(const double* p) { return Vector3d(p[0], p[1], p[2]); }
void put(const Vector3d& v, double* out) {
  for (int k = 0; k < 3; ++k) out[k] = v(k);
}
}  // namespace

// ViewNode::vm_, yd_, w_dir_, astar_ (astar/* parameters, max_search_time on the tick clock), caster_, map_
API void ref_tour_setup(void* sdf_map_handle, double vm, double yd, double w_dir, double lambda, int32_t allocate_num,
                        double max_search_time) {
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
}

API void ref_tour_teardown() {
  delete g_mgr;  // ViewNode::astar_.reset(), caster_.reset(), map_.reset()
  g_mgr = nullptr;
  g_env.reset();
}

// refineLocalTour over ng groups of gsize[i] viewpoints: refined points and yaws ([kmax] rows, *n_refined of them),
// ed_->refined_tour_ (its first tour_max rows, *n_tour of them) and ViewNode::astar_->lambda_heu_ afterwards
API void ref_tour_refine(const double cur_pos[3], const double cur_vel[3], const double cur_yaw[3], int32_t ng,
                         const int32_t* gsize, const double* vp_pos, const double* vp_yaw, int32_t kmax,
                         int32_t* n_refined, double* refined_pos, double* refined_yaw, int32_t tour_max,
                         int32_t* n_tour, double* tour, double* lambda_after) {
  std::vector<std::vector<Vector3d>> n_points(ng);
  std::vector<std::vector<double>> n_yaws(ng);
  for (int i = 0, k = 0; i < ng; ++i)
    for (int j = 0; j < gsize[i]; ++j, ++k) n_points[i].push_back(v3(vp_pos + 3 * k)), n_yaws[i].push_back(vp_yaw[k]);
  FastExplorationManager& mgr = *g_mgr;
  mgr.ed_.reset(new ExplorationData);
  std::vector<Vector3d> pts;
  std::vector<double> ys;
  mgr.refineLocalTour(v3(cur_pos), v3(cur_vel), v3(cur_yaw), n_points, n_yaws, pts, ys);
  *n_refined = (int32_t)pts.size();
  for (int i = 0; i < kmax && i < (int)pts.size(); ++i) put(pts[i], refined_pos + 3 * i), refined_yaw[i] = ys[i];
  const auto& t = mgr.ed_->refined_tour_;
  *n_tour = (int32_t)t.size();
  for (int i = 0; i < tour_max && i < (int)t.size(); ++i) put(t[i], tour + 3 * i);
  *lambda_after = ViewNode::astar_->lambda_heu_;
}

// A frontier list of n clusters (nv[i] viewpoints each: pos, yaw, visib_num_; id_ = ids[i]) with min_candidate_dist_,
// then getViewpointsInfo (the rows of each returned group: counts[], pos, yaw) and getTopViewpointsInfo (top_pos,
// top_yaw [n]).  Returns the number of groups getViewpointsInfo returned.
API int32_t ref_tour_viewpoints(int32_t n, const int32_t* fids, const int32_t* nv, const double* pos, const double* yaw,
                                const int32_t* visib, double min_dist, const double cur_pos[3], int32_t n_ids,
                                const int32_t* ids, int32_t view_num, double max_decay, int32_t* counts,
                                double* out_pos, double* out_yaw, double* top_pos, double* top_yaw) {
  ros::NodeHandle nh;
  FrontierFinder ff(g_env, nh);
  ff.min_candidate_dist_ = min_dist;
  for (int i = 0, k = 0; i < n; ++i) {
    Frontier f;
    f.id_ = fids[i];
    f.average_ = Vector3d(0, 0, 0);
    for (int j = 0; j < nv[i]; ++j, ++k) {
      Viewpoint v;
      v.pos_ = v3(pos + 3 * k);
      v.yaw_ = yaw[k];
      v.visib_num_ = visib[k];
      f.viewpoints_.push_back(v);
    }
    ff.frontiers_.push_back(f);
  }
  std::vector<std::vector<Vector3d>> points;
  std::vector<std::vector<double>> yaws;
  ff.getViewpointsInfo(v3(cur_pos), std::vector<int>(ids, ids + n_ids), view_num, max_decay, points, yaws);
  int r = 0;
  for (size_t g = 0; g < points.size(); ++g) {
    counts[g] = (int32_t)points[g].size();
    for (size_t j = 0; j < points[g].size(); ++j, ++r) put(points[g][j], out_pos + 3 * r), out_yaw[r] = yaws[g][j];
  }
  std::vector<Vector3d> tp, av;
  std::vector<double> ty;
  ff.getTopViewpointsInfo(v3(cur_pos), tp, ty, av);
  for (size_t i = 0; i < tp.size(); ++i) put(tp[i], top_pos + 3 * i), top_yaw[i] = ty[i];
  return (int32_t)points.size();
}

// planExploreMotion :139-147: the refined ids of the tour `indices` over the top viewpoints `points`
API int32_t ref_tour_select_ids(const double* points, int32_t n_idx, const int32_t* indices, const double pos[3],
                                int32_t refined_num, double refined_radius, int32_t* out_ids) {
  std::vector<int> refined_ids;
  std::vector<Vector3d> unrefined_points;
  int knum = std::min(int(n_idx), refined_num);
  for (int i = 0; i < knum; ++i) {
    auto tmp = v3(points + 3 * indices[i]);
    unrefined_points.push_back(tmp);
    refined_ids.push_back(indices[i]);
    if ((tmp - v3(pos)).norm() > refined_radius && refined_ids.size() >= 2) break;
  }
  for (size_t i = 0; i < refined_ids.size(); ++i) out_ids[i] = refined_ids[i];
  return (int32_t)refined_ids.size();
}

// planExploreMotion :202-214: the index of the min-cost viewpoint (-1 where the reference indexes out of range)
API int32_t ref_tour_pick(const double pos[3], const double vel[3], const double yaw[3], int32_t n, const double* pts,
                          const double* yaws) {
  double min_cost = 100000;
  int min_cost_id = -1;
  std::vector<Vector3d> tmp_path;
  for (int i = 0; i < n; ++i) {
    auto tmp_cost = ViewNode::computeCost(v3(pos), v3(pts + 3 * i), yaw[0], yaws[i], v3(vel), yaw[1], tmp_path);
    if (tmp_cost < min_cost) {
      min_cost = tmp_cost;
      min_cost_id = i;
    }
  }
  return min_cost_id;
}
