// Drives the reference's own ViewNode::searchPath / computeCost (active_perception/src/graph_node.cpp) and the cost
// bookkeeping of FrontierFinder (updateFrontierCostMatrix, getFullCostMatrix, getPathForTour in
// active_perception/src/frontier_finder.cpp), both compiled unmodified with the reference's astar2.cpp into
// oracle/_ref/libfuel_ref_view.so (oracle/view.mk), over the SDFMap and RayCaster of oracle/_ref/libfuel_ref.so.
// ViewNode's statics are set as FastExplorationManager::initialize sets them (fast_exploration_manager.cpp:55-69).
// TEST INFRASTRUCTURE ONLY.
#include <stdint.h>
#include <string.h>

#include <list>
#include <memory>
#include <vector>

#include <plan_env/edt_environment.h>
#include <plan_env/raycast.h>
#include <plan_env/sdf_map.h>
// the search's counters and the frontier list are private: this translation unit -- the test wrapper, not the
// reference sources -- reads and installs them
#define private public
#include <path_searching/astar2.h>
#include <active_perception/frontier_finder.h>
#undef private
#include <active_perception/graph_node.h>

using namespace fast_planner;
using Eigen::Vector3d;

#define API extern "C" __attribute__((visibility("default")))

namespace {
// the layout of FuelViewCostInfo (include/fuelgpu.h)
struct Info {
  int32_t kind, reason, iter_num, use_node_num, n_path, reserved;
  double length, cost;
};
EDTEnvironment::Ptr g_env;

void put_path(const std::vector<Vector3d>& p, int32_t path_max, double* out) {
  memset(out, 0, sizeof(double) * 3 * (size_t)path_max);
  for (int i = 0; i < path_max && i < (int)p.size(); ++i)
    for (int k = 0; k < 3; ++k) out[3 * i + k] = p[i](k);
}
Vector3d v3(const double* p) { return Vector3d(p[0], p[1], p[2]); }
}  // namespace

// ViewNode::vm_, yd_, w_dir_, astar_ (astar/* parameters, max_search_time on the tick clock), caster_, map_
API void ref_view_setup(void* sdf_map_handle, double vm, double yd, double w_dir, double lambda, int32_t allocate_num,
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
}

API void ref_view_teardown() {
  ViewNode::astar_.reset();
  ViewNode::caster_.reset();
  ViewNode::map_.reset();
  g_env.reset();
}

// searchPath (kind, the search's counters, length, path) then computeCost (cost) for one pair
API void ref_view_cost(const double p1[3], const double p2[3], double y1, double y2, const double v1[3], Info* inf,
                       int32_t path_max, double* path) {
  memset(inf, 0, sizeof(*inf));
  Astar& a = *ViewNode::astar_;
  std::vector<Vector3d> pa, pb;
  const double t0 = ros::Time::clock();  // Astar::search reads the clock: it moved iff the line was blocked
  inf->length = ViewNode::searchPath(v3(p1), v3(p2), pa);
  if (ros::Time::clock() == t0) {
    inf->kind = 1;
  } else {
    inf->kind = a.path_nodes_.empty() ? 3 : 2;
    inf->iter_num = a.iter_num_;
    inf->use_node_num = a.use_node_num_;
    if (inf->kind == 2)
      inf->reason = 0;
    else if (a.use_node_num_ == a.allocate_num_)
      inf->reason = 2;
    else if (a.open_set_.empty())
      inf->reason = 1;
    else
      inf->reason = 3;
  }
  inf->n_path = (int32_t)pa.size();
  inf->cost = ViewNode::computeCost(v3(p1), v3(p2), y1, y2, v3(v1), 0, pb);
  put_path(pa, path_max, path);
}

// ---- FrontierFinder's cost bookkeeping over an installed frontier list ----------------------------------------------
API void* ref_ffc_create(void* sdf_map_handle) {
  ros::NodeHandle nh;
  EDTEnvironment::Ptr env(new EDTEnvironment);
  env->sdf_map_ = std::shared_ptr<SDFMap>((SDFMap*)sdf_map_handle, [](SDFMap*) {});
  return new FrontierFinder(env, nh);
}
API void ref_ffc_destroy(void* h) { delete (FrontierFinder*)h; }

// frontiers_ = n clusters, each with one viewpoint (pos, yaw) and the cost / path lists given (ncost[i] entries;
// path_rows[k] points per entry, in order), first_new_ftr_ = the cluster first_new (n: end()), removed_ids_
API void ref_ffc_install(void* h, int32_t n, const double* pos, const double* yaw, const int32_t* ncost,
                         const double* costs, const int32_t* path_rows, const double* pts, int32_t first_new,
                         int32_t n_removed, const int32_t* removed) {
  FrontierFinder& ff = *(FrontierFinder*)h;
  ff.frontiers_.clear();
  int k = 0, r = 0;
  for (int i = 0; i < n; ++i) {
    Frontier f;
    Viewpoint v;
    v.pos_ = v3(pos + 3 * i);
    v.yaw_ = yaw[i];
    v.visib_num_ = 0;
    f.viewpoints_.push_back(v);
    f.id_ = i;
    for (int c = 0; c < ncost[i]; ++c, ++k) {
      f.costs_.push_back(costs[k]);
      std::vector<Vector3d> p;
      for (int j = 0; j < path_rows[k]; ++j, ++r) p.push_back(v3(pts + 3 * r));
      f.paths_.push_back(p);
    }
    ff.frontiers_.push_back(f);
  }
  ff.first_new_ftr_ = ff.frontiers_.begin();
  std::advance(ff.first_new_ftr_, first_new);
  ff.removed_ids_.assign(removed, removed + n_removed);
}

API void ref_ffc_update(void* h) { ((FrontierFinder*)h)->updateFrontierCostMatrix(); }

// cluster i's cost list: its length and the total of its paths' points
API void ref_ffc_sizes(void* h, int32_t i, int32_t* ncost, int32_t* npts) {
  auto it = ((FrontierFinder*)h)->frontiers_.begin();
  std::advance(it, i);
  *ncost = (int32_t)it->costs_.size();
  int s = 0;
  for (const auto& p : it->paths_) s += (int)p.size();
  *npts = s;
}
API void ref_ffc_lists(void* h, int32_t i, double* costs, int32_t* path_rows, double* pts) {
  auto it = ((FrontierFinder*)h)->frontiers_.begin();
  std::advance(it, i);
  int k = 0, r = 0;
  for (double c : it->costs_) costs[k++] = c;
  k = 0;
  for (const auto& p : it->paths_) {
    path_rows[k++] = (int32_t)p.size();
    for (const auto& q : p)
      for (int a = 0; a < 3; ++a) pts[3 * r + a] = q(a), r += a == 2;
  }
}

// getFullCostMatrix: mat [(n + 1) * (n + 1)], row-major
API void ref_ffc_full(void* h, const double cur_pos[3], const double cur_vel[3], const double cur_yaw[3], double* mat) {
  Eigen::MatrixXd m;
  ((FrontierFinder*)h)->getFullCostMatrix(v3(cur_pos), v3(cur_vel), v3(cur_yaw), m);
  for (int i = 0; i < m.rows(); ++i)
    for (int j = 0; j < m.cols(); ++j) mat[(size_t)i * m.cols() + j] = m(i, j);
}

// getPathForTour: the path's row count; its first max_rows rows into out
API int32_t ref_ffc_tour(void* h, const double pos[3], int32_t n_ids, const int32_t* ids, int32_t max_rows, double* out) {
  std::vector<int> fid(ids, ids + n_ids);
  std::vector<Vector3d> path;
  ((FrontierFinder*)h)->getPathForTour(v3(pos), fid, path);
  put_path(path, max_rows, out);
  return (int32_t)path.size();
}
