// Drives the reference's own Astar (path_searching/src/astar2.cpp, compiled unmodified from /root/reference against
// oracle/ref_standin_astar, then oracle/ref_standin) on the reference's SDFMap of oracle/_ref/libfuel_ref.so the way
// FastExplorationManager::planExploreMotion does (exploration_manager/src/fast_exploration_manager.cpp:238-263):
// reset(), search(pos, next_pos), getPath(); then restates shortenPath (:295-325) over the compiled RayCaster and
// SDFMap, and the radius_close / radius_far branch -- fast_exploration_manager.cpp cannot be compiled here.
// TEST INFRASTRUCTURE ONLY; built into oracle/_ref/libfuel_ref_astar.so by oracle/astar.mk.
#include <stdint.h>
#include <string.h>

#include <plan_env/edt_environment.h>
#include <plan_env/raycast.h>
#include <plan_env/sdf_map.h>
// iter_num_, use_node_num_, open_set_ and early_terminate_cost_ are private: this translation unit -- the test
// wrapper, not the reference sources -- reads them
#define private public
#include <path_searching/astar2.h>
#undef private

using namespace fast_planner;
using Eigen::Vector3d;

namespace {
struct RefAstar {
  Astar astar;
  EDTEnvironment::Ptr env;
  RayCaster caster;
};
// the layout of FuelPathInfo (include/fuelgpu.h)
struct Info {
  int32_t status, reason, iter_num, use_node_num, n_path, n_wp, branch, tour_status;
  double early_terminate_cost, length, next_goal[3];
};
}  // namespace

extern "C" {

__attribute__((visibility("default"))) void* ref_astar_create(void* sdf_map_handle, double resolution, double lambda,
                                                              int32_t allocate_num, double max_search_time) {
  RefAstar* r = new RefAstar;
  r->env.reset(new EDTEnvironment);
  r->env->sdf_map_ = std::shared_ptr<SDFMap>((SDFMap*)sdf_map_handle, [](SDFMap*) {});
  ros::NodeHandle nh;
  nh.values["astar/resolution_astar"] = resolution;
  nh.values["astar/lambda_heu"] = lambda;
  nh.values["astar/max_search_time"] = max_search_time;
  nh.values["astar/allocate_num"] = allocate_num;
  r->astar.init(nh, r->env);
  // ViewNode::caster_ as FastExplorationManager::initialize sets it (:66-69): the map's resolution and origin
  Vector3d origin, size;
  r->env->sdf_map_->getRegion(origin, size);
  r->caster.setParams(r->env->sdf_map_->getResolution(), origin);
  return r;
}

__attribute__((visibility("default"))) void ref_astar_destroy(void* h) { delete (RefAstar*)h; }

// one query -> info, the first path_max rows of getPath(), the first w_max rows of the tour; returns the n_wp the
// device writes (the tour's count when usable, else 0)
__attribute__((visibility("default"))) int32_t ref_astar_run(void* h, const double s[3], const double e[3],
                                                             int32_t w_max, Info* inf, int32_t path_max, double* path,
                                                             double* waypts) {
  RefAstar& r = *(RefAstar*)h;
  Astar& a = r.astar;
  SDFMap& map = *r.env->sdf_map_;
  memset(inf, 0, sizeof(*inf));
  const Vector3d pos(s[0], s[1], s[2]), next_pos(e[0], e[1], e[2]);
  a.reset();
  a.early_terminate_cost_ = 0.0;  // reset() keeps the last value; report it for the time cut alone
  inf->status = a.search(pos, next_pos);
  inf->iter_num = a.iter_num_;
  inf->use_node_num = a.use_node_num_;
  if (inf->status == Astar::REACH_END)
    inf->reason = 0;
  else if (a.use_node_num_ == a.allocate_num_)
    inf->reason = 2;  // run out of node pool
  else if (a.open_set_.empty())
    inf->reason = 1;
  else
    inf->reason = 3;  // time cut
  inf->early_terminate_cost = a.getEarlyTerminateCost();
  if (inf->status != Astar::REACH_END) return 0;

  std::vector<Vector3d> path_next_goal = a.getPath();
  inf->n_path = (int32_t)path_next_goal.size();
  for (int i = 0; i < path_max && i < (int)path_next_goal.size(); ++i)
    for (int k = 0; k < 3; ++k) path[3 * i + k] = path_next_goal[i](k);

  // shortenPath (:295-325)
  {
    std::vector<Vector3d>& path = path_next_goal;
    const double dist_thresh = 3.0;
    std::vector<Vector3d> short_tour = { path.front() };
    for (int i = 1; i < (int)path.size() - 1; ++i) {
      if ((path[i] - short_tour.back()).norm() > dist_thresh)
        short_tour.push_back(path[i]);
      else {
        r.caster.input(short_tour.back(), path[i + 1]);
        Eigen::Vector3i idx;
        while (r.caster.nextId(idx) && ros::ok()) {
          if (map.getInflateOccupancy(idx) == 1 || map.getOccupancy(idx) == SDFMap::UNKNOWN) {
            short_tour.push_back(path[i]);
            break;
          }
        }
      }
    }
    if ((path.back() - short_tour.back()).norm() > 1e-3) short_tour.push_back(path.back());
    if (short_tour.size() == 2) short_tour.insert(short_tour.begin() + 1, 0.5 * (short_tour[0] + short_tour[1]));
    path = short_tour;
  }

  // the branch (:243-263)
  const double radius_far = 5.0;
  const double radius_close = 1.5;
  const double len = Astar::pathLength(path_next_goal);
  inf->length = len;
  std::vector<Vector3d> tour;
  Vector3d next_goal;
  if (len < radius_close) {
    inf->branch = 1;
    tour = path_next_goal;
    next_goal = next_pos;
  } else if (len > radius_far) {
    inf->branch = 3;
    double len2 = 0.0;
    std::vector<Vector3d> truncated_path = { path_next_goal.front() };
    for (int i = 1; i < (int)path_next_goal.size() && len2 < radius_far; ++i) {
      auto cur_pt = path_next_goal[i];
      len2 += (cur_pt - truncated_path.back()).norm();
      truncated_path.push_back(cur_pt);
    }
    next_goal = truncated_path.back();
    tour = truncated_path;
  } else {
    inf->branch = 2;  // kinodynamicReplan in the reference
    tour = path_next_goal;
    next_goal = next_pos;
  }
  for (int k = 0; k < 3; ++k) inf->next_goal[k] = next_goal(k);
  const int nt = (int)tour.size();
  inf->n_wp = nt;
  inf->tour_status = nt < 3 ? 2 : ((nt > 32 || nt > w_max) ? 1 : 0);
  for (int i = 0; i < nt && i < w_max; ++i)
    for (int k = 0; k < 3; ++k) waypts[3 * i + k] = tour[i](k);
  return inf->tour_status == 0 ? nt : 0;
}

}  // extern "C"
