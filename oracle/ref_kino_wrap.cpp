// Drives the reference's own KinodynamicAstar (path_searching/src/kinodynamic_astar.cpp, compiled unmodified from the
// reference against oracle/ref_standin_kino, then oracle/ref_standin_astar and oracle/ref_standin) on the reference's
// SDFMap of oracle/_ref/libfuel_ref.so, restating only FastPlannerManager::kinodynamicReplan's lines 131-164
// (plan_manage/src/planner_manager.cpp): the close-goal refusal, reset / search(init = true), the retry at
// init = false after NO_PATH, and getSamples at ts = ctrl_pt_dist / max_vel.  Outputs are laid out like the oracle's.
// TEST INFRASTRUCTURE ONLY; built into oracle/_ref/libfuel_ref_kino.so by oracle/kino.mk.
#include <stdint.h>
#include <string.h>

#include <cmath>

#include <plan_env/edt_environment.h>
#include <plan_env/sdf_map.h>
// path_nodes_, use_node_num_, iter_num_, is_shot_succ_, coef_shot_, t_shot_ are private: this translation unit -- the
// test wrapper, not the reference sources -- reads them
#define private public
#include <path_searching/kinodynamic_astar.h>
#undef private

using namespace fast_planner;
using Eigen::Vector3d;

namespace {
struct RefKino {
  KinodynamicAstar kino;
  EDTEnvironment::Ptr env;
  double ctrl_pt_dist, manager_max_vel;
};
// the layout of FuelKinoInfo (include/fuelgpu.h)
struct Info {
  int32_t status, reason, retried, traj_status, iter_num, use_node_num, n_nodes, shot, seg_num, n_pts;
  double t_shot, T_sum;
};
constexpr int K_MAX = 62;  // FUELGPU_MAX_PTS - 2
}  // namespace

extern "C" {

__attribute__((visibility("default"))) void* ref_kino_create(void* sdf_map_handle, const double* dparams,
                                                             const int32_t* iparams) {
  // dparams: max_tau, init_max_tau, max_vel, vel_margin, max_acc, w_time, horizon, lambda_heu, resolution_astar,
  // ctrl_pt_dist, manager_max_vel; iparams: allocate_num, check_num, optimistic
  RefKino* r = new RefKino;
  r->env.reset(new EDTEnvironment);
  r->env->sdf_map_ = std::shared_ptr<SDFMap>((SDFMap*)sdf_map_handle, [](SDFMap*) {});
  ros::NodeHandle nh;
  const char* dk[] = { "search/max_tau", "search/init_max_tau", "search/max_vel", "search/vel_margin", "search/max_acc",
                       "search/w_time", "search/horizon", "search/lambda_heu", "search/resolution_astar" };
  for (int i = 0; i < 9; ++i) nh.values[dk[i]] = dparams[i];
  nh.values["search/allocate_num"] = iparams[0];
  nh.values["search/check_num"] = iparams[1];
  nh.values["search/optimistic"] = iparams[2];
  r->ctrl_pt_dist = dparams[9];
  r->manager_max_vel = dparams[10];
  r->kino.setParam(nh);
  r->kino.setEnvironment(r->env);
  r->kino.init();
  return r;
}

__attribute__((visibility("default"))) void ref_kino_destroy(void* h) { delete (RefKino*)h; }

// one kinodynamicReplan(start, vel, acc, goal, 0) up to getSamples; points [62][3], derivs [4][3], dt [1],
// nodes [node_max][12], shot [3][4], as the oracle writes them
__attribute__((visibility("default"))) void ref_kino_run(void* h, const double s[3], const double v[3], const double a[3],
                                                         const double e[3], Info* out, double* points, double* derivs,
                                                         double* dt, int32_t node_max, double* nodes, double* shot) {
  RefKino* r = (RefKino*)h;
  KinodynamicAstar& k = r->kino;
  memset(out, 0, sizeof(*out));
  memset(points, 0, sizeof(double) * K_MAX * 3);
  memset(derivs, 0, sizeof(double) * 12);
  if (nodes) memset(nodes, 0, sizeof(double) * 12 * (size_t)node_max);
  if (shot) memset(shot, 0, sizeof(double) * 12);
  *dt = NAN;
  out->traj_status = 2;
  const Vector3d start_pt(s[0], s[1], s[2]), start_vel(v[0], v[1], v[2]), start_acc(a[0], a[1], a[2]);
  const Vector3d end_pt(e[0], e[1], e[2]), end_vel(0.0, 0.0, 0.0);
  if ((start_pt - end_pt).norm() < 1e-2) {  // :131-134
    out->status = KinodynamicAstar::NO_PATH;
    out->reason = 4;
    return;
  }
  k.reset();
  int status = k.search(start_pt, start_vel, start_acc, end_pt, end_vel, true);
  if (status == KinodynamicAstar::NO_PATH) {
    out->retried = 1;
    k.reset();
    status = k.search(start_pt, start_vel, start_acc, end_pt, end_vel, false);
  }
  out->status = status;
  out->iter_num = k.iter_num_;
  out->use_node_num = k.use_node_num_;
  if (status == KinodynamicAstar::NO_PATH) {
    // why: the pool ran out, the open set ran empty, or the start node lay within the goal tolerance
    out->reason = k.use_node_num_ == k.allocate_num_ ? 2 : (k.path_nodes_.size() == 1 ? 3 : 1);
    return;
  }
  out->shot = k.is_shot_succ_;
  out->t_shot = k.is_shot_succ_ ? k.t_shot_ : 0.0;
  out->n_nodes = (int32_t)k.path_nodes_.size();
  if (nodes)
    for (int i = 0; i < out->n_nodes && i < node_max; ++i) {
      PathNode* n = k.path_nodes_[i];
      double* o = nodes + 12 * (size_t)i;
      for (int j = 0; j < 6; ++j) o[j] = n->state(j);
      for (int j = 0; j < 3; ++j) o[6 + j] = n->parent ? n->input(j) : 0.0;
      o[9] = n->parent ? n->duration : 0.0, o[10] = n->g_score, o[11] = n->f_score;
    }
  if (shot && k.is_shot_succ_)
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 4; ++j) shot[4 * i + j] = k.coef_shot_(i, j);
  double ts = r->ctrl_pt_dist / r->manager_max_vel;  // :162
  std::vector<Vector3d> point_set, start_end_derivatives;
  k.getSamples(ts, point_set, start_end_derivatives);
  // getSamples' own seg_num and T_sum, restated from its first lines (:546-573)
  double T_sum = k.is_shot_succ_ ? k.t_shot_ : 0.0;
  for (PathNode* n = k.path_nodes_.back(); n->parent != NULL; n = n->parent) T_sum += n->duration;
  out->T_sum = T_sum;
  out->seg_num = std::max(8, (int)std::floor(T_sum / (r->ctrl_pt_dist / r->manager_max_vel)));
  if ((int)point_set.size() > K_MAX) {
    out->traj_status = 1;
    return;
  }
  out->traj_status = 0;
  out->n_pts = (int32_t)point_set.size() + 2;
  for (size_t i = 0; i < point_set.size(); ++i)
    for (int j = 0; j < 3; ++j) points[3 * i + j] = point_set[i](j);
  for (int i = 0; i < 4; ++i)
    for (int j = 0; j < 3; ++j) derivs[3 * i + j] = start_end_derivatives[i](j);
  *dt = ts;
}
}
