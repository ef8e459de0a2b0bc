// fuelgpu_shim.hpp -- C++ host-side mirror of the reference classes on the hot path, over the C ABI.
//
// Same class names, method names, argument meaning and sentinel behaviour as the reference
// (file:line under /root/reference/fuel_planner/):
//   fast_planner::SDFMap           plan_env/include/plan_env/sdf_map.h:27-84
//   fast_planner::EDTEnvironment   plan_env/include/plan_env/edt_environment.h:21-51
//   fast_planner::FrontierFinder   active_perception/include/active_perception/frontier_finder.h:53-131
//   fast_planner::ViewNode         active_perception/include/active_perception/graph_node.h:49-84 (the statics and
//                                  the two static cost methods)
//   fast_planner::BsplineOptimizer bspline_opt/include/bspline_opt/bspline_optimizer.h:20-145
// Only the members the hot path needs are mirrored (SURVEY.md 8b); everything voxel-scale is a
// call into libfuelgpu (hand-written sm_90a CUDA).  The reference uses Eigen::Vector3d/3i and a
// ros::NodeHandle for parameters; define FUELGPU_SHIM_USE_EIGEN before including this header to
// get the Eigen types, otherwise a minimal 3-vector with the same element access is used (Eigen
// is not installed in the build image).  Parameters arrive as plain structs instead of ROS params.
#pragma once

#include <cmath>
#include <cstdint>
#include <cstring>
#include <algorithm>
#include <list>
#include <memory>
#include <stdexcept>
#include <string>
#include <vector>

#include "fuelgpu.h"

#ifdef FUELGPU_SHIM_USE_EIGEN
#include <Eigen/Eigen>
namespace fuelgpu_shim {
using Vector3d = Eigen::Vector3d;
using Vector3i = Eigen::Vector3i;
}  // namespace fuelgpu_shim
#else
namespace fuelgpu_shim {
template <typename T>
struct Vec3 {
  T v[3];
  Vec3() : v{ 0, 0, 0 } {}
  Vec3(T a, T b, T c) : v{ a, b, c } {}
  T& operator()(int i) { return v[i]; }
  const T& operator()(int i) const { return v[i]; }
  T& operator[](int i) { return v[i]; }
  const T& operator[](int i) const { return v[i]; }
  T* data() { return v; }
  const T* data() const { return v; }
};
using Vector3d = Vec3<double>;
using Vector3i = Vec3<int32_t>;
}  // namespace fuelgpu_shim
#endif

namespace fast_planner {
using fuelgpu_shim::Vector3d;
using fuelgpu_shim::Vector3i;

struct FuelGpuError : std::runtime_error {
  int code;
  FuelGpuError(int c, const char* msg) : std::runtime_error(msg ? msg : ""), code(c) {}
};
inline void fuelgpu_check(int rc, const FuelMap* h) {
  if (rc != FUELGPU_OK) throw FuelGpuError(rc, fuelgpu_last_error(h));
}

// ---- SDFMap (sdf_map.h:27-84) --------------------------------------------------------------
struct MapParam {  // the ROS parameters of initMap (sdf_map.cpp:19-47,79-84) as a struct
  Vector3i map_voxel_num_;
  double resolution_ = 0.1;
  Vector3d map_origin_;
  Vector3d map_size_;  // sdf_map/map_size_x,y,z; a zero component means n * resolution (sdf_map.cpp:34-39)
  Vector3d box_mind_, box_maxd_;
  bool optimistic_ = false, signed_dist_ = false;
  double p_min_ = 0.12, p_occ_ = 0.80;
  double default_dist_ = 0.0;
  int device = 0;
};

class SDFMap {
public:
  enum OCCUPANCY { UNKNOWN, FREE, OCCUPIED };
  typedef std::shared_ptr<SDFMap> Ptr;

  SDFMap() {}
  ~SDFMap() {
    if (gpu_) fuelgpu_map_destroy(gpu_);
  }
  SDFMap(const SDFMap&) = delete;
  SDFMap& operator=(const SDFMap&) = delete;

  // initMap (sdf_map.cpp:12-93)
  void initMap(const MapParam& p) {
    mp_ = p;
    resolution_inv_ = 1 / mp_.resolution_;
    auto logit = [](double x) { return std::log(x / (1 - x)); };
    clamp_min_log_ = logit(mp_.p_min_);
    min_occupancy_log_ = logit(mp_.p_occ_);
    const size_t n = (size_t)mp_.map_voxel_num_(0) * mp_.map_voxel_num_(1) * mp_.map_voxel_num_(2);
    occupancy_buffer_.assign(n, clamp_min_log_ - 0.01);  // unknown_flag_, sdf_map.cpp:56,64
    occupancy_buffer_inflate_.assign(n, 0);
    distance_buffer_.assign(n, mp_.default_dist_);
    for (int i = 0; i < 3; ++i) {
      map_max_boundary_(i) = mp_.map_origin_(i) + (mp_.map_size_(i) > 0.0 ? mp_.map_size_(i) : mp_.map_voxel_num_(i) * mp_.resolution_);
      local_bound_min_(i) = 0;
      local_bound_max_(i) = mp_.map_voxel_num_(i) - 1;
    }
    posToIndex(mp_.box_mind_, box_min_);
    posToIndex(mp_.box_maxd_, box_max_);
    FuelGridDesc d;
    for (int i = 0; i < 3; ++i) {
      d.n[i] = mp_.map_voxel_num_(i);
      d.origin[i] = mp_.map_origin_(i);
      d.box_mind[i] = mp_.box_mind_(i);
      d.box_maxd[i] = mp_.box_maxd_(i);
      d.map_size[i] = mp_.map_size_(i);
    }
    d.resolution = mp_.resolution_;
    fuelgpu_check(fuelgpu_map_create(&d, mp_.device, &gpu_), nullptr);
  }

  // index helpers (sdf_map.h:127-192)
  void posToIndex(const Vector3d& pos, Vector3i& id) const {
    for (int i = 0; i < 3; ++i) id(i) = (int32_t)std::floor((pos(i) - mp_.map_origin_(i)) * resolution_inv_);
  }
  void indexToPos(const Vector3i& id, Vector3d& pos) const {
    for (int i = 0; i < 3; ++i) pos(i) = (id(i) + 0.5) * mp_.resolution_ + mp_.map_origin_(i);
  }
  void boundIndex(Vector3i& id) const {
    for (int i = 0; i < 3; ++i) id(i) = std::max(std::min(id(i), mp_.map_voxel_num_(i) - 1), 0);
  }
  int toAddress(const Vector3i& id) const { return toAddress(id[0], id[1], id[2]); }
  int toAddress(int x, int y, int z) const {
    return x * mp_.map_voxel_num_(1) * mp_.map_voxel_num_(2) + y * mp_.map_voxel_num_(2) + z;
  }
  bool isInMap(const Vector3d& pos) const {
    for (int i = 0; i < 3; ++i)
      if (pos(i) < mp_.map_origin_(i) + 1e-4 || pos(i) > map_max_boundary_(i) - 1e-4) return false;
    return true;
  }
  bool isInMap(const Vector3i& idx) const {
    for (int i = 0; i < 3; ++i)
      if (idx(i) < 0 || idx(i) > mp_.map_voxel_num_(i) - 1) return false;
    return true;
  }
  bool isInBox(const Vector3i& id) const {
    for (int i = 0; i < 3; ++i)
      if (id[i] < box_min_[i] || id[i] >= box_max_[i]) return false;
    return true;
  }
  bool isInBox(const Vector3d& pos) const {
    for (int i = 0; i < 3; ++i)
      if (pos[i] <= mp_.box_mind_[i] || pos[i] >= mp_.box_maxd_[i]) return false;
    return true;
  }
  int getOccupancy(const Vector3i& id) const {
    if (!isInMap(id)) return -1;
    const double occ = occupancy_buffer_[toAddress(id)];
    if (occ < clamp_min_log_ - 1e-3) return UNKNOWN;
    if (occ > min_occupancy_log_) return OCCUPIED;
    return FREE;
  }
  int getOccupancy(const Vector3d& pos) const {
    Vector3i id;
    posToIndex(pos, id);
    return getOccupancy(id);
  }
  int getInflateOccupancy(const Vector3i& id) const {
    if (!isInMap(id)) return -1;
    return (int)occupancy_buffer_inflate_[toAddress(id)];
  }
  void setOccupied(const Vector3d& pos, const int& occ = 1) {
    if (!isInMap(pos)) return;
    Vector3i id;
    posToIndex(pos, id);
    occupancy_buffer_inflate_[toAddress(id)] = (int8_t)occ;
  }
  void resetBuffer() {  // sdf_map.cpp:95-99
    std::fill(occupancy_buffer_inflate_.begin(), occupancy_buffer_inflate_.end(), 0);
    std::fill(distance_buffer_.begin(), distance_buffer_.end(), mp_.default_dist_);
    for (int i = 0; i < 3; ++i) {
      local_bound_min_(i) = 0;
      local_bound_max_(i) = mp_.map_voxel_num_(i) - 1;
    }
  }
  double getDistance(const Vector3i& id) const {
    if (!isInMap(id)) return -1;
    return distance_buffer_[toAddress(id)];
  }
  double getDistance(const Vector3d& pos) const {
    Vector3i id;
    posToIndex(pos, id);
    return getDistance(id);
  }
  double getResolution() const { return mp_.resolution_; }
  int getVoxelNum() const { return mp_.map_voxel_num_[0] * mp_.map_voxel_num_[1] * mp_.map_voxel_num_[2]; }
  void getRegion(Vector3d& ori, Vector3d& size) const {
    ori = mp_.map_origin_;
    for (int i = 0; i < 3; ++i) size(i) = mp_.map_voxel_num_(i) * mp_.resolution_;
  }
  void getBox(Vector3d& bmin, Vector3d& bmax) const {
    bmin = mp_.box_mind_;
    bmax = mp_.box_maxd_;
  }
  void getUpdatedBox(Vector3d& bmin, Vector3d& bmax, bool reset = false) {
    if (fused_) {  // the box is accumulated by the device fusion calls (sdf_map.cpp:321-324)
      fuelgpu_check(fuelgpu_map_get_updated_box(gpu_, bmin.data(), bmax.data(), reset ? 1 : 0), gpu_);
      return;
    }
    bmin = update_min_;
    bmax = update_max_;
    if (reset) reset_updated_box_ = true;
  }

  // inputPointCloud (sdf_map.cpp:259-345): fuses one frame into the device-resident log-odds volume and
  // sets local_bound_min_/max_.  `points` = cloud.points.data() of a pcl::PointCloud<pcl::PointXYZ>
  // (point_stride 4) or packed xyz (point_stride 3).  From here on the occupancy lives on the device:
  // updateESDF3d() no longer uploads occupancy_buffer_.
  FuelFusionParams fusion_ = { 0.65, 0.35, 0.12, 0.90, 0.80, 4.5, 0.5 };  // algorithm.xml:39-50
  void inputPointCloud(const float* points, int point_num, const Vector3d& camera_pos, int point_stride = 4) {
    if (point_num == 0) return;
    fuelgpu_check(fuelgpu_map_input_point_cloud(gpu_, points, point_num, point_stride, camera_pos.data(), &fusion_,
                                                local_bound_min_.data(), local_bound_max_.data()),
                  gpu_);
    fused_ = true;
  }
  // MapROS::proessDepthImage + inputPointCloud (map_ros.cpp:139-140,176-215) as one device call; camera_R is
  // camera_q_.toRotationMatrix() in row-major order.  Returns proj_points_cnt.
  FuelCameraParams camera_ = { 387.229248046875, 387.229248046875, 321.04638671875, 243.44969177246094, 1000.0, 5.0, 0.2, 2, 2 };
  int inputDepthImage(const uint16_t* depth, int rows, int cols, const double camera_R[9], const Vector3d& camera_pos) {
    int32_t cnt = 0;
    fuelgpu_check(fuelgpu_map_input_depth_image(gpu_, depth, rows, cols, &camera_, camera_R, camera_pos.data(), &fusion_,
                                                local_bound_min_.data(), local_bound_max_.data(), &cnt),
                  gpu_);
    if (cnt > 0) fused_ = true;
    return cnt;
  }

  // updateESDF3d (sdf_map.cpp:152-241): occupancy H2D for the x-slabs of the local box, the three
  // sweeps on the device, and the fp64 host mirror the scattered getDistance() readers use.
  void updateESDF3d() {
    if (!fused_)
      fuelgpu_check(fuelgpu_map_upload_occupancy(gpu_, occupancy_buffer_inflate_.data(), occupancy_buffer_.data(), nullptr,
                                               clamp_min_log_, min_occupancy_log_, local_bound_min_.data(),
                                               local_bound_max_.data()),
                  gpu_);
    const int flags = (mp_.optimistic_ ? FUELGPU_ESDF_OPTIMISTIC : 0) | (mp_.signed_dist_ ? FUELGPU_ESDF_SIGNED : 0);
    fuelgpu_check(fuelgpu_esdf_update(gpu_, local_bound_min_.data(), local_bound_max_.data(), flags), gpu_);
    fuelgpu_check(fuelgpu_esdf_download(gpu_, local_bound_min_.data(), local_bound_max_.data(), nullptr,
                                        distance_buffer_.data()),
                  gpu_);
  }
  // clearAndInflateLocalMap (sdf_map.cpp:364-472) on the resident occupancy byte (the byte must have been
  // uploaded, e.g. by the previous updateESDF3d); refreshes occupancy_buffer_inflate_
  void clearAndInflateLocalMap(double obstacles_inflation, double virtual_ceil_height) {
    const int inf_step = (int)std::ceil(obstacles_inflation / mp_.resolution_);
    const int ceil_id = virtual_ceil_height > -0.5
                            ? (int)std::floor((virtual_ceil_height - mp_.map_origin_(2)) * resolution_inv_)
                            : -1;
    fuelgpu_check(fuelgpu_map_inflate(gpu_, local_bound_min_.data(), local_bound_max_.data(), inf_step, ceil_id), gpu_);
    fuelgpu_check(fuelgpu_map_download_occupancy(gpu_, occupancy_buffer_inflate_.data(), nullptr), gpu_);
  }
  // getDistWithGrad (sdf_map.cpp:497-536) on the device ESDF
  double getDistWithGrad(const Vector3d& pos, Vector3d& grad) {
    double d = 0;
    fuelgpu_check(fuelgpu_esdf_sample(gpu_, 1, pos.data(), &d, grad.data()), gpu_);
    return d;
  }

  FuelMap* gpu() const { return gpu_; }
  // MapData (sdf_map.h:107-125): the reference's friend MapROS pokes these directly
  std::vector<double> occupancy_buffer_;
  std::vector<int8_t> occupancy_buffer_inflate_;
  std::vector<double> distance_buffer_;
  Vector3i local_bound_min_, local_bound_max_;
  Vector3d update_min_, update_max_;
  bool reset_updated_box_ = true;
  bool fused_ = false;
  MapParam mp_;

private:
  double resolution_inv_ = 10.0, clamp_min_log_ = 0, min_occupancy_log_ = 0;
  Vector3d map_max_boundary_;
  Vector3i box_min_, box_max_;
  FuelMap* gpu_ = nullptr;
};

// ---- EDTEnvironment (edt_environment.h:21-51) --------------------------------------------------
class EDTEnvironment {
public:
  typedef std::shared_ptr<EDTEnvironment> Ptr;
  void setMap(std::shared_ptr<SDFMap>& map) {
    sdf_map_ = map;
    resolution_inv_ = 1 / sdf_map_->getResolution();
  }
  // edt_environment.cpp:78-87: pass-through, `time` unused
  void evaluateEDTWithGrad(const Vector3d& pos, double /*time*/, double& dist, Vector3d& grad) {
    dist = sdf_map_->getDistWithGrad(pos, grad);
  }
  double evaluateCoarseEDT(Vector3d& pos, double /*time*/) { return sdf_map_->getDistance(pos); }
  std::shared_ptr<SDFMap> sdf_map_;

private:
  double resolution_inv_ = 10.0;
};

// ---- Astar (path_searching/include/path_searching/astar2.h) over fuelgpu_astar_batch -----------------------
// One search per call on the device of the environment's map.  init() takes the astar/* parameters as a struct;
// max_search_time_ is an iteration cap here (max_iter): NO_PATH at loop iteration max_iter + 1.
struct AstarParam {
  double resolution_astar = 0.1, lambda_heu = 10000.0;
  int allocate_num = 100000, max_iter = 100000;
};
class Astar {
public:
  enum { REACH_END = 1, NO_PATH = 2 };
  void init(const AstarParam& p, const EDTEnvironment::Ptr& env) {
    resolution_ = p.resolution_astar;
    lambda_heu_ = p.lambda_heu;
    allocate_num_ = p.allocate_num;
    max_iter = p.max_iter;
    edt_env_ = env;
  }
  void setResolution(const double& res) { resolution_ = res; }
  void reset() {
    path_nodes_.clear();
    use_node_num_ = iter_num_ = 0;
  }
  int search(const Vector3d& start_pt, const Vector3d& end_pt) {
    FuelMap* h = edt_env_->sdf_map_->gpu();
    const FuelAstarParams ap{ resolution_, lambda_heu_, allocate_num_, max_iter };
    const double s[3] = { start_pt(0), start_pt(1), start_pt(2) }, e[3] = { end_pt(0), end_pt(1), end_pt(2) };
    FuelPathInfo info;
    int32_t n_wp = 0;
    std::vector<double> path(3 * ((size_t)allocate_num_ + 1));  // getPath() has at most allocate_num + 1 points
    double wp[3 * FUELGPU_MAX_WAYPTS];
    fuelgpu_check(fuelgpu_astar_batch(h, 1, s, e, &ap, &info, allocate_num_ + 1, path.data(), FUELGPU_MAX_WAYPTS, &n_wp,
                                      wp),
                  h);
    use_node_num_ = info.use_node_num;
    iter_num_ = info.iter_num;
    if (info.reason == FUELGPU_ASTAR_ITER_CAP) early_terminate_cost_ = info.early_terminate_cost;
    path_nodes_.clear();
    for (int i = 0; i < info.n_path; ++i) path_nodes_.push_back(Vector3d(path[3 * i], path[3 * i + 1], path[3 * i + 2]));
    return info.status;
  }
  std::vector<Vector3d> getPath() { return path_nodes_; }
  static double pathLength(const std::vector<Vector3d>& path) {  // astar2.cpp:169-175
    double length = 0.0;
    for (size_t i = 0; i + 1 < path.size(); ++i) {
      const double dx = path[i + 1](0) - path[i](0), dy = path[i + 1](1) - path[i](1), dz = path[i + 1](2) - path[i](2);
      length += std::sqrt((dx * dx + dy * dy) + dz * dz);
    }
    return length;
  }
  double getEarlyTerminateCost() { return early_terminate_cost_; }
  int use_node_num() const { return use_node_num_; }
  int iter_num() const { return iter_num_; }

  double lambda_heu_ = 10000.0;
  int max_iter = 100000;  // stands for max_search_time_

private:
  EDTEnvironment::Ptr edt_env_;
  std::vector<Vector3d> path_nodes_;
  double resolution_ = 0.1, early_terminate_cost_ = 0.0;
  int allocate_num_ = 100000, use_node_num_ = 0, iter_num_ = 0;
};

// ---- KinodynamicAstar (path_searching/include/path_searching/kinodynamic_astar.h) over fuelgpu_kino_search_batch ------
// What FastPlannerManager::kinodynamicReplan (planner_manager.cpp:131-164) does with kino_path_finder_, on the device of
// the environment's map: search() runs the close-goal refusal, search(init = true) and, after NO_PATH, reset and
// search(init = false), and returns the status of the attempt that counted; getSamples() returns the samples at
// ts = ctrl_pt_dist / manager_max_vel.  setParam() takes the search/ parameters as FuelKinoParams.
class KinodynamicAstar {
public:
  enum { REACH_HORIZON = 1, REACH_END = 2, NO_PATH = 3, NEAR_END = 4 };
  void setParam(const FuelKinoParams& p) { p_ = p; }
  void setEnvironment(const EDTEnvironment::Ptr& env) { edt_env_ = env; }
  void init() {}
  void reset() {
    info_ = FuelKinoInfo();
    points_.clear();
  }
  int search(const Vector3d& start_pt, const Vector3d& start_vel, const Vector3d& start_acc, const Vector3d& end_pt) {
    FuelMap* h = edt_env_->sdf_map_->gpu();
    const double s[3] = { start_pt(0), start_pt(1), start_pt(2) }, v[3] = { start_vel(0), start_vel(1), start_vel(2) };
    const double a[3] = { start_acc(0), start_acc(1), start_acc(2) }, e[3] = { end_pt(0), end_pt(1), end_pt(2) };
    double pts[3 * (FUELGPU_MAX_PTS - 2)], der[12], shot[12];
    fuelgpu_check(fuelgpu_kino_search_batch(h, 1, s, v, a, e, &p_, &info_, pts, der, &ts_, 0, nullptr, shot), h);
    points_.clear();
    for (int i = 0; i + 2 < info_.n_pts; ++i) points_.push_back(Vector3d(pts[3 * i], pts[3 * i + 1], pts[3 * i + 2]));
    derivs_.clear();
    for (int i = 0; i < 4; ++i) derivs_.push_back(Vector3d(der[3 * i], der[3 * i + 1], der[3 * i + 2]));
    return info_.status;
  }
  // false when the search left no samples (NO_PATH or more than FUELGPU_MAX_PTS - 2 of them)
  bool getSamples(double& ts, std::vector<Vector3d>& point_set, std::vector<Vector3d>& start_end_derivatives) const {
    if (info_.traj_status != 0) return false;
    ts = ts_;
    point_set = points_;
    start_end_derivatives = derivs_;
    return true;
  }
  const FuelKinoInfo& info() const { return info_; }

private:
  EDTEnvironment::Ptr edt_env_;
  FuelKinoParams p_{ 0.8, 1.0, 2.0, 0.25, 2.0, 10.0, 5.0, 10.0, 0.025, 0.35, 2.0, 100000, 10, 0, 0 };  // algorithm.xml
  FuelKinoInfo info_{};
  double ts_ = 0.0;
  std::vector<Vector3d> points_, derivs_;
};

// ---- ViewNode (graph_node.h:49-84) over fuelgpu_view_cost_batch ------------------------------------------------
// Set the statics as FastExplorationManager::initialize does (fast_exploration_manager.cpp:55-69): vm_, yd_, w_dir_ from
// exploration/*, astar_param_ from astar/* (max_iter standing for max_search_time_; searchPath searches at resolution
// 0.4 whatever resolution_astar says), map_ the map searched.  Defaults: algorithm.xml:95-99,164-167, max_vel 2.0.
template <class Unused = void>
struct ViewNodeStatics {  // header-only definitions of the statics (C++14 has no inline variables)
  static double vm_, yd_, w_dir_;
  static AstarParam astar_param_;
  static std::shared_ptr<SDFMap> map_;
};
template <class U>
double ViewNodeStatics<U>::vm_ = 2.0;
template <class U>
double ViewNodeStatics<U>::yd_ = 60 * 3.1415926 / 180.0;
template <class U>
double ViewNodeStatics<U>::w_dir_ = 1.5;
template <class U>
AstarParam ViewNodeStatics<U>::astar_param_ = { 0.4, 10000.0, 1000000, 10000 };
template <class U>
std::shared_ptr<SDFMap> ViewNodeStatics<U>::map_;

class ViewNode : public ViewNodeStatics<> {
public:
  // computeCost (graph_node.cpp:63-85) for every pair in one device call: cost[q], searchPath's path[q] and, if
  // asked, its return value length[q]
  static void costBatch(const std::vector<Vector3d>& p1, const std::vector<Vector3d>& p2, const std::vector<double>& y1,
                        const std::vector<double>& y2, const std::vector<Vector3d>& v1, std::vector<double>& cost,
                        std::vector<std::vector<Vector3d>>& paths, std::vector<double>* length = nullptr) {
    FuelMap* h = map_->gpu();
    const size_t P = p1.size();
    std::vector<double> a(3 * P), b(3 * P), v(3 * P);
    for (size_t q = 0; q < P; ++q)
      for (int k = 0; k < 3; ++k) a[3 * q + k] = p1[q](k), b[3 * q + k] = p2[q](k), v[3 * q + k] = v1[q](k);
    const FuelViewCostParams prm{ vm_, yd_, w_dir_,
                                  { 0.4, astar_param_.lambda_heu, astar_param_.allocate_num, astar_param_.max_iter } };
    std::vector<FuelViewCostInfo> info(P);
    int path_max = 256;
    std::vector<double> path;
    for (;;) {  // a search path longer than path_max rows: run again with room for it
      path.assign(3 * P * (size_t)path_max, 0.0);
      fuelgpu_check(fuelgpu_view_cost_batch(h, (int32_t)P, a.data(), b.data(), y1.data(), y2.data(), v.data(), &prm,
                                            info.data(), path_max, path.data()),
                    h);
      int need = 0;
      for (const auto& i : info) need = std::max(need, (int)i.n_path);
      if (need <= path_max) break;
      path_max = need;
    }
    cost.resize(P);
    if (length) length->resize(P);
    paths.assign(P, {});
    for (size_t q = 0; q < P; ++q) {
      if (info[q].kind == 0) throw std::runtime_error("ViewNode: a pair has a non-finite input");
      cost[q] = info[q].cost;
      if (length) (*length)[q] = info[q].length;
      for (int i = 0; i < info[q].n_path; ++i) {
        const double* r = &path[(q * path_max + i) * 3];
        paths[q].push_back(Vector3d(r[0], r[1], r[2]));
      }
    }
  }
  static double computeCost(const Vector3d& p1, const Vector3d& p2, const double& y1, const double& y2,
                            const Vector3d& v1, const double& /*yd1: unused, as in the reference*/,
                            std::vector<Vector3d>& path) {
    std::vector<double> cost;
    std::vector<std::vector<Vector3d>> paths;
    costBatch({ p1 }, { p2 }, { y1 }, { y2 }, { v1 }, cost, paths);
    path = paths[0];
    return cost[0];
  }
  static double searchPath(const Vector3d& p1, const Vector3d& p2, std::vector<Vector3d>& path) {
    std::vector<double> cost, length;
    std::vector<std::vector<Vector3d>> paths;
    costBatch({ p1 }, { p2 }, { 0.0 }, { 0.0 }, { Vector3d(0, 0, 0) }, cost, paths, &length);
    path = paths[0];
    return length[0];
  }
};

// ---- FrontierFinder (frontier_finder.h:25-131) ---------------------------------------------------
struct Viewpoint {  // frontier_finder.h:25-31
  Vector3d pos_;
  double yaw_;
  int visib_num_;
};

struct Frontier {  // frontier_finder.h:34-51
  std::vector<Vector3d> cells_;
  std::vector<Viewpoint> viewpoints_;
  std::vector<Vector3d> filtered_cells_;
  Vector3d average_;
  int id_ = -1;
  Vector3d box_min_, box_max_;
  std::vector<int32_t> cell_addr_;  // toAddress of every cell (what the C ABI speaks)
  std::list<std::vector<Vector3d>> paths_;  // searchPath to every cluster, in frontiers_ order
  std::list<double> costs_;                 // computeCost to every cluster
};

struct FrontierParam {  // frontier_finder.cpp:29-40
  int cluster_min_ = 100;
  double cluster_size_xy_ = 2.0;
  int down_sample_ = 3;
  double min_candidate_dist_ = 0.75;  // frontier/min_candidate_dist (getTopViewpointsInfo, getViewpointsInfo)
};

class FrontierFinder {
public:
  FrontierFinder(const std::shared_ptr<EDTEnvironment>& edt, const FrontierParam& p) : edt_env_(edt), p_(p) {
    fuelgpu_check(fuelgpu_frontier_reset_flags(gpu()), gpu());  // frontier_flag_ fill, :26-27
  }

  // searchFrontiers (frontier_finder.cpp:54-121)
  void searchFrontiers() {
    tmp_frontiers_.clear();
    Vector3d update_min, update_max;
    edt_env_->sdf_map_->getUpdatedBox(update_min, update_max, true);
    removed_ids_.clear();
    removeChanged(frontiers_, update_min, update_max, true);           // :71-86
    removeChanged(dormant_frontiers_, update_min, update_max, false);  // :87-92
    FuelFrontierParams fp{ p_.cluster_min_, p_.cluster_size_xy_, p_.down_sample_, 0.4 };
    int32_t nc = 0, ncell = 0, nf = 0;
    fuelgpu_check(fuelgpu_frontier_search(gpu(), update_min.data(), update_max.data(), &fp, &nc, &ncell, &nf), gpu());
    std::vector<int32_t> co(nc + 1), ca(ncell), fo(nc + 1);
    std::vector<double> filt(3 * (size_t)nf), avg(3 * (size_t)nc), bmin(3 * (size_t)nc), bmax(3 * (size_t)nc);
    fuelgpu_check(fuelgpu_frontier_fetch(gpu(), co.data(), ca.data(), fo.data(), filt.data(), avg.data(), bmin.data(),
                                         bmax.data()),
                  gpu());
    const SDFMap& m = *edt_env_->sdf_map_;
    const int ny = m.mp_.map_voxel_num_(1), nz = m.mp_.map_voxel_num_(2);
    for (int c = 0; c < nc; ++c) {
      Frontier f;
      for (int i = co[c]; i < co[c + 1]; ++i) {
        const int a = ca[i];
        Vector3i id(a / (ny * nz), (a / nz) % ny, a % nz);
        Vector3d pos;
        m.indexToPos(id, pos);
        f.cells_.push_back(pos);
        f.cell_addr_.push_back(a);
      }
      for (int i = fo[c]; i < fo[c + 1]; ++i) f.filtered_cells_.emplace_back(filt[3 * i], filt[3 * i + 1], filt[3 * i + 2]);
      for (int k = 0; k < 3; ++k) {
        f.average_(k) = avg[3 * c + k];
        f.box_min_(k) = bmin[3 * c + k];
        f.box_max_(k) = bmax[3 * c + k];
      }
      tmp_frontiers_.push_back(f);
    }
  }
  // computeFrontiersToVisit (frontier_finder.cpp:392-423): sampleViewpoints (:662-695) of every new cluster in one
  // device call; clusters without a qualified viewpoint go dormant.
  FuelViewParams view_ = { 1.5, 2.5, 3, 15 * 3.1415926 / 180.0, 0.21, 0.56125, 0.69222, 0.68901, 4.5 };  // algorithm.xml:106-121
  int min_visib_num_ = 15;
  void computeFrontiersToVisit() {
    first_new_ftr_ = frontiers_.end();
    const int n = (int)tmp_frontiers_.size(), nc = fuelgpu_viewpoint_candidate_count(&view_);
    std::vector<int32_t> fo(n + 1, 0);
    std::vector<double> filt, avg;
    int i = 0;
    for (auto& f : tmp_frontiers_) {
      for (auto& c : f.filtered_cells_) filt.insert(filt.end(), { c(0), c(1), c(2) });
      avg.insert(avg.end(), { f.average_(0), f.average_(1), f.average_(2) });
      fo[i + 1] = fo[i] + (int)f.filtered_cells_.size();
      ++i;
    }
    std::vector<double> pos(3 * (size_t)n * nc), yaw((size_t)n * nc);
    std::vector<int32_t> vis((size_t)n * nc);
    if (n > 0)
      fuelgpu_check(fuelgpu_frontier_sample_viewpoints(gpu(), n, fo.data(), filt.data(), avg.data(), &view_, nc, pos.data(),
                                                       yaw.data(), vis.data()),
                    gpu());
    i = 0;
    for (auto& f : tmp_frontiers_) {
      for (int k = 0; k < nc; ++k) {
        const size_t o = (size_t)i * nc + k;
        if (vis[o] > min_visib_num_) {  // :688
          Viewpoint vp;
          for (int d = 0; d < 3; ++d) vp.pos_(d) = pos[3 * o + d];
          vp.yaw_ = yaw[o];
          vp.visib_num_ = vis[o];
          f.viewpoints_.push_back(vp);
        }
      }
      if (!f.viewpoints_.empty()) {
        auto inserted = frontiers_.insert(frontiers_.end(), f);
        std::sort(inserted->viewpoints_.begin(), inserted->viewpoints_.end(),
                  [](const Viewpoint& a, const Viewpoint& b) { return a.visib_num_ > b.visib_num_; });  // :404-406
        if (first_new_ftr_ == frontiers_.end()) first_new_ftr_ = inserted;
      } else
        dormant_frontiers_.push_back(f);
      ++i;
    }
    int idx = 0;
    for (auto& ft : frontiers_) ft.id_ = idx++;
  }
  std::list<Frontier>::iterator first_new_ftr_;

  // updateFrontierCostMatrix (frontier_finder.cpp:260-326): erase the removed clusters' entries (removed_ids_ are
  // indices after the removal), then every old x new and new x new pair in one ViewNode::costBatch, appended in the
  // reference's order
  void updateFrontierCostMatrix() {
    if (!removed_ids_.empty()) {
      for (auto it = frontiers_.begin(); it != first_new_ftr_; ++it)
        for (int r : removed_ids_) {
          auto c = it->costs_.begin();
          auto p = it->paths_.begin();
          std::advance(c, r);
          std::advance(p, r);
          it->costs_.erase(c);
          it->paths_.erase(p);
        }
      removed_ids_.clear();
    }
    typedef std::list<Frontier>::iterator It;
    std::vector<std::pair<It, It>> pairs;
    for (It i = frontiers_.begin(); i != first_new_ftr_; ++i)
      for (It j = first_new_ftr_; j != frontiers_.end(); ++j) pairs.push_back({ i, j });
    for (It i = first_new_ftr_; i != frontiers_.end(); ++i)
      for (It j = i; j != frontiers_.end(); ++j) pairs.push_back({ i, j });
    std::vector<Vector3d> p1, p2, v1;
    std::vector<double> y1, y2, cost;
    for (auto& e : pairs)
      if (e.first != e.second) {
        p1.push_back(e.first->viewpoints_.front().pos_), y1.push_back(e.first->viewpoints_.front().yaw_);
        p2.push_back(e.second->viewpoints_.front().pos_), y2.push_back(e.second->viewpoints_.front().yaw_);
        v1.push_back(Vector3d(0, 0, 0));
      }
    std::vector<std::vector<Vector3d>> paths;
    if (!p1.empty()) ViewNode::costBatch(p1, p2, y1, y2, v1, cost, paths);
    size_t k = 0;
    for (auto& e : pairs) {
      if (e.first == e.second) {
        e.first->costs_.push_back(0);
        e.first->paths_.push_back({});
        continue;
      }
      e.first->costs_.push_back(cost[k]);
      e.first->paths_.push_back(paths[k]);
      std::reverse(paths[k].begin(), paths[k].end());
      e.second->costs_.push_back(cost[k]);
      e.second->paths_.push_back(paths[k]);
      ++k;
    }
  }
  // getFullCostMatrix, the asymmetric form (frontier_finder.cpp:562-591): mat is (n + 1) x (n + 1), row-major
  void getFullCostMatrix(const Vector3d& cur_pos, const Vector3d& cur_vel, const Vector3d& cur_yaw,
                         std::vector<double>& mat) {
    const size_t n = frontiers_.size(), d = n + 1;
    mat.assign(d * d, 0.0);
    size_t i = 1;
    for (auto& f : frontiers_) {
      size_t j = 1;
      for (double c : f.costs_) mat[i * d + j++] = c;
      ++i;
    }
    for (size_t r = 0; r < d; ++r) mat[r * d] = 0.0;
    std::vector<Vector3d> p1(n, cur_pos), p2, v1(n, cur_vel);
    std::vector<double> y1(n, cur_yaw(0)), y2, cost;
    for (auto& f : frontiers_) p2.push_back(f.viewpoints_.front().pos_), y2.push_back(f.viewpoints_.front().yaw_);
    std::vector<std::vector<Vector3d>> paths;
    if (n) ViewNode::costBatch(p1, p2, y1, y2, v1, cost, paths);
    for (size_t j = 0; j < n; ++j) mat[j + 1] = cost[j];
  }
  // getPathForTour (frontier_finder.cpp:508-529)
  void getPathForTour(const Vector3d& pos, const std::vector<int>& frontier_ids, std::vector<Vector3d>& path) {
    std::vector<std::list<Frontier>::iterator> idx;
    for (auto it = frontiers_.begin(); it != frontiers_.end(); ++it) idx.push_back(it);
    std::vector<Vector3d> segment;
    ViewNode::searchPath(pos, idx[frontier_ids[0]]->viewpoints_.front().pos_, segment);
    path.insert(path.end(), segment.begin(), segment.end());
    for (size_t i = 0; i + 1 < frontier_ids.size(); ++i) {
      auto p = idx[frontier_ids[i]]->paths_.begin();
      std::advance(p, frontier_ids[i + 1]);
      path.insert(path.end(), p->begin(), p->end());
    }
  }

  // getTopViewpointsInfo (frontier_finder.cpp:425-450): each cluster's first viewpoint at least min_candidate_dist_
  // away, else its first
  void getTopViewpointsInfo(const Vector3d& cur_pos, std::vector<Vector3d>& points, std::vector<double>& yaws,
                            std::vector<Vector3d>& averages) const {
    points.clear(), yaws.clear(), averages.clear();
    for (const auto& f : frontiers_) {
      const Viewpoint* v = &f.viewpoints_.front();  // all too close: the first (highest coverage)
      for (const auto& w : f.viewpoints_) {
        if (dist(w.pos_, cur_pos) < p_.min_candidate_dist_) continue;
        v = &w;
        break;
      }
      points.push_back(v->pos_), yaws.push_back(v->yaw_), averages.push_back(f.average_);
    }
  }
  // getViewpointsInfo (frontier_finder.cpp:452-484): for each id, up to view_num viewpoints while visib_num_ stays above
  // int(front visib_num_ * max_decay), the too-close ones skipped unless that leaves none
  void getViewpointsInfo(const Vector3d& cur_pos, const std::vector<int>& ids, const int& view_num,
                         const double& max_decay, std::vector<std::vector<Vector3d>>& points,
                         std::vector<std::vector<double>>& yaws) const {
    points.clear(), yaws.clear();
    for (int id : ids)
      for (const auto& f : frontiers_) {
        if (f.id_ != id) continue;
        std::vector<Vector3d> pts;
        std::vector<double> ys;
        const int visib_thresh = f.viewpoints_.front().visib_num_ * max_decay;
        for (int pass = 0; pass < 2 && pts.empty(); ++pass)
          for (const auto& v : f.viewpoints_) {
            if ((int)pts.size() >= view_num || v.visib_num_ <= visib_thresh) break;
            if (pass == 0 && dist(v.pos_, cur_pos) < p_.min_candidate_dist_) continue;
            pts.push_back(v.pos_), ys.push_back(v.yaw_);
          }
        points.push_back(pts), yaws.push_back(ys);
      }
  }

  void getFrontiers(std::vector<std::vector<Vector3d>>& clusters) const {
    clusters.clear();
    for (auto& f : frontiers_) clusters.push_back(f.cells_);
  }
  void getDormantFrontiers(std::vector<std::vector<Vector3d>>& clusters) const {
    clusters.clear();
    for (auto& f : dormant_frontiers_) clusters.push_back(f.cells_);
  }

  std::list<Frontier> frontiers_, dormant_frontiers_, tmp_frontiers_;
  std::vector<int> removed_ids_;

private:
  FuelMap* gpu() const { return edt_env_->sdf_map_->gpu(); }
  static double dist(const Vector3d& a, const Vector3d& b) {  // (a - b).norm()
    const double x = a(0) - b(0), y = a(1) - b(1), z = a(2) - b(2);
    return std::sqrt((x * x + y * y) + z * z);
  }
  static bool haveOverlap(const Vector3d& min1, const Vector3d& max1, const Vector3d& min2, const Vector3d& max2) {
    for (int i = 0; i < 3; ++i) {  // frontier_finder.cpp:353-363
      const double bmin = std::max(min1[i], min2[i]), bmax = std::min(max1[i], max2[i]);
      if (bmin > bmax + 1e-3) return false;
    }
    return true;
  }
  void removeChanged(std::list<Frontier>& ftrs, const Vector3d& umin, const Vector3d& umax, bool record) {
    std::vector<std::list<Frontier>::iterator> cand;
    std::vector<int32_t> offs(1, 0), addr;
    for (auto it = ftrs.begin(); it != ftrs.end(); ++it)
      if (haveOverlap(it->box_min_, it->box_max_, umin, umax)) {
        cand.push_back(it);
        addr.insert(addr.end(), it->cell_addr_.begin(), it->cell_addr_.end());
        offs.push_back((int32_t)addr.size());
      }
    std::vector<uint8_t> changed(cand.size(), 0);
    if (!cand.empty())  // isFrontierChanged (:365-372) for all candidates in one call
      fuelgpu_check(fuelgpu_frontier_is_changed(gpu(), (int32_t)cand.size(), offs.data(), addr.data(), changed.data()), gpu());
    std::vector<int32_t> clear;
    size_t ci = 0;
    int rmv_idx = 0;
    for (auto it = ftrs.begin(); it != ftrs.end();) {
      const bool is_cand = ci < cand.size() && cand[ci] == it;
      if (is_cand && changed[ci]) {
        clear.insert(clear.end(), it->cell_addr_.begin(), it->cell_addr_.end());  // resetFlag (:62-69)
        it = ftrs.erase(it);
        if (record) removed_ids_.push_back(rmv_idx);
      } else {
        ++rmv_idx;
        ++it;
      }
      if (is_cand) ++ci;
    }
    if (!clear.empty()) fuelgpu_check(fuelgpu_frontier_clear_flags(gpu(), (int32_t)clear.size(), clear.data()), gpu());
  }
  std::shared_ptr<EDTEnvironment> edt_env_;
  FrontierParam p_;
};

// ---- FastExplorationManager's local tour (fast_exploration_manager.cpp:129-216, 429-503) --------------------------
// refineLocalTour with the reference's arguments plus ed_->refined_tour_, in one fuelgpu_local_tour_batch call with
// ViewNode's statics.  Returns the FUELGPU_TOUR_* status: FUELGPU_TOUR_UNREACHABLE leaves refined_pts empty and the tour
// {cur_pos}, where the reference's caller reads refined_points_[0] of an empty vector.  n_points must have at least one
// group and a nonempty last group (the reference dereferences a null final_node otherwise).  Afterwards
// ViewNode::astar_param_.lambda_heu is 10000, as the reference leaves ViewNode::astar_->lambda_heu_ (:499).
inline int refineLocalTour(const Vector3d& cur_pos, const Vector3d& cur_vel, const Vector3d& cur_yaw,
                           const std::vector<std::vector<Vector3d>>& n_points,
                           const std::vector<std::vector<double>>& n_yaws, std::vector<Vector3d>& refined_pts,
                           std::vector<double>& refined_yaws, std::vector<Vector3d>& refined_tour) {
  FuelMap* h = ViewNode::map_->gpu();
  const int32_t G = (int32_t)n_points.size();
  std::vector<int32_t> group_off(1, 0);
  std::vector<double> vp, vy;
  for (int i = 0; i < G; ++i) {
    for (size_t j = 0; j < n_points[i].size(); ++j)
      vp.insert(vp.end(), { n_points[i][j](0), n_points[i][j](1), n_points[i][j](2) }), vy.push_back(n_yaws[i][j]);
    group_off.push_back((int32_t)vy.size());
  }
  const int32_t prob_off[2] = { 0, G };
  const auto& a = ViewNode::astar_param_;
  const FuelLocalTourParams prm{ { ViewNode::vm_, ViewNode::yd_, ViewNode::w_dir_,
                                   { 0.4, a.lambda_heu, a.allocate_num, a.max_iter } },
                                 1.0 };  // ViewNode::astar_->lambda_heu_ = 1.0 for the tour (:490)
  FuelLocalTourInfo info;
  std::vector<int32_t> refined(std::max(G, 1));
  std::vector<double> tour;
  for (int32_t tour_max = 256;;) {  // a tour longer than tour_max rows: run again with room for it
    tour.assign(3 * (size_t)tour_max, 0.0);
    fuelgpu_check(fuelgpu_local_tour_batch(h, 1, prob_off, group_off.data(), cur_pos.data(), cur_vel.data(),
                                           &cur_yaw(0), vp.data(), vy.data(), &prm, &info, std::max(G, 1),
                                           refined.data(), tour_max, tour.data(), nullptr),
                  h);
    if (info.status != FUELGPU_TOUR_TRUNCATED) break;
    tour_max = info.n_tour;
  }
  refined_pts.clear(), refined_yaws.clear(), refined_tour.clear();
  for (int i = 0; i < info.n_refined; ++i)
    refined_pts.push_back(Vector3d(vp[3 * refined[i]], vp[3 * refined[i] + 1], vp[3 * refined[i] + 2])),
        refined_yaws.push_back(vy[refined[i]]);
  for (int i = 0; i < info.n_tour; ++i) refined_tour.push_back(Vector3d(tour[3 * i], tour[3 * i + 1], tour[3 * i + 2]));
  ViewNode::astar_param_.lambda_heu = 10000;  // ViewNode::astar_->lambda_heu_ = 10000 (:499)
  return info.status;
}

// planExploreMotion's one-frontier pick (:202-214): the first strict minimum of computeCost(pos, p, yaw[0], y, vel)
// below 100000 over the frontier's viewpoints, in one ViewNode::costBatch call; -1 when there is none (the reference
// then indexes n_points_[0][-1])
inline int pickOneViewpoint(const Vector3d& pos, const Vector3d& vel, const Vector3d& yaw,
                            const std::vector<Vector3d>& points, const std::vector<double>& yaws) {
  if (points.empty()) return -1;
  const size_t n = points.size();
  std::vector<double> cost;
  std::vector<std::vector<Vector3d>> paths;
  ViewNode::costBatch(std::vector<Vector3d>(n, pos), points, std::vector<double>(n, yaw(0)), yaws,
                      std::vector<Vector3d>(n, vel), cost, paths);
  double min_cost = 100000;
  int min_cost_id = -1;
  for (size_t i = 0; i < n; ++i)
    if (cost[i] < min_cost) min_cost = cost[i], min_cost_id = (int)i;
  return min_cost_id;
}

// FastExplorationManager::findGlobalTour (:327-427) over the finder's frontier list: updateFrontierCostMatrix,
// getFullCostMatrix, then the ATSP it writes for LKH solved exactly in one fuelgpu_global_tour_batch call (the
// lexicographically smallest optimal tour), then getPathForTour into global_tour.  Returns the FUELGPU_GTOUR_* status;
// on FUELGPU_GTOUR_BAD_INPUT (a cost whose int(cost * 100) is undefined) and FUELGPU_GTOUR_TOO_LARGE (more than
// FUELGPU_GTOUR_MAX_CLUSTERS clusters: keep LKH for such a list) indices and global_tour are left empty.
inline int findGlobalTour(FrontierFinder& ff, const Vector3d& cur_pos, const Vector3d& cur_vel,
                          const Vector3d& cur_yaw, std::vector<int>& indices, std::vector<Vector3d>& global_tour) {
  FuelMap* h = ViewNode::map_->gpu();  // the map the finder's costs are searched on
  ff.updateFrontierCostMatrix();
  std::vector<double> mat;
  ff.getFullCostMatrix(cur_pos, cur_vel, cur_yaw, mat);
  const int32_t dim = (int32_t)ff.frontiers_.size() + 1;
  FuelGlobalTourInfo info;
  std::vector<int32_t> ids((size_t)dim - 1);
  fuelgpu_check(fuelgpu_global_tour_batch(h, 1, &dim, mat.data(), &info, ids.data()), h);
  indices.clear(), global_tour.clear();
  if (info.status != FUELGPU_GTOUR_OK) return info.status;
  indices.assign(ids.begin(), ids.end());
  ff.getPathForTour(cur_pos, indices, global_tour);
  return info.status;
}

// ---- BsplineOptimizer (bspline_optimizer.h:20-145) -------------------------------------------------
class BsplineOptimizer {
public:
  static const int SMOOTHNESS = FUELGPU_SMOOTHNESS, DISTANCE = FUELGPU_DISTANCE, FEASIBILITY = FUELGPU_FEASIBILITY,
                   START = FUELGPU_START, END = FUELGPU_END, GUIDE = FUELGPU_GUIDE, WAYPOINTS = FUELGPU_WAYPOINTS,
                   VIEWCONS = FUELGPU_VIEWCONS, MINTIME = FUELGPU_MINTIME;
  static const int GUIDE_PHASE = SMOOTHNESS | GUIDE | START | END;                      // bspline_optimizer.cpp:20-21
  static const int NORMAL_PHASE = SMOOTHNESS | DISTANCE | FEASIBILITY | START | END;    // :22-23
  typedef std::unique_ptr<BsplineOptimizer> Ptr;

  void setEnvironment(const std::shared_ptr<EDTEnvironment>& env) { edt_environment_ = env; }
  void setParam(const FuelOptParams& p, const int max_iteration_num[4]) {  // :25-57
    params_ = p;
    for (int i = 0; i < 4; ++i) max_iteration_num_[i] = max_iteration_num[i];
    time_lb_ = -1;
  }
  void setBoundaryStates(const std::vector<Vector3d>& start, const std::vector<Vector3d>& end) {
    start_state_ = start;
    end_state_ = end;
  }
  void setTimeLowerBound(const double& lb) { time_lb_ = lb; }
  void setGuidePath(const std::vector<Vector3d>& guide_pt) { guide_pts_ = guide_pt; }
  void setWaypoints(const std::vector<Vector3d>& waypts, const std::vector<int>& waypt_idx) {
    waypoints_ = waypts;
    waypt_idx_ = waypt_idx;
  }
  // setViewConstraint (:91-93): the fields of ViewConstraint (traj_visibility.h:18-24) that calcViewCost reads
  void setViewConstraint(const Vector3d& pt, const Vector3d& dir, int idx) {
    view_pt_ = pt;
    view_dir_ = dir;
    view_idx_ = idx;
  }

  // optimize (:110-163): points = N x 3 control points, row-major; dt in/out.  The NLopt driver
  // loop (:165-253) runs on the device (fuelgpu_bspline_optimize_batch, B = 1).
  void optimize(std::vector<Vector3d>& points, double& dt, const int& cost_function, const int& max_num_id,
                const int& /*max_time_id*/) {
    if (start_state_.empty()) throw std::runtime_error("Initial state undefined!");  // :112-115
    const int n = (int)points.size();
    const bool optimize_time = cost_function & MINTIME;
    const int nvar = 3 * n + (optimize_time ? 1 : 0);
    std::vector<double> x(nvar);
    for (int i = 0; i < n; ++i)
      for (int k = 0; k < 3; ++k) x[3 * i + k] = points[i](k);
    if (optimize_time) x[nvar - 1] = dt;
    fillTrajConst(points, dt);
    FuelSolveParams sp{ max_iteration_num_[max_num_id], 6, 1e-5 };
    double fbest = 0;
    int32_t neval = 0;
    FuelMap* h = edt_environment_->sdf_map_->gpu();
    fuelgpu_check(fuelgpu_bspline_optimize_batch(h, 1, n, cost_function, &params_, &tc_, &sp, x.data(), &fbest, &neval), h);
    for (int i = 0; i < n; ++i)
      for (int k = 0; k < 3; ++k) points[i](k) = x[3 * i + k];
    if (optimize_time) dt = x[nvar - 1];
    iter_num_ = neval;
    min_cost_ = fbest;
    start_state_.clear();  // :161-162
    time_lb_ = -1;
  }
  // combineCost (:518-647) through the device, the costFunction trampoline (:693-706)
  double combineCost(const std::vector<double>& x, std::vector<double>& grad, int n_pts, int cost_function) {
    double f = 0;
    grad.resize(x.size());
    FuelMap* h = edt_environment_->sdf_map_->gpu();
    fuelgpu_check(fuelgpu_bspline_cost_batch(h, 1, n_pts, cost_function, &params_, &tc_, x.data(), &f, grad.data()), h);
    return f;
  }
  void fillTrajConst(const std::vector<Vector3d>& points, double dt) {
    std::memset(&tc_, 0, sizeof(tc_));
    double d = 0.0;  // pt_dist_ (:136-140)
    for (size_t i = 0; i + 1 < points.size(); ++i) {
      double s = 0;
      for (int k = 0; k < 3; ++k) s += (points[i + 1](k) - points[i](k)) * (points[i + 1](k) - points[i](k));
      d += std::sqrt(s);
    }
    tc_.pt_dist = d / double(points.size());
    tc_.knot_span = dt;
    for (size_t i = 0; i < start_state_.size() && i < 3; ++i)
      for (int k = 0; k < 3; ++k) tc_.start[i][k] = start_state_[i](k);
    tc_.n_end = (int32_t)std::min<size_t>(end_state_.size(), 3);
    for (int i = 0; i < tc_.n_end; ++i)
      for (int k = 0; k < 3; ++k) tc_.end[i][k] = end_state_[i](k);
    tc_.time_lb = time_lb_;
    tc_.n_guide = (int32_t)std::min<size_t>(guide_pts_.size(), FUELGPU_MAX_PTS);
    for (int i = 0; i < tc_.n_guide; ++i)
      for (int k = 0; k < 3; ++k) tc_.guide[i][k] = guide_pts_[i](k);
    tc_.n_waypt = (int32_t)std::min<size_t>(waypoints_.size(), FUELGPU_MAX_PTS);
    for (int i = 0; i < tc_.n_waypt; ++i) {
      for (int k = 0; k < 3; ++k) tc_.waypt[i][k] = waypoints_[i](k);
      tc_.waypt_idx[i] = waypt_idx_[i];
    }
    tc_.view_idx = view_idx_;
    for (int k = 0; k < 3; ++k) {
      tc_.view_pt[k] = view_pt_(k);
      tc_.view_dir[k] = view_dir_(k);
    }
  }
  int iter_num_ = 0;
  double min_cost_ = 0;

private:
  std::shared_ptr<EDTEnvironment> edt_environment_;
  FuelOptParams params_;
  FuelTrajConst tc_;
  int max_iteration_num_[4] = { 2, 2000, 200, 200 };
  std::vector<Vector3d> start_state_, end_state_, guide_pts_, waypoints_;
  std::vector<int> waypt_idx_;
  Vector3d view_pt_, view_dir_;
  int view_idx_ = -1;
  double time_lb_ = -1;
};

}  // namespace fast_planner
