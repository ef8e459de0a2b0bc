// Drives the local tour of the C++ shim (include/fuelgpu_shim.hpp) the way planExploreMotion does: refineLocalTour over
// three groups of viewpoints, then the one-viewpoint pick, on the scene of tests/shim_smoke.cpp, and
// FrontierFinder::getViewpointsInfo / getTopViewpointsInfo on a hand-made frontier list.  Writes the status, the refined
// points and yaws, the tour rows, the pick, ViewNode's lambda_heu afterwards and the two viewpoint lists that
// tests/test_shim_tour.py compares with the oracle and the Python bookkeeping.
#include <cstdio>
#include <cstdlib>

#include "fuelgpu_shim.hpp"

using namespace fast_planner;

int main(int argc, char** argv) {
  const char* out_path = argc > 1 ? argv[1] : "shim_tour_out.txt";
  MapParam mp;
  mp.map_voxel_num_ = Vector3i(48, 40, 24);
  mp.resolution_ = 0.1;
  mp.map_origin_ = Vector3d(-2.4, -2.0, -0.5);
  mp.box_mind_ = Vector3d(-2.2, -1.8, -0.3);
  mp.box_maxd_ = Vector3d(2.2, 1.8, 1.7);
  mp.optimistic_ = true;
  std::shared_ptr<SDFMap> map(new SDFMap);
  try {
    map->initMap(mp);
  } catch (const FuelGpuError& e) {
    std::printf("initMap failed (code %d): %s\n", e.code, e.what());
    return e.code == FUELGPU_ENODEVICE ? 42 : 1;
  }
  const double clamp_min = std::log(0.12 / 0.88);
  for (int x = 0; x < 48; ++x)
    for (int y = 0; y < 40; ++y)
      for (int z = 0; z < 24; ++z) {
        const int a = map->toAddress(x, y, z);
        const bool known = x >= 4 && x < 44 && y >= 4 && y < 36 && z >= 2 && z < 22;
        const int dx = x - 24, dy = y - 20, dz = z - 12;
        const bool ball = dx * dx + dy * dy + 2 * dz * dz < 81;
        const bool wall = x >= 12 && x <= 13 && y >= 8 && y < 30 && z < 18;
        if (known && !ball) map->occupancy_buffer_[a] = wall ? 3.0 : clamp_min;
        if (known && !ball && wall) map->occupancy_buffer_inflate_[a] = 1;
      }
  map->update_min_ = mp.map_origin_;
  map->update_max_ = Vector3d(2.4, 2.0, 1.9);
  map->updateESDF3d();  // uploads the occupancy
  ViewNode::map_ = map;
  ViewNode::astar_param_ = { 0.4, 10000.0, 20000, 2000 };

  const std::vector<std::vector<Vector3d>> n_points = {
    { Vector3d(-1.6, 0.8, 0.6), Vector3d(-1.2, 1.2, 0.7), Vector3d(-1.7, -0.6, 0.5) },
    { Vector3d(1.0, -1.2, 0.6), Vector3d(1.5, 1.2, 0.6), Vector3d(0.0, 0.0, 0.7), Vector3d(1.6, -0.4, 0.8) },
    { Vector3d(1.8, 1.4, 0.6), Vector3d(-1.0, 0.0, 0.6) }
  };
  const std::vector<std::vector<double>> n_yaws = { { 0.3, -1.0, 2.5 }, { 0.0, 1.2, -2.8, 0.6 }, { 1.5, 0.0 } };
  const Vector3d pos(-1.5, -1.2, 0.6), vel(0.5, 0.3, 0.0), yaw(0.2, 0.0, 0.0);
  std::vector<Vector3d> pts, tour;
  std::vector<double> ys;
  const int status = refineLocalTour(pos, vel, yaw, n_points, n_yaws, pts, ys, tour);
  const int pick = pickOneViewpoint(pos, vel, yaw, n_points[1], n_yaws[1]);
  FILE* f = std::fopen(out_path, "w");
  std::fprintf(f, "%d %d %d %d %.17g\n", status, (int)pts.size(), (int)tour.size(), pick,
               ViewNode::astar_param_.lambda_heu);
  for (size_t i = 0; i < pts.size(); ++i) std::fprintf(f, "%.17g %.17g %.17g %.17g\n", pts[i](0), pts[i](1), pts[i](2), ys[i]);
  for (const auto& r : tour) std::fprintf(f, "%.17g %.17g %.17g\n", r(0), r(1), r(2));

  // a hand-made frontier list: (pos, yaw, visib_num_) of each viewpoint, best first
  std::shared_ptr<EDTEnvironment> env(new EDTEnvironment);
  env->setMap(map);
  FrontierFinder ff(env, FrontierParam());
  const double views[3][4][5] = { { { 3.0, 0.0, 1.0, 0.0, 10 }, { 4.0, 0.0, 1.0, 0.1, 9 }, { 5.0, 0.0, 1.0, 0.2, 8 },
                                    { 6.0, 0.0, 1.0, 0.3, 7 } },
                                  { { 0.0, 0.0, 1.0, 0.0, 20 }, { 0.1, 0.0, 1.0, 0.2, 19 }, { 0.2, 0.0, 1.0, 0.4, 18 },
                                    { 0.3, 0.0, 1.0, 0.6, 15 } },
                                  { { 0.2, 0.0, 1.0, 0.0, 30 }, { 2.0, 0.0, 1.0, 0.5, 29 }, { 0.3, 0.0, 1.0, 0.7, 28 },
                                    { 4.0, 0.0, 1.0, 0.9, 27 } } };
  for (int i = 0; i < 3; ++i) {
    Frontier fr;
    fr.id_ = i;
    for (int j = 0; j < 4; ++j)
      fr.viewpoints_.push_back({ Vector3d(views[i][j][0], views[i][j][1], views[i][j][2]), views[i][j][3],
                                 (int)views[i][j][4] });
    ff.frontiers_.push_back(fr);
  }
  const Vector3d cur(0.0, 0.0, 1.0);
  std::vector<std::vector<Vector3d>> vpts;
  std::vector<std::vector<double>> vys;
  ff.getViewpointsInfo(cur, { 2, 0, 1, 7 }, 15, 0.8, vpts, vys);
  std::fprintf(f, "V %d\n", (int)vpts.size());
  for (size_t g = 0; g < vpts.size(); ++g) {
    std::fprintf(f, "%d", (int)vpts[g].size());
    for (size_t j = 0; j < vpts[g].size(); ++j)
      std::fprintf(f, " %.17g %.17g %.17g %.17g", vpts[g][j](0), vpts[g][j](1), vpts[g][j](2), vys[g][j]);
    std::fprintf(f, "\n");
  }
  std::vector<Vector3d> tpts, avgs;
  std::vector<double> tys;
  ff.getTopViewpointsInfo(cur, tpts, tys, avgs);
  std::fprintf(f, "T %d\n", (int)tpts.size());
  for (size_t i = 0; i < tpts.size(); ++i) std::fprintf(f, "%.17g %.17g %.17g %.17g\n", tpts[i](0), tpts[i](1), tpts[i](2), tys[i]);
  std::fclose(f);
  return 0;
}
