// Drives findGlobalTour of the C++ shim (include/fuelgpu_shim.hpp) on the scene of tests/shim_smoke.cpp over a
// hand-made list of five frontiers, each with one viewpoint, all new: updateFrontierCostMatrix, getFullCostMatrix, the
// device's exact ATSP, getPathForTour.  Writes the status, the tour, the full cost matrix and the global tour that
// tests/test_shim_gtour.py compares with the oracle and the Python findGlobalTour.
#include <cstdio>
#include <cstdlib>

#include "fuelgpu_shim.hpp"

using namespace fast_planner;

int main(int argc, char** argv) {
  const char* out_path = argc > 1 ? argv[1] : "shim_gtour_out.txt";
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

  std::shared_ptr<EDTEnvironment> env(new EDTEnvironment);
  env->setMap(map);
  FrontierFinder ff(env, FrontierParam());
  const double vps[5][4] = { { -1.6, 0.8, 0.6, 0.3 }, { 1.0, -1.2, 0.6, 0.0 }, { 1.5, 1.2, 0.6, 1.2 },
                             { 0.0, 0.0, 0.7, -2.8 }, { 1.8, 1.4, 0.6, 1.5 } };
  for (int i = 0; i < 5; ++i) {
    Frontier f;
    f.id_ = i;
    f.viewpoints_.push_back({ Vector3d(vps[i][0], vps[i][1], vps[i][2]), vps[i][3], 10 });
    ff.frontiers_.push_back(f);
  }
  ff.first_new_ftr_ = ff.frontiers_.begin();
  const Vector3d pos(-1.5, -1.2, 0.6), vel(0.5, 0.3, 0.0), yaw(0.2, 0.0, 0.0);
  std::vector<int> indices;
  std::vector<Vector3d> tour;
  const int status = findGlobalTour(ff, pos, vel, yaw, indices, tour);
  std::vector<double> mat;
  ff.getFullCostMatrix(pos, vel, yaw, mat);
  FILE* f = std::fopen(out_path, "w");
  std::fprintf(f, "%d %d %d\n", status, (int)indices.size(), (int)tour.size());
  for (int i : indices) std::fprintf(f, "%d ", i);
  std::fprintf(f, "\n");
  for (double c : mat) std::fprintf(f, "%.17g ", c);
  std::fprintf(f, "\n");
  for (const Vector3d& p : tour) std::fprintf(f, "%.17g %.17g %.17g\n", p(0), p(1), p(2));
  std::fclose(f);
  return 0;
}
