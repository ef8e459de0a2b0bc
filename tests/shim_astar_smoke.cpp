// Drives fast_planner::Astar of the C++ shim (include/fuelgpu_shim.hpp) the way planExploreMotion does:
// reset -> search(pos, next_pos) -> getPath -> pathLength, on the scene of tests/shim_smoke.cpp.  Writes one line per
// query (status, iter_num, use_node_num, path size, length, the path) that tests/test_shim_astar.py compares with the
// oracle.
#include <cstdio>
#include <cstdlib>

#include "fuelgpu_shim.hpp"

using namespace fast_planner;

int main(int argc, char** argv) {
  const char* out_path = argc > 1 ? argv[1] : "shim_astar_out.txt";
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
  std::shared_ptr<EDTEnvironment> env(new EDTEnvironment);
  env->setMap(map);

  AstarParam ap;
  ap.resolution_astar = 0.1;
  ap.lambda_heu = 10000.0;
  ap.allocate_num = 20000;
  ap.max_iter = 100000;
  Astar astar;
  astar.init(ap, env);
  const double q[4][6] = { { -1.5, -1.2, 0.6, 1.4, -1.2, 0.6 },  // past the wall
                           { -1.5, 0.0, 0.6, -0.9, 0.4, 0.7 },   // close
                           { -1.5, -1.2, 0.6, 0.0, 0.0, 0.7 },   // into the unknown ball
                           { 1.2, -1.0, 0.4, 1.2, -1.0, 0.4 } };  // start == goal
  FILE* f = std::fopen(out_path, "w");
  for (int k = 0; k < 4; ++k) {
    astar.reset();
    const int st = astar.search(Vector3d(q[k][0], q[k][1], q[k][2]), Vector3d(q[k][3], q[k][4], q[k][5]));
    const std::vector<Vector3d> path = astar.getPath();
    std::fprintf(f, "query %d %d %d %d %.17g", st, astar.iter_num(), astar.use_node_num(), (int)path.size(),
                 Astar::pathLength(path));
    for (const Vector3d& p : path) std::fprintf(f, " %.17g %.17g %.17g", p(0), p(1), p(2));
    std::fprintf(f, "\n");
  }
  std::fclose(f);
  return 0;
}
