// Drives fast_planner::KinodynamicAstar of the C++ shim (include/fuelgpu_shim.hpp) the way kinodynamicReplan uses
// kino_path_finder_: reset -> search(pos, vel, acc, goal) -> getSamples, on the scene of tests/shim_smoke.cpp (optimistic).
// Writes one line per query (status, retried, use_node_num, samples?, K, ts, the samples) that tests/test_shim_kino.py
// compares with the oracle.
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

  FuelKinoParams kp{ 0.8, 1.0, 2.0, 0.25, 2.0, 10.0, 5.0, 10.0, 0.025, 0.35, 2.0, 100000, 10, 1, 0 };
  KinodynamicAstar kino;
  kino.setParam(kp);
  kino.setEnvironment(env);
  kino.init();
  const double q[4][9] = { { -1.5, -1.2, 0.6, 0.5, 0.0, 0.0, 0.0, 0.0, 0.0 },     // towards the wall
                           { -1.5, 0.0, 0.6, 0.0, 0.0, 0.0, 0.0, 0.3, 0.0 },      // a short hop
                           { -1.5, -1.2, 0.6, 0.0, 0.5, 0.0, 0.2, 0.0, 0.0 },
                           { 1.2, -1.0, 0.4, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0 } };    // start == goal: Close goal
  const double goal[4][3] = { { 1.4, -1.2, 0.6 }, { -0.9, 0.4, 0.7 }, { -0.2, 0.5, 0.8 }, { 1.2, -1.0, 0.4 } };
  FILE* f = std::fopen(out_path, "w");
  for (int k = 0; k < 4; ++k) {
    kino.reset();
    const int st = kino.search(Vector3d(q[k][0], q[k][1], q[k][2]), Vector3d(q[k][3], q[k][4], q[k][5]),
                               Vector3d(q[k][6], q[k][7], q[k][8]), Vector3d(goal[k][0], goal[k][1], goal[k][2]));
    double ts = 0.0;
    std::vector<Vector3d> pts, der;
    const bool ok = kino.getSamples(ts, pts, der);
    std::fprintf(f, "query %d %d %d %d %d %.17g", st, kino.info().retried, kino.info().use_node_num, ok ? 1 : 0,
                 (int)pts.size(), ts);
    for (const Vector3d& p : pts) std::fprintf(f, " %.17g %.17g %.17g", p(0), p(1), p(2));
    std::fprintf(f, "\n");
  }
  std::fclose(f);
  return 0;
}
