// raycast.cuh -- the RayCaster walk over the resident occupancy byte, shared by the viewpoint visibility test
// (viewpoints.cu, FrontierFinder::countVisibleCells) and the path shortening after A* (astar.cu,
// FastExplorationManager::shortenPath).  Both call RayCaster::input(start, end) then nextId until it returns false, and
// stop at the first inflated-occupied or UNKNOWN voxel.
#pragma once
#include "common.cuh"

namespace {

__device__ __forceinline__ bool idx_in_map(const Geom& g, int x, int y, int z) {
  return !(x < 0 || y < 0 || z < 0 || x > g.nx - 1 || y > g.ny - 1 || z > g.nz - 1);
}

__device__ __forceinline__ double intbound(double s, double ds) {  // raycast.cpp:14-23
  if (ds < 0) {
    s = -s;
    ds = -ds;
  }
  s = fmod(fmod(s, 1.0) + 1.0, 1.0);
  return (1 - s) / ds;
}

// RayCaster::input(start, end) then nextId until the end voxel (raycast.cpp:329-394); blocked by an inflated-occupied or
// UNKNOWN voxel (voxels outside the map read -1 in the reference: neither).  Returns true when the ray is clear.
// kBox: a voxel outside the exploration box blocks too (!isInBox(idx), sdf_map.h:171-178), as ViewNode::searchPath's
// straight-line test has it (graph_node.cpp:36-43).
template <bool kBox = false>
__device__ bool ray_is_clear(const Geom& g, const uint8_t* __restrict__ occ, const double start[3], const double end[3]) {
  const double res = g.res;
  const double s0 = start[0] / res, s1 = start[1] / res, s2 = start[2] / res;
  int x = (int)floor(s0), y = (int)floor(s1), z = (int)floor(s2);
  const int ex = (int)floor(end[0] / res), ey = (int)floor(end[1] / res), ez = (int)floor(end[2] / res);
  const double dx = ex - x, dy = ey - y, dz = ez - z;
  const int sx = dx == 0 ? 0 : (dx < 0 ? -1 : 1), sy = dy == 0 ? 0 : (dy < 0 ? -1 : 1), sz = dz == 0 ? 0 : (dz < 0 ? -1 : 1);
  double tmx = intbound(s0, dx), tmy = intbound(s1, dy), tmz = intbound(s2, dz);
  const double tdx = ((double)sx) / dx, tdy = ((double)sy) / dy, tdz = ((double)sz) / dz;
  const double o0 = 0.5 - g.origin[0] / res, o1 = 0.5 - g.origin[1] / res, o2 = 0.5 - g.origin[2] / res;  // raycast.cpp:323-327
  for (int guard = 0; guard < 4096; ++guard) {
    const int ix = (int)(x + o0), iy = (int)(y + o1), iz = (int)(z + o2);
    if (x == ex && y == ey && z == ez) return true;
    if (tmx < tmy) {
      if (tmx < tmz) {
        x += sx;
        tmx += tdx;
      } else {
        z += sz;
        tmz += tdz;
      }
    } else {
      if (tmy < tmz) {
        y += sy;
        tmy += tdy;
      } else {
        z += sz;
        tmz += tdz;
      }
    }
    if (idx_in_map(g, ix, iy, iz)) {
      const uint8_t o = occ[addr_of(g, ix, iy, iz)];
      if ((o & 4) || (o & 3) == FUELGPU_UNKNOWN) return false;
    }
    if (kBox && (ix < g.box_min[0] || ix >= g.box_max[0] || iy < g.box_min[1] || iy >= g.box_max[1] ||
                 iz < g.box_min[2] || iz >= g.box_max[2]))
      return false;
  }
  return true;
}

}  // namespace
