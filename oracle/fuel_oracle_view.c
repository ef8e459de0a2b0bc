/* CPU restatement of ViewNode::searchPath and ViewNode::computeCost (active_perception/src/graph_node.cpp:32-85): the
 * straight-line test over the occupancy byte the device reads (bits 0-1 tri-state, bit 2 inflate) with the box test of
 * searchPath, then Astar::search of the A* oracle (orc_astar, fuel_oracle_astar.c) when the line is blocked, then the
 * cost.  TEST INFRASTRUCTURE ONLY (tests/test_oracle_view_cost.py pins it to the compiled reference, the GPU tests
 * compare the device with it). */
#include "fuel_oracle_view.h"

#include <math.h>
#include <stdlib.h>
#include <string.h>

static double norm3(double x, double y, double z) { return sqrt((x * x + y * y) + z * z); }

static double intbound(double s, double ds) { /* raycast.cpp:14-23 */
  if (ds < 0) {
    s = -s;
    ds = -ds;
  }
  s = fmod(fmod(s, 1.0) + 1.0, 1.0);
  return (1 - s) / ds;
}

/* RayCaster::input(a, b) + nextId until the end voxel (raycast.cpp:329-394); a voxel blocks the line when it is
 * inflated-occupied or UNKNOWN (outside the map both read -1: neither) or outside the exploration box
 * (!isInBox(idx), sdf_map.h:171-178, with box_min_ / box_max_ = posToIndex(box_mind_ / box_maxd_), sdf_map.cpp:83-84).
 * Bounded like the device's walk: a line that misses its end voxel counts as clear after 4096 steps. */
static int line_blocked(const OrcAstarMap* m, const double a[3], const double b[3]) {
  const double res = m->res;
  int bmin[3], bmax[3];
  for (int k = 0; k < 3; ++k) {
    bmin[k] = (int)floor((m->box_mind[k] - m->origin[k]) * m->res_inv);
    bmax[k] = (int)floor((m->box_maxd[k] - m->origin[k]) * m->res_inv);
  }
  const double s0 = a[0] / res, s1 = a[1] / res, s2 = a[2] / res;
  int x = (int)floor(s0), y = (int)floor(s1), z = (int)floor(s2);
  const int ex = (int)floor(b[0] / res), ey = (int)floor(b[1] / res), ez = (int)floor(b[2] / res);
  const double dx = ex - x, dy = ey - y, dz = ez - z;
  const int sx = dx == 0 ? 0 : (dx < 0 ? -1 : 1), sy = dy == 0 ? 0 : (dy < 0 ? -1 : 1), sz = dz == 0 ? 0 : (dz < 0 ? -1 : 1);
  double tmx = intbound(s0, dx), tmy = intbound(s1, dy), tmz = intbound(s2, dz);
  const double tdx = ((double)sx) / dx, tdy = ((double)sy) / dy, tdz = ((double)sz) / dz;
  const double o0 = 0.5 - m->origin[0] / res, o1 = 0.5 - m->origin[1] / res, o2 = 0.5 - m->origin[2] / res;
  for (int guard = 0; guard < 4096; ++guard) {
    const int id[3] = { (int)(x + o0), (int)(y + o1), (int)(z + o2) };
    if (x == ex && y == ey && z == ez) return 0;
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
    int in_map = 1;
    for (int k = 0; k < 3; ++k)
      if (id[k] < 0 || id[k] > m->n[k] - 1) in_map = 0;
    if (in_map) {
      const uint8_t o = m->occ[((int64_t)id[0] * m->n[1] + id[1]) * m->n[2] + id[2]];
      if ((o & 4) || (o & 3) == 0) return 1;
    }
    for (int k = 0; k < 3; ++k)
      if (id[k] < bmin[k] || id[k] >= bmax[k]) return 1;
  }
  return 0;
}

int orc_view_cost(const OrcAstarMap* m, const double p1[3], const double p2[3], double y1, double y2, const double v1[3],
                  double vm, double yd, double w_dir, double resolution, double lambda, int32_t allocate_num,
                  int32_t max_iter, OrcViewCostInfo* inf, int32_t path_max, double* path) {
  memset(inf, 0, sizeof(*inf));
  if (path) memset(path, 0, sizeof(double) * 3 * (size_t)path_max);
  int finite = isfinite(y1) && isfinite(y2);
  for (int k = 0; k < 3; ++k) finite = finite && isfinite(p1[k]) && isfinite(p2[k]) && isfinite(v1[k]);
  if (!finite) {
    inf->reason = 5;
    return 0;
  }
  /* searchPath (graph_node.cpp:32-61) */
  int two = 1;
  if (!line_blocked(m, p1, p2)) {
    inf->kind = 1;
    inf->length = norm3(p1[0] - p2[0], p1[1] - p2[1], p1[2] - p2[2]);
  } else {
    /* a search holds at most 1 + 26 * max_iter nodes: the clamped pool ends it where allocate_num does */
    const long long cap = 26LL * max_iter + 2;
    const int32_t A = allocate_num < cap ? allocate_num : (int32_t)cap;
    double* full = malloc(sizeof(double) * 3 * ((size_t)A + 1));
    double wp[32 * 3];
    OrcPathInfo pi;
    if (!full || orc_astar(m, p1, p2, resolution, lambda, A, max_iter, 32, &pi, A + 1, full, wp) < 0) {
      free(full);
      return -1;
    }
    inf->reason = pi.reason, inf->iter_num = pi.iter_num, inf->use_node_num = pi.use_node_num;
    if (pi.status == 1) {
      inf->kind = 2;
      inf->n_path = pi.n_path;
      double len = 0.0; /* Astar::pathLength (astar2.cpp:169-175) */
      for (int j = 0; j + 1 < pi.n_path; ++j)
        len += norm3(full[3 * j + 3] - full[3 * j], full[3 * j + 4] - full[3 * j + 1], full[3 * j + 5] - full[3 * j + 2]);
      inf->length = len;
      if (path)
        for (int r = 0; r < path_max && r < pi.n_path; ++r) memcpy(path + 3 * r, full + 3 * r, sizeof(double) * 3);
      two = 0;
    } else {
      inf->kind = 3;
      inf->length = 1000;
    }
    free(full);
  }
  if (two) {
    inf->n_path = 2;
    if (path && path_max > 0) memcpy(path, p1, sizeof(double) * 3);
    if (path && path_max > 1) memcpy(path + 3, p2, sizeof(double) * 3);
  }
  /* computeCost (:63-85) */
  double pos_cost = inf->length / vm;
  if (norm3(v1[0], v1[1], v1[2]) > 1e-3) {
    double dir[3] = { p2[0] - p1[0], p2[1] - p1[1], p2[2] - p1[2] }, vdir[3] = { v1[0], v1[1], v1[2] };
    const double zd = (dir[0] * dir[0] + dir[1] * dir[1]) + dir[2] * dir[2];
    if (zd > 0.0) {
      const double n = sqrt(zd);
      dir[0] /= n, dir[1] /= n, dir[2] /= n;
    }
    const double zv = (vdir[0] * vdir[0] + vdir[1] * vdir[1]) + vdir[2] * vdir[2];
    if (zv > 0.0) {
      const double n = sqrt(zv);
      vdir[0] /= n, vdir[1] /= n, vdir[2] /= n;
    }
    pos_cost += w_dir * acos((vdir[0] * dir[0] + vdir[1] * dir[1]) + vdir[2] * dir[2]);
  }
  double diff = fabs(y2 - y1);
  const double other = 2 * M_PI - diff;
  diff = other < diff ? other : diff; /* std::min(diff, 2 * M_PI - diff) */
  const double yaw_cost = diff / yd;
  inf->cost = pos_cost < yaw_cost ? yaw_cost : pos_cost; /* std::max */
  return 0;
}
