/* CPU restatement of Astar::search (path_searching/src/astar2.cpp:47-149, backtrack :177-186, getDiagHeu :192-212),
 * FastExplorationManager::shortenPath (exploration_manager/src/fast_exploration_manager.cpp:295-325) and the goal branch
 * of planExploreMotion (:238-263), over the occupancy byte the device reads (bits 0-1 tri-state, bit 2 inflate).
 * The open set is libstdc++'s std::priority_queue (push_heap / pop_heap -> __adjust_heap -> __push_heap) over node ids,
 * compared through each node's current f; open_set_map_ and close_set_map_ are one open-addressing table keyed by the
 * node index.  The wall-clock cut is the iteration cap max_iter; the open set holds at most 2 * allocate_num entries.
 * TEST INFRASTRUCTURE ONLY (tests/test_oracle_astar.py pins it to the compiled reference, the GPU tests compare the
 * device with it). */
#include "fuel_oracle_astar.h"

#include <math.h>
#include <stdlib.h>
#include <string.h>

typedef struct {
  int x, y, z, w; /* w = 2 * node id + closed, -1 empty */
} Slot;

static double norm3(double x, double y, double z) { return sqrt((x * x + y * y) + z * z); }

static double diag_heu(const double a[3], const double b[3]) {
  double dx = fabs(a[0] - b[0]), dy = fabs(a[1] - b[1]), dz = fabs(a[2] - b[2]);
  double h = 0.0;
  const double diag = fmin(fmin(dx, dy), dz);
  dx -= diag;
  dy -= diag;
  dz -= diag;
  if (dx < 1e-4) h = 1.0 * sqrt(3.0) * diag + sqrt(2.0) * fmin(dy, dz) + 1.0 * fabs(dy - dz);
  if (dy < 1e-4) h = 1.0 * sqrt(3.0) * diag + sqrt(2.0) * fmin(dx, dz) + 1.0 * fabs(dx - dz);
  if (dz < 1e-4) h = 1.0 * sqrt(3.0) * diag + sqrt(2.0) * fmin(dx, dy) + 1.0 * fabs(dx - dy);
  return (1.0 + 1.0 / 1000) * h;
}

static int in_map(const OrcAstarMap* m, const int id[3]) {
  for (int k = 0; k < 3; ++k)
    if (id[k] < 0 || id[k] > m->n[k] - 1) return 0;
  return 1;
}
static int blocked_idx(const OrcAstarMap* m, const int id[3]) {
  if (!in_map(m, id)) return 0; /* getInflateOccupancy / getOccupancy read -1 outside */
  const uint8_t o = m->occ[((int64_t)id[0] * m->n[1] + id[1]) * m->n[2] + id[2]];
  return (o & 4) || (o & 3) == 0;
}
static int blocked(const OrcAstarMap* m, const double p[3]) {
  int id[3];
  for (int k = 0; k < 3; ++k) id[k] = (int)floor((p[k] - m->origin[k]) * m->res_inv);
  return blocked_idx(m, id);
}
static void node_index(const OrcAstarMap* m, double inv, const double p[3], int id[3]) {
  for (int k = 0; k < 3; ++k) id[k] = (int)floor((p[k] - m->origin[k]) * inv);
}

static unsigned key_hash(const int id[3]) {
  unsigned h = (unsigned)id[0] * 73856093u ^ (unsigned)id[1] * 19349663u ^ (unsigned)id[2] * 83492791u;
  h ^= h >> 15;
  h *= 0x2c1b3c6du;
  h ^= h >> 12;
  return h;
}
static int tab_find(const Slot* t, unsigned mask, const int id[3]) {
  for (unsigned s = key_hash(id) & mask;; s = (s + 1) & mask) {
    if (t[s].w < 0) return -1;
    if (t[s].x == id[0] && t[s].y == id[1] && t[s].z == id[2]) return (int)s;
  }
}
static int tab_insert(Slot* t, unsigned mask, const int id[3], int w) {
  unsigned s = key_hash(id) & mask;
  while (t[s].w >= 0) s = (s + 1) & mask;
  t[s].x = id[0], t[s].y = id[1], t[s].z = id[2], t[s].w = w;
  return (int)s;
}

/* libstdc++ __push_heap with NodeComparator0 (node1->f_score > node2->f_score) */
static void sift_up(int* heap, const double* f, int hole, int v) {
  int parent = (hole - 1) / 2;
  while (hole > 0 && f[heap[parent]] > f[v]) {
    heap[hole] = heap[parent];
    hole = parent;
    parent = (hole - 1) / 2;
  }
  heap[hole] = v;
}
/* pop_heap: __pop_heap -> __adjust_heap(first, 0, len - 1, last) */
static void heap_pop(int* heap, int len, const double* f) {
  if (len <= 1) return;
  const int n = len - 1, v = heap[n];
  heap[n] = heap[0];
  int hole = 0, child = 0;
  while (child < (n - 1) / 2) {
    child = 2 * (child + 1);
    if (f[heap[child]] > f[heap[child - 1]]) child--;
    heap[hole] = heap[child];
    hole = child;
  }
  if ((n & 1) == 0 && child == (n - 2) / 2) {
    child = 2 * (child + 1);
    heap[hole] = heap[child - 1];
    hole = child - 1;
  }
  sift_up(heap, f, hole, v);
}

/* RayCaster::input(a, b) + nextId until the end voxel (raycast.cpp:14-23, 329-394), blocked as shortenPath tests */
static double intbound(double s, double ds) {
  if (ds < 0) {
    s = -s;
    ds = -ds;
  }
  s = fmod(fmod(s, 1.0) + 1.0, 1.0);
  return (1 - s) / ds;
}
static int ray_blocked(const OrcAstarMap* m, const double a[3], const double b[3]) {
  const double res = m->res;
  const double s0 = a[0] / res, s1 = a[1] / res, s2 = a[2] / res;
  int x = (int)floor(s0), y = (int)floor(s1), z = (int)floor(s2);
  const int ex = (int)floor(b[0] / res), ey = (int)floor(b[1] / res), ez = (int)floor(b[2] / res);
  const double dx = ex - x, dy = ey - y, dz = ez - z;
  const int sx = dx == 0 ? 0 : (dx < 0 ? -1 : 1), sy = dy == 0 ? 0 : (dy < 0 ? -1 : 1), sz = dz == 0 ? 0 : (dz < 0 ? -1 : 1);
  double tmx = intbound(s0, dx), tmy = intbound(s1, dy), tmz = intbound(s2, dz);
  const double tdx = ((double)sx) / dx, tdy = ((double)sy) / dy, tdz = ((double)sz) / dz;
  const double o0 = 0.5 - m->origin[0] / res, o1 = 0.5 - m->origin[1] / res, o2 = 0.5 - m->origin[2] / res;
  /* bounded like the device's walk (raycast.cuh): a ray that misses its end voxel -- possible when it runs through
   * voxel corners -- counts as clear after 4096 steps, where the reference's nextId loop never ends */
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
    if (blocked_idx(m, id)) return 1;
  }
  return 0;
}

int orc_astar(const OrcAstarMap* m, const double start[3], const double goal[3], double resolution, double lambda,
              int32_t allocate_num, int32_t max_iter, int32_t w_max, OrcPathInfo* inf, int32_t path_max, double* path,
              double* waypts) {
  memset(inf, 0, sizeof(*inf));
  inf->status = 2;
  const int A = allocate_num;
  unsigned T = 64;
  while (T < 2u * (unsigned)A) T <<= 1;
  double* pos = malloc(sizeof(double) * 3 * (size_t)A);
  double* gs = malloc(sizeof(double) * (size_t)A);
  double* fs = malloc(sizeof(double) * (size_t)A);
  int* par = malloc(sizeof(int) * (size_t)A);
  int* slot = malloc(sizeof(int) * (size_t)A);
  int* heap = malloc(sizeof(int) * 2 * (size_t)A);
  double* ps = malloc(sizeof(double) * 3 * ((size_t)A + 1));
  Slot* tab = malloc(sizeof(Slot) * (size_t)T);
  if (!pos || !gs || !fs || !par || !slot || !heap || !ps || !tab) return -1;
  memset(tab, 0xff, sizeof(Slot) * (size_t)T);
  const unsigned mask = T - 1;
  const double inv = 1.0 / resolution;
  int end_idx[3], id[3];
  node_index(m, inv, goal, end_idx);
  /* start node (:48-60) */
  memcpy(pos, start, sizeof(double) * 3);
  par[0] = -1;
  gs[0] = 0.0;
  fs[0] = lambda * diag_heu(start, goal);
  heap[0] = 0;
  int heap_len = 1, use = 1, iter = 0, loops = 0, end_node = -1;
  node_index(m, inv, start, id);
  slot[0] = tab_insert(tab, mask, id, 0);
  inf->reason = 1;
  int nb_idx[26][3];
  for (;;) {
    if (heap_len == 0) break;
    const int cur = heap[0];
    const double* cp = pos + 3 * cur;
    int ci[3];
    node_index(m, inv, cp, ci);
    if (abs(ci[0] - end_idx[0]) <= 1 && abs(ci[1] - end_idx[1]) <= 1 && abs(ci[2] - end_idx[2]) <= 1) {
      inf->status = 1;
      inf->reason = 0;
      end_node = cur;
      break;
    }
    if (++loops > max_iter) {
      inf->reason = 3;
      inf->early_terminate_cost = gs[cur] + diag_heu(cp, goal);
      break;
    }
    heap_pop(heap, heap_len, fs);
    --heap_len;
    tab[slot[cur]].w = 2 * cur + 1;
    ++iter;
    const double cpos[3] = { cp[0], cp[1], cp[2] }, cg = gs[cur];
    int k = -1, stop = 0;
    for (double dx = -resolution; dx <= resolution + 1e-3 && !stop; dx += resolution)
      for (double dy = -resolution; dy <= resolution + 1e-3 && !stop; dy += resolution)
        for (double dz = -resolution; dz <= resolution + 1e-3 && !stop; dz += resolution) {
          const double step[3] = { dx, dy, dz };
          const double sn = norm3(dx, dy, dz);
          if (sn < 1e-3) continue;
          ++k;
          const double np[3] = { cpos[0] + step[0], cpos[1] + step[1], cpos[2] + step[2] };
          int inbox = 1;
          for (int a = 0; a < 3; ++a)
            if (np[a] <= m->box_mind[a] || np[a] >= m->box_maxd[a]) inbox = 0;
          if (!inbox || blocked(m, np)) continue;
          double dir[3] = { np[0] - cpos[0], np[1] - cpos[1], np[2] - cpos[2] };
          const double len = norm3(dir[0], dir[1], dir[2]);
          const double z = (dir[0] * dir[0] + dir[1] * dir[1]) + dir[2] * dir[2];
          if (z > 0.0) {
            const double n = sqrt(z);
            dir[0] /= n, dir[1] /= n, dir[2] /= n;
          }
          int safe = 1;
          for (double l = 0.1; l < len; l += 0.1) {
            const double ck[3] = { cpos[0] + l * dir[0], cpos[1] + l * dir[1], cpos[2] + l * dir[2] };
            if (blocked(m, ck)) {
              safe = 0;
              break;
            }
          }
          if (!safe) continue;
          node_index(m, inv, np, nb_idx[k]);
          const int s = tab_find(tab, mask, nb_idx[k]);
          if (s >= 0 && (tab[s].w & 1)) continue;
          const double tg = sn + cg;
          int nb, fresh = 0;
          if (s < 0) {
            nb = use++;
            if (use == A) {
              inf->reason = 2;
              stop = 1;
              break;
            }
            memcpy(pos + 3 * nb, np, sizeof(np));
            fresh = 1;
          } else if (tg < gs[tab[s].w >> 1]) {
            nb = tab[s].w >> 1;
          } else {
            continue;
          }
          par[nb] = cur;
          gs[nb] = tg;
          fs[nb] = tg + lambda * diag_heu(np, goal);
          if (heap_len == 2 * A) {
            inf->reason = 4;
            stop = 1;
            break;
          }
          sift_up(heap, fs, heap_len++, nb);
          if (fresh) slot[nb] = tab_insert(tab, mask, nb_idx[k], 2 * nb);
        }
    if (stop) break;
  }
  inf->iter_num = iter;
  inf->use_node_num = use;
  int nt = 0;
  if (end_node >= 0) {
    int cnt = 0;
    for (int n = end_node; n >= 0; n = par[n]) ++cnt;
    const int np_ = cnt + 1;
    memcpy(ps + 3 * cnt, goal, sizeof(double) * 3);
    int i = cnt - 1;
    for (int n = end_node; n >= 0; n = par[n], --i) memcpy(ps + 3 * i, pos + 3 * n, sizeof(double) * 3);
    inf->n_path = np_;
    if (path)
      for (int r = 0; r < path_max && r < np_; ++r) memcpy(path + 3 * r, ps + 3 * r, sizeof(double) * 3);
    /* shortenPath, in place */
    const double last[3] = { ps[3 * (np_ - 1)], ps[3 * (np_ - 1) + 1], ps[3 * (np_ - 1) + 2] };
    int mm = 1;
    for (int j = 1; j < np_ - 1; ++j) {
      const double* q = ps + 3 * j;
      const double* t = ps + 3 * (mm - 1);
      int keep = norm3(q[0] - t[0], q[1] - t[1], q[2] - t[2]) > 3.0 ? 1 : ray_blocked(m, t, ps + 3 * (j + 1));
      if (keep) {
        const double v[3] = { q[0], q[1], q[2] };
        memcpy(ps + 3 * mm, v, sizeof(v));
        ++mm;
      }
    }
    {
      const double* t = ps + 3 * (mm - 1);
      if (norm3(last[0] - t[0], last[1] - t[1], last[2] - t[2]) > 1e-3) {
        memcpy(ps + 3 * mm, last, sizeof(last));
        ++mm;
      }
    }
    if (mm == 2) {
      for (int a = 0; a < 3; ++a) {
        const double p0 = ps[a], p1 = ps[3 + a];
        ps[6 + a] = p1;
        ps[3 + a] = 0.5 * (p0 + p1);
      }
      mm = 3;
    }
    double len = 0.0;
    for (int j = 0; j + 1 < mm; ++j)
      len += norm3(ps[3 * j + 3] - ps[3 * j], ps[3 * j + 4] - ps[3 * j + 1], ps[3 * j + 5] - ps[3 * j + 2]);
    inf->length = len;
    nt = mm;
    if (len < 1.5) {
      inf->branch = 1;
    } else if (len > 5.0) {
      inf->branch = 3;
      double len2 = 0.0;
      int t = 1;
      for (int j = 1; j < mm && len2 < 5.0; ++j) {
        len2 += norm3(ps[3 * j] - ps[3 * t - 3], ps[3 * j + 1] - ps[3 * t - 2], ps[3 * j + 2] - ps[3 * t - 1]);
        ++t;
      }
      nt = t;
    } else {
      inf->branch = 2;
    }
    if (inf->branch == 3)
      memcpy(inf->next_goal, ps + 3 * (nt - 1), sizeof(double) * 3);
    else
      memcpy(inf->next_goal, goal, sizeof(double) * 3);
    inf->n_wp = nt;
    inf->tour_status = nt < 3 ? 2 : ((nt > 32 || nt > w_max) ? 1 : 0);
    for (int r = 0; r < nt && r < w_max; ++r) memcpy(waypts + 3 * r, ps + 3 * r, sizeof(double) * 3);
  }
  free(pos), free(gs), free(fs), free(par), free(slot), free(heap), free(ps), free(tab);
  return (end_node >= 0 && inf->tour_status == 0) ? nt : 0;
}
