/* CPU restatement of FastExplorationManager::refineLocalTour (exploration_manager/src/fast_exploration_manager.cpp:
 * 429-503): the layered GraphSearch<ViewNode> as :441-469 builds it, DijkstraSearch (active_perception/include/
 * active_perception/graph_search.h:76-118) with its std::priority_queue restated as libstdc++ implements push and pop,
 * ViewNode::costTo (graph_node.cpp:25-30) through orc_view_cost, lazily, in the order the search asks for it, and the
 * refined tour (:487-498).  TEST INFRASTRUCTURE ONLY (the GPU tests compare the device with it). */
#include "fuel_oracle_tour.h"

#include <math.h>
#include <stdlib.h>
#include <string.h>

/* std::priority_queue<shared_ptr<ViewNode>, vector, NodeCompare>: push_heap / pop_heap -> __adjust_heap ->
 * __push_heap, comparing node1->g_value_ > node2->g_value_ through each node's current g */
static void sift_up(int* heap, const double* g, int hole, int v) {
  const double gv = g[v];
  int parent = (hole - 1) / 2;
  while (hole > 0 && g[heap[parent]] > gv) {
    heap[hole] = heap[parent];
    hole = parent;
    parent = (hole - 1) / 2;
  }
  heap[hole] = v;
}
static void pop_top(int* heap, int len, const double* g) {
  if (len <= 1) return;
  const int n = len - 1, v = heap[n];
  heap[n] = heap[0];
  int hole = 0, child = 0;
  while (child < (n - 1) / 2) {
    child = 2 * (child + 1);
    if (g[heap[child]] > g[heap[child - 1]]) child--;
    heap[hole] = heap[child];
    hole = child;
  }
  if ((n & 1) == 0 && child == (n - 2) / 2) {
    child = 2 * (child + 1);
    heap[hole] = heap[child - 1];
    hole = child - 1;
  }
  sift_up(heap, g, hole, v);
}

typedef struct {
  const double* pos;
  double yaw, vel[3];
  int vp; /* index into vp_*, -1 for the current state */
} Node;

int orc_local_tour(const OrcAstarMap* m, int32_t ng, const int32_t* gsize, const double* vp_pos, const double* vp_yaw,
                   const double cur_pos[3], const double cur_vel[3], double cur_yaw, double vm, double yd, double w_dir,
                   double resolution, double lambda, int32_t allocate_num, int32_t max_iter, double tour_lambda,
                   const double* table, OrcLocalTourInfo* info, int32_t kmax, int32_t* refined, int32_t tour_max,
                   double* tour, double* edge_cost) {
  if (ng < 1 || ng > kmax || gsize[ng - 1] < 1 || tour_max < 1 || (!table && !m)) return -2;
  memset(info, 0, sizeof(*info));
  for (int i = 0; i < kmax; ++i) refined[i] = -1;
  memset(tour, 0, sizeof(double) * 3 * (size_t)tour_max);
  int32_t N = 0, maxdeg = 1;
  for (int i = 0; i < ng; ++i) {
    N += gsize[i];
    if (gsize[i] > maxdeg) maxdeg = gsize[i];
  }
  /* the graph (:436-469): node 0 the current state, then each group's nodes; the last group keeps its first */
  Node* nodes = malloc(sizeof(Node) * ((size_t)N + 2));
  int* nbr = malloc(sizeof(int) * ((size_t)N + 2) * (size_t)maxdeg); /* neighbors_ of each node */
  int* eid = malloc(sizeof(int) * ((size_t)N + 2) * (size_t)maxdeg); /* the addEdge index of each */
  int* deg = calloc((size_t)N + 2, sizeof(int));
  int* last = malloc(sizeof(int) * ((size_t)N + 2));
  int* cur = malloc(sizeof(int) * ((size_t)N + 2));
  if (!nodes || !nbr || !eid || !deg || !last || !cur) goto oom;
  int n_nodes = 1, n_edges = 0, n_last = 1, n_cur = 0, final_node = -1;
  nodes[0].pos = cur_pos;
  nodes[0].yaw = cur_yaw;
  memcpy(nodes[0].vel, cur_vel, sizeof(double) * 3); /* first->vel_ = cur_vel */
  nodes[0].vp = -1;
  last[0] = 0;
  int vp0 = 0;
  for (int i = 0; i < ng; ++i) {
    for (int j = 0; j < gsize[i]; ++j) {
      const int id = n_nodes++;
      nodes[id].pos = vp_pos + 3 * (size_t)(vp0 + j);
      nodes[id].yaw = vp_yaw[vp0 + j];
      nodes[id].vel[0] = nodes[id].vel[1] = nodes[id].vel[2] = 0.0; /* vel_.setZero() */
      nodes[id].vp = vp0 + j;
      for (int k = 0; k < n_last; ++k) { /* g_search.addEdge(nd->id_, node->id_) */
        const int nd = last[k];
        nbr[(size_t)nd * maxdeg + deg[nd]] = id;
        eid[(size_t)nd * maxdeg + deg[nd]] = n_edges++;
        deg[nd]++;
      }
      cur[n_cur++] = id;
      if (i == ng - 1) {
        final_node = id;
        break;
      }
    }
    memcpy(last, cur, sizeof(int) * (size_t)n_cur);
    n_last = n_cur;
    n_cur = 0;
    vp0 += gsize[i];
  }
  info->n_nodes = n_nodes;
  info->n_edges = n_edges;
  if (edge_cost)
    for (int e = 0; e < n_edges; ++e) edge_cost[e] = NAN;

  int bad = 0;
  for (int k = 0; k < 3; ++k) bad = bad || !isfinite(cur_pos[k]) || !isfinite(cur_vel[k]);
  bad = bad || !isfinite(cur_yaw);
  for (int n = 1; n < n_nodes; ++n)
    bad = bad || !isfinite(nodes[n].pos[0]) || !isfinite(nodes[n].pos[1]) || !isfinite(nodes[n].pos[2]) ||
          !isfinite(nodes[n].yaw);
  if (bad) {
    info->status = 2;
    goto done;
  }

  /* DijkstraSearch (graph_search.h:76-118) */
  {
    double* g = malloc(sizeof(double) * (size_t)n_nodes);
    int* parent = malloc(sizeof(int) * (size_t)n_nodes);
    char* closed = calloc((size_t)n_nodes, 1);
    int* heap = malloc(sizeof(int) * ((size_t)n_edges + 1));
    if (!g || !parent || !closed || !heap) {
      free(g), free(parent), free(closed), free(heap);
      goto oom;
    }
    for (int n = 0; n < n_nodes; ++n) g[n] = 1000000, parent[n] = -1; /* BaseNode() */
    g[0] = 0.0;
    heap[0] = 0;
    int len = 1, reached = 0;
    info->pushes = 1;
    while (len > 0) {
      const int vc = heap[0];
      pop_top(heap, len, g);
      --len;
      info->pops++;
      closed[vc] = 1;
      if (vc == final_node) {
        reached = 1;
        break;
      }
      for (int t = 0; t < deg[vc]; ++t) {
        const int vb = nbr[(size_t)vc * maxdeg + t], e = eid[(size_t)vc * maxdeg + t];
        if (closed[vb]) continue;
        double c;
        if (table) {
          c = table[e];
        } else { /* vc->costTo(vb): computeCost(pos_, node->pos_, yaw_, node->yaw_, vel_, yaw_dot_, path) */
          OrcViewCostInfo vi;
          if (orc_view_cost(m, nodes[vc].pos, nodes[vb].pos, nodes[vc].yaw, nodes[vb].yaw, nodes[vc].vel, vm, yd,
                            w_dir, resolution, lambda, allocate_num, max_iter, &vi, 0, NULL) < 0) {
            free(g), free(parent), free(closed), free(heap);
            goto oom;
          }
          c = vi.cost;
        }
        info->n_evals++;
        if (edge_cost) edge_cost[e] = c;
        const double g_tmp = g[vc] + c;
        if (g_tmp < g[vb]) {
          g[vb] = g_tmp;
          parent[vb] = vc;
          sift_up(heap, g, len++, vb);
          info->pushes++;
        }
      }
    }
    info->g = g[final_node];
    if (reached) { /* path: final_node back through parent_, reversed; refined = path[1..] */
      int depth = 0;
      for (int v = final_node; v > 0; v = parent[v]) ++depth;
      info->n_refined = depth;
      int i = depth - 1;
      for (int v = final_node; v > 0; v = parent[v]) refined[i--] = nodes[v].vp;
    } else {
      info->status = 1;
    }
    free(g), free(parent), free(closed), free(heap);
  }

  /* the refined tour (:487-498): searchPath from refined_tour_.back() to each refined point at tour_lambda */
  if (m) {
    double back[3];
    memcpy(back, cur_pos, sizeof(back));
    memcpy(tour, cur_pos, sizeof(double) * 3);
    int n = 1;
    double* seg = malloc(sizeof(double) * 3 * (size_t)tour_max);
    if (!seg) goto oom;
    for (int i = 0; i < info->n_refined; ++i) {
      const double* pt = vp_pos + 3 * (size_t)refined[i];
      OrcViewCostInfo vi;
      const double zero[3] = { 0, 0, 0 };
      if (orc_view_cost(m, back, pt, 0.0, 0.0, zero, vm, yd, w_dir, resolution, tour_lambda, allocate_num, max_iter,
                        &vi, tour_max, seg) < 0) {
        free(seg);
        goto oom;
      }
      if (vi.length != 0.0) { /* if (ViewNode::searchPath(...)): insert the path */
        for (int r = 0; r < vi.n_path && n + r < tour_max; ++r) memcpy(tour + 3 * (size_t)(n + r), seg + 3 * r, 24);
        /* the path's last row: the goal for {p1, p2}, the goal again for getPath() */
        if (vi.n_path <= tour_max) memcpy(back, seg + 3 * (size_t)(vi.n_path - 1), sizeof(back));
        else memcpy(back, pt, sizeof(back));
        n += vi.n_path;
      } else { /* refined_tour_.push_back(pt) */
        if (n < tour_max) memcpy(tour + 3 * (size_t)n, pt, 24);
        memcpy(back, pt, sizeof(back));
        n += 1;
      }
    }
    free(seg);
    info->n_tour = n;
    if (info->status == 0 && n > tour_max) info->status = 3;
  }
done:
  free(nodes), free(nbr), free(eid), free(deg), free(last), free(cur);
  return 0;
oom:
  free(nodes), free(nbr), free(eid), free(deg), free(last), free(cur);
  return -1;
}
