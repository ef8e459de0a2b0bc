// local_tour.cu -- FastExplorationManager::refineLocalTour (exploration_manager/src/fast_exploration_manager.cpp:429-503)
// on sm_90a for a batch of problems: the layered GraphSearch<ViewNode>, its DijkstraSearch (active_perception/include/
// active_perception/graph_search.h:76-118) over ViewNode::costTo edges, and the refined tour.
//
// Five stages on the map's main stream, with no host synchronisation between them:
//   1. lt_edges_kernel: every edge of every problem's graph, one per thread, in addEdge order (:441-469);
//   2. view_cost_impl (view_cost.cu) over those pairs: the edge cost table;
//   3. lt_dijkstra_kernel: one warp per problem runs DijkstraSearch over the table, writes the refined viewpoints and
//      the tour's segment pairs (the previous refined point, or cur_pos, to the refined point);
//   4. view_cost_impl over the segments with astar.lambda_heu = tour_lambda_heu: searchPath's length and path;
//   5. lt_tour_kernel: one warp per problem assembles ed_->refined_tour_ (:487-498).
// The reference's searchPath returns a path that ends exactly at its goal ({p1, p2}, or getPath()), and pushes the
// goal itself otherwise, so the tour's end is always the last refined point and the segments are independent.
// Built with -fmad=false: the only arithmetic here is the search's g_tmp = g + cost, which rounds as the reference's.
#include "common.cuh"
#include "heap.cuh"

#include <math.h>

#include <algorithm>
#include <vector>

namespace {

constexpr int LT_THREADS = 128;
constexpr int LT_WARPS = LT_THREADS / 32;
constexpr double LT_G0 = 1000000;  // BaseNode(): g_value_ = 1000000 (graph_node.h)

// One group of one problem's graph (a layer of nodes).
struct LtGroup {
  int prob;
  int first_vp;  // its first viewpoint in vp_*
  int n_eff;     // its nodes: every viewpoint, only the first in the problem's last group
  int in_vp;     // the first viewpoint of the group before, -1 when that is node 0 (the current state)
  int n_in;      // nodes of the group before (1 for node 0)
  int edge_off;  // its first incoming edge, global
  int node_off;  // its first node, numbered inside the problem (node 0 is the current state)
};
// One problem.
struct LtProb {
  int g0, ng;              // its groups
  int node_base, n_nodes;  // its search state in the per-node arrays
  int edge_off, n_edges;   // its edges; its heap starts at edge_off + problem index
};

struct LtEdges {
  double *p1, *p2, *y1, *y2, *v1;
};

__device__ __forceinline__ bool lt_finite3(const double* p) {
  return isfinite(p[0]) && isfinite(p[1]) && isfinite(p[2]);
}

// stage 1: edge e of the G groups (edge_off ascending) -> its (p1, p2, y1, y2, v1) as costTo passes them
__global__ void __launch_bounds__(LT_THREADS)
lt_edges_kernel(int E, int G, const LtGroup* __restrict__ grp, const double* __restrict__ cur_pos,
                const double* __restrict__ cur_vel, const double* __restrict__ cur_yaw,
                const double* __restrict__ vp_pos, const double* __restrict__ vp_yaw, LtEdges out) {
  const int e = blockIdx.x * LT_THREADS + threadIdx.x;
  if (e >= E) return;
  int lo = 0, hi = G;  // the last group whose edge_off <= e: the one with edges when several share the offset
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (grp[mid].edge_off <= e) lo = mid;
    else hi = mid;
  }
  const LtGroup gr = grp[lo];
  const int local = e - gr.edge_off, j = local / gr.n_in, k = local % gr.n_in;
  const double* a = gr.in_vp < 0 ? cur_pos + 3 * gr.prob : vp_pos + 3 * (size_t)(gr.in_vp + k);
  const double* b = vp_pos + 3 * (size_t)(gr.first_vp + j);
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    out.p1[3 * (size_t)e + c] = a[c];
    out.p2[3 * (size_t)e + c] = b[c];
    out.v1[3 * (size_t)e + c] = gr.in_vp < 0 ? cur_vel[3 * gr.prob + c] : 0.0;  // ViewNode(): vel_.setZero()
  }
  out.y1[e] = gr.in_vp < 0 ? cur_yaw[gr.prob] : vp_yaw[gr.in_vp + k];
  out.y2[e] = vp_yaw[gr.first_vp + j];
}

// the group (index into grp, from pr.g0) holding node n >= 1 of problem pr
__device__ __forceinline__ int lt_group_of(const LtGroup* grp, const LtProb& pr, int n) {
  int lo = pr.g0, hi = pr.g0 + pr.ng;
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (grp[mid].node_off <= n) lo = mid;
    else hi = mid;
  }
  return lo;
}

// stage 3: DijkstraSearch of one problem per warp.  Lane 0 pops the open set; the lanes read the neighbours' closed
// flags and compute g_tmp = g + cost in parallel; lane 0 then applies the relaxations and pushes in neighbours_ order.
__global__ void __launch_bounds__(LT_THREADS)
lt_dijkstra_kernel(int B, const LtProb* __restrict__ probs, const LtGroup* __restrict__ grp,
                   const double* __restrict__ cur_pos, const double* __restrict__ cur_vel,
                   const double* __restrict__ cur_yaw, const double* __restrict__ vp_pos,
                   const double* __restrict__ vp_yaw, const FuelViewCostInfo* __restrict__ einfo, double* g_all,
                   int* par_all, int* closed_all, int* heap_all, FuelLocalTourInfo* __restrict__ info, int kmax,
                   int32_t* __restrict__ refined, double* __restrict__ edge_cost, LtEdges seg) {
  const int b = blockIdx.x * LT_WARPS + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (b >= B) return;
  const LtProb pr = probs[b];
  double* g = g_all + pr.node_base;
  int* par = par_all + pr.node_base;
  int* closed = closed_all + pr.node_base;
  int* heap = heap_all + pr.edge_off + b;
  for (int i = lane; i < pr.n_nodes; i += 32) {
    g[i] = LT_G0;
    par[i] = -1;
    closed[i] = 0;
  }
  if (edge_cost)
    for (int i = lane; i < pr.n_edges; i += 32) edge_cost[pr.edge_off + i] = einfo[pr.edge_off + i].cost;
  for (int i = lane; i < kmax; i += 32) refined[(size_t)b * kmax + i] = -1;
  // a non-finite coordinate of the current state or of a graph node
  bool bad = false;
  if (lane == 0) bad = !lt_finite3(cur_pos + 3 * b) || !lt_finite3(cur_vel + 3 * b) || !isfinite(cur_yaw[b]);
  for (int gi = pr.g0; gi < pr.g0 + pr.ng; ++gi) {
    const LtGroup gr = grp[gi];
    for (int j = lane; j < gr.n_eff; j += 32)
      bad = bad || !lt_finite3(vp_pos + 3 * (size_t)(gr.first_vp + j)) || !isfinite(vp_yaw[gr.first_vp + j]);
  }
  bad = __any_sync(0xffffffffu, bad);
  __syncwarp();

  const int final_node = pr.n_nodes - 1;  // the first viewpoint of the last group, added last
  int len = 0, pops = 0, pushes = 0, evals = 0;
  bool reached = false;
  if (!bad) {
    if (lane == 0) {
      g[0] = 0.0;
      heap[0] = 0;
      len = 1;
      pushes = 1;
    }
    for (;;) {
      int vc = -1;
      if (lane == 0 && len > 0) {
        vc = heap[0];
        heap_pop(heap, len, g);
        --len;
        ++pops;
        closed[vc] = 1;
      }
      vc = __shfl_sync(0xffffffffu, vc, 0);
      __syncwarp();
      if (vc < 0) break;
      if (vc == final_node) {
        reached = true;
        break;
      }
      // neighbours_: every node of the next group, in order; the edge from the k-th node of this group to the j-th
      // of the next is edge_off + j * n_in + k
      int nxt, k;
      if (vc == 0) {
        nxt = pr.g0, k = 0;
      } else {
        const int gi = lt_group_of(grp, pr, vc);
        nxt = gi + 1, k = vc - grp[gi].node_off;
      }
      if (nxt >= pr.g0 + pr.ng) continue;
      const LtGroup gn = grp[nxt];
      const double gv = g[vc];
      for (int base = 0; base < gn.n_eff; base += 32) {
        const int j = base + lane;
        int vb = -1, cl = 1;
        double gt = 0.0;
        if (j < gn.n_eff) {
          vb = gn.node_off + j;
          cl = closed[vb];
          gt = gv + einfo[gn.edge_off + j * gn.n_in + k].cost;  // vc->g_value_ + vc->costTo(vb)
        }
        const int cnt = min(32, gn.n_eff - base);
        for (int t = 0; t < cnt; ++t) {
          const int tb = __shfl_sync(0xffffffffu, vb, t), tc = __shfl_sync(0xffffffffu, cl, t);
          const double tg = __shfl_sync(0xffffffffu, gt, t);
          if (lane == 0 && !tc) {
            ++evals;
            if (tg < g[tb]) {
              g[tb] = tg;
              par[tb] = vc;
              heap_sift_up(heap, g, len++, tb);
              ++pushes;
            }
          }
        }
      }
      __syncwarp();
    }
  }
  if (lane != 0) return;
  FuelLocalTourInfo r;
  memset(&r, 0, sizeof(r));
  r.n_nodes = pr.n_nodes;
  r.n_edges = pr.n_edges;
  r.n_tour = 1;
  double nan = __longlong_as_double(0x7ff8000000000000ll);
  if (bad) {
    r.status = FUELGPU_TOUR_BAD_INPUT;
    r.n_tour = 0;
  } else {
    r.pops = pops, r.pushes = pushes, r.n_evals = evals;
    r.g = g[final_node];
    if (reached) {
      r.n_refined = pr.ng;
      int v = final_node;  // path[ng] back to path[1] through parent_
      for (int i = pr.ng - 1; i >= 0; --i) {
        const LtGroup gr = grp[pr.g0 + i];
        refined[(size_t)b * kmax + i] = gr.first_vp + (v - gr.node_off);
        v = par[v];
      }
    } else {
      r.status = FUELGPU_TOUR_UNREACHABLE;
    }
  }
  info[b] = r;
  // the tour's segments: refined_tour_.back() (cur_pos, then the previous refined point) -> the refined point; unused
  // slots are NaN rows, which the view-cost pipeline marks bad without a search
  for (int i = 0; i < pr.ng; ++i) {
    const size_t s = (size_t)pr.g0 + i;
    const bool on = i < r.n_refined;
    const double* a = i == 0 ? cur_pos + 3 * b : vp_pos + 3 * (size_t)(on ? refined[(size_t)b * kmax + i - 1] : 0);
    const double* c = vp_pos + 3 * (size_t)(on ? refined[(size_t)b * kmax + i] : 0);
    for (int q = 0; q < 3; ++q) {
      seg.p1[3 * s + q] = on ? a[q] : nan;
      seg.p2[3 * s + q] = on ? c[q] : nan;
      seg.v1[3 * s + q] = 0.0;
    }
    seg.y1[s] = 0.0;
    seg.y2[s] = 0.0;
  }
}

// stage 5: refined_tour_ of one problem per warp
__global__ void __launch_bounds__(LT_THREADS)
lt_tour_kernel(int B, const LtProb* __restrict__ probs, const double* __restrict__ cur_pos,
               const FuelViewCostInfo* __restrict__ sinfo, const double* __restrict__ seg_p2,
               const double* __restrict__ seg_path, int tour_max, FuelLocalTourInfo* __restrict__ info,
               double* __restrict__ tour) {
  const int b = blockIdx.x * LT_WARPS + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (b >= B) return;
  const int g0 = probs[b].g0, status = info[b].status, n_refined = info[b].n_refined;
  double* dst = tour + (size_t)b * tour_max * 3;
  int n = 0;
  if (status != FUELGPU_TOUR_BAD_INPUT) {
    if (lane == 0)
      for (int q = 0; q < 3; ++q) dst[q] = cur_pos[3 * b + q];
    n = 1;
    for (int i = 0; i < n_refined; ++i) {
      const size_t s = (size_t)g0 + i;
      const int n_path = sinfo[s].n_path;
      if (sinfo[s].length != 0.0) {  // if (ViewNode::searchPath(...)): insert the path
        const double* src = seg_path + s * tour_max * 3;
        for (int r = lane; r < n_path && n + r < tour_max; r += 32) {
          dst[3 * (n + r)] = src[3 * r];
          dst[3 * (n + r) + 1] = src[3 * r + 1];
          dst[3 * (n + r) + 2] = src[3 * r + 2];
        }
        n += n_path;
      } else {  // else refined_tour_.push_back(pt)
        if (lane == 0 && n < tour_max)
          for (int q = 0; q < 3; ++q) dst[3 * n + q] = seg_p2[3 * s + q];
        n += 1;
      }
    }
  }
  for (int q = 3 * n + lane; q < 3 * tour_max; q += 32) dst[q] = 0.0;
  if (lane == 0) {
    info[b].n_tour = n;
    if (status == FUELGPU_TOUR_OK && n > tour_max) info[b].status = FUELGPU_TOUR_TRUNCATED;
  }
}

}  // namespace

int local_tour_impl(FuelMap* m, int B, const int32_t* prob_off, const int32_t* group_off, const FuelLocalTourParams* p,
                    const LocalTourIO& io) {
  if (B == 0) return 0;
  // the graph's layout from the host-side structure alone
  const int G = prob_off[B];
  std::vector<LtGroup> grp((size_t)std::max(G, 1));
  std::vector<LtProb> probs((size_t)B);
  long long E = 0, N = 0;
  for (int b = 0; b < B; ++b) {
    LtProb& pr = probs[b];
    pr.g0 = prob_off[b];
    pr.ng = prob_off[b + 1] - prob_off[b];
    pr.node_base = (int)N;
    pr.edge_off = (int)E;
    int node = 1, in_vp = -1, n_in = 1;
    for (int i = 0; i < pr.ng; ++i) {
      const int gi = pr.g0 + i, sz = group_off[gi + 1] - group_off[gi];
      LtGroup& gr = grp[gi];
      gr.prob = b;
      gr.first_vp = group_off[gi];
      gr.n_eff = i == pr.ng - 1 ? std::min(sz, 1) : sz;
      gr.in_vp = in_vp;
      gr.n_in = n_in;
      gr.edge_off = (int)E;
      gr.node_off = node;
      E += (long long)gr.n_eff * n_in;
      node += gr.n_eff;
      in_vp = gr.first_vp;
      n_in = gr.n_eff;
    }
    pr.n_nodes = node;
    pr.n_edges = (int)(E - pr.edge_off);
    N += node;
  }
  auto al = [](size_t x) { return (x + 255) & ~(size_t)255; };
  const size_t nE = (size_t)E, nG = (size_t)G, tm = (size_t)io.tour_max;
  size_t o = 0;
  const size_t o_grp = o;
  o += al(sizeof(LtGroup) * grp.size());
  const size_t o_prob = o;
  o += al(sizeof(LtProb) * (size_t)B);
  const size_t o_ep = o;  // edge pairs: p1, p2, v1 [E][3], y1, y2 [E]
  o += 5 * al(24 * nE);
  const size_t o_ei = o;
  o += al(sizeof(FuelViewCostInfo) * nE);
  const size_t o_g = o;
  o += al(8 * (size_t)N);
  const size_t o_par = o;
  o += al(4 * (size_t)N);
  const size_t o_cl = o;
  o += al(4 * (size_t)N);
  const size_t o_heap = o;
  o += al(4 * (nE + (size_t)B));
  const size_t o_sp = o;  // segment pairs
  o += 5 * al(24 * nG);
  const size_t o_si = o;
  o += al(sizeof(FuelViewCostInfo) * nG);
  const size_t o_path = o;
  o += al(24 * nG * tm);
  int rc = m->lt_buf.ensure(m, o);
  if (rc) return rc;
  uint8_t* base = m->lt_buf.p;
  LtGroup* d_grp = (LtGroup*)(base + o_grp);
  LtProb* d_prob = (LtProb*)(base + o_prob);
  auto pairs = [&](size_t off, size_t n) {
    const size_t s = al(24 * n);
    return LtEdges{ (double*)(base + off), (double*)(base + off + s), (double*)(base + off + 2 * s),
                    (double*)(base + off + 3 * s), (double*)(base + off + 4 * s) };
  };
  const LtEdges ep = pairs(o_ep, nE), sp = pairs(o_sp, nG);
  FuelViewCostInfo* einfo = (FuelViewCostInfo*)(base + o_ei);
  FuelViewCostInfo* sinfo = (FuelViewCostInfo*)(base + o_si);
  FUEL_CUDA(m, cudaMemcpyAsync(d_grp, grp.data(), sizeof(LtGroup) * grp.size(), cudaMemcpyHostToDevice, m->stream));
  FUEL_CUDA(m, cudaMemcpyAsync(d_prob, probs.data(), sizeof(LtProb) * (size_t)B, cudaMemcpyHostToDevice, m->stream));
  // 1-2: the edges and their costs
  if (E > 0) {
    lt_edges_kernel<<<(unsigned)((E + LT_THREADS - 1) / LT_THREADS), LT_THREADS, 0, m->stream>>>(
        (int)E, G, d_grp, io.cur_pos, io.cur_vel, io.cur_yaw, io.vp_pos, io.vp_yaw, ep);
    FUEL_LAUNCHES(m, 1);
    FUEL_CUDA(m, cudaGetLastError());
    rc = view_cost_impl(m, (int)E, ep.p1, ep.p2, ep.y1, ep.y2, ep.v1, &p->view, einfo, 0, nullptr);
    if (rc) return rc;
  }
  // 3: the search
  const unsigned wblocks = (unsigned)((B + LT_WARPS - 1) / LT_WARPS);
  lt_dijkstra_kernel<<<wblocks, LT_THREADS, 0, m->stream>>>(
      B, d_prob, d_grp, io.cur_pos, io.cur_vel, io.cur_yaw, io.vp_pos, io.vp_yaw, einfo, (double*)(base + o_g),
      (int*)(base + o_par), (int*)(base + o_cl), (int*)(base + o_heap), io.info, io.kmax, io.refined, io.edge_cost,
      sp);
  FUEL_LAUNCHES(m, 1);
  FUEL_CUDA(m, cudaGetLastError());
  // 4-5: the tour's segments (ViewNode::astar_->lambda_heu_ = tour_lambda_heu), then the tour
  FuelViewCostParams tp = p->view;
  tp.astar.lambda_heu = p->tour_lambda_heu;
  double* seg_path = (double*)(base + o_path);
  rc = view_cost_impl(m, G, sp.p1, sp.p2, sp.y1, sp.y2, sp.v1, &tp, sinfo, io.tour_max, seg_path);
  if (rc) return rc;
  lt_tour_kernel<<<wblocks, LT_THREADS, 0, m->stream>>>(B, d_prob, io.cur_pos, sinfo, sp.p2, seg_path, io.tour_max,
                                                        io.info, io.tour);
  FUEL_LAUNCHES(m, 1);
  FUEL_CUDA(m, cudaGetLastError());
  return 0;
}
