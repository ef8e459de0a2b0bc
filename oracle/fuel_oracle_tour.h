/* CPU restatement of FastExplorationManager::refineLocalTour (exploration_manager/src/fast_exploration_manager.cpp:
 * 429-503) over the view-cost oracle (fuel_oracle_tour.c).  TEST INFRASTRUCTURE ONLY. */
#pragma once
#include <stdint.h>

#include "fuel_oracle_view.h"

/* the layout of FuelLocalTourInfo (include/fuelgpu.h) */
typedef struct {
  int32_t status, n_nodes, n_edges, n_evals, n_refined, n_tour, pops, pushes;
  double g;
} OrcLocalTourInfo;

/* One refineLocalTour problem: ng groups of gsize[i] viewpoints (vp_pos [N][3], vp_yaw [N], group by group), the
 * current state.  table NULL: every costTo is orc_view_cost at (vm, yd, w_dir, resolution, lambda, allocate_num,
 * max_iter), evaluated lazily as DijkstraSearch asks for it and counted in n_evals; else table [n_edges] holds the edge
 * costs in addEdge order.  m NULL (table mode only): no tour.  The tour's searches run at tour_lambda.  Outputs as
 * fuelgpu_local_tour_batch writes one problem: refined [kmax] (indices into this problem's vp_*), tour [tour_max][3];
 * edge_cost [n_edges] or NULL gets each edge's cost where it was evaluated, NaN elsewhere.  Returns 0, -1 when out of
 * memory, -2 on a structure fuelgpu_local_tour_batch refuses. */
int orc_local_tour(const OrcAstarMap* m, int32_t ng, const int32_t* gsize, const double* vp_pos, const double* vp_yaw,
                   const double cur_pos[3], const double cur_vel[3], double cur_yaw, double vm, double yd, double w_dir,
                   double resolution, double lambda, int32_t allocate_num, int32_t max_iter, double tour_lambda,
                   const double* table, OrcLocalTourInfo* info, int32_t kmax, int32_t* refined, int32_t tour_max,
                   double* tour, double* edge_cost);
