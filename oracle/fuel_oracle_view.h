/* CPU restatement of ViewNode::searchPath + computeCost (active_perception/src/graph_node.cpp:32-85) over the A* oracle
 * (fuel_oracle_view.c).  TEST INFRASTRUCTURE ONLY. */
#pragma once
#include <stdint.h>

#include "fuel_oracle_astar.h"

/* the layout of FuelViewCostInfo (include/fuelgpu.h) */
typedef struct {
  int32_t kind, reason, iter_num, use_node_num, n_path, reserved;
  double length, cost;
} OrcViewCostInfo;

/* ViewNode::computeCost(p1, p2, y1, y2, v1, 0, path) with searchPath's A* at (resolution, lambda, allocate_num,
 * max_iter); path [path_max][3] or NULL gets the first rows of searchPath's path.  Returns 0, -1 when out of memory. */
int orc_view_cost(const OrcAstarMap* m, const double p1[3], const double p2[3], double y1, double y2, const double v1[3],
                  double vm, double yd, double w_dir, double resolution, double lambda, int32_t allocate_num,
                  int32_t max_iter, OrcViewCostInfo* info, int32_t path_max, double* path);
