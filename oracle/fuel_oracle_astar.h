/* CPU restatement of Astar::search + shortenPath + planExploreMotion's goal branch (fuel_oracle_astar.c).
 * TEST INFRASTRUCTURE ONLY. */
#pragma once
#include <stdint.h>

typedef struct {
  int32_t n[3];
  double res, res_inv; /* the map's resolution_ and resolution_inv_ = 1 / resolution_ */
  double origin[3];
  double box_mind[3], box_maxd[3];
  const uint8_t* occ; /* [nx][ny][nz]: bits 0-1 tri-state (0 = UNKNOWN), bit 2 inflate */
} OrcAstarMap;

/* the layout of FuelPathInfo (include/fuelgpu.h) */
typedef struct {
  int32_t status, reason, iter_num, use_node_num, n_path, n_wp, branch, tour_status;
  double early_terminate_cost, length, next_goal[3];
} OrcPathInfo;

/* One search; path [path_max][3] or NULL gets the first rows of getPath(), waypts [w_max][3] the tour's first rows.
 * Returns the n_wp the device writes (the tour's count when it is usable, else 0), -1 when out of memory. */
int orc_astar(const OrcAstarMap* m, const double start[3], const double goal[3], double resolution, double lambda,
              int32_t allocate_num, int32_t max_iter, int32_t w_max, OrcPathInfo* info, int32_t path_max, double* path,
              double* waypts);
