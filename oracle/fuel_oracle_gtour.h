/* CPU restatement of the tour FastExplorationManager::findGlobalTour (exploration_manager/src/
 * fast_exploration_manager.cpp:327-427) asks LKH for: the ATSP over the int(cost * 100) matrix, solved exactly by
 * Held-Karp dynamic programming over subsets (fuel_oracle_gtour.c).  TEST INFRASTRUCTURE ONLY. */
#pragma once
#include <stdint.h>

#define ORC_GTOUR_MAX_CLUSTERS 20
#define ORC_GTOUR_OK 0
#define ORC_GTOUR_BAD_INPUT 1
#define ORC_GTOUR_TOO_LARGE 2

/* One d x d row-major matrix (node 0 the current state, nodes 1 .. d-1 the clusters), as fuelgpu_global_tour_batch
 * solves one instance: returns the status (or -1 when out of memory); on ORC_GTOUR_OK *cost is the optimal cycle cost,
 * *n_optimal the number of optimal tours (saturating at INT32_MAX) and indices [d - 1] the lexicographically smallest
 * optimal sequence of 0-based cluster ids.  Otherwise nothing is written. */
int orc_global_tour(int32_t d, const double* mat, int64_t* cost, int32_t* n_optimal, int32_t* indices);
