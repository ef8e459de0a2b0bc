/* CPU restatement of kinodynamicReplan's search: KinodynamicAstar::search, its retry and getSamples
 * (fuel_oracle_kino.c).  TEST INFRASTRUCTURE ONLY. */
#pragma once
#include <stdint.h>

#include "fuel_oracle_astar.h"

/* the layout of FuelKinoParams (include/fuelgpu.h) */
typedef struct {
  double max_tau, init_max_tau, max_vel, vel_margin, max_acc, w_time, horizon, lambda_heu, resolution;
  double ctrl_pt_dist, manager_max_vel;
  int32_t allocate_num, check_num, optimistic, reserved;
} OrcKinoParams;

/* the layout of FuelKinoInfo (include/fuelgpu.h) */
typedef struct {
  int32_t status, reason, retried, traj_status;
  int32_t iter_num, use_node_num, n_nodes, shot;
  int32_t seg_num, n_pts;
  double t_shot, T_sum;
} OrcKinoInfo;

#define ORC_KINO_GLIBC 0  /* libm exactly as the reference calls it */
#define ORC_KINO_DEVICE 1 /* the device's arithmetic: correctly rounded powers outside the search, acos / cos of the
                             three-root branch correctly rounded (libquadmath rounded to double) */

/* One kinodynamicReplan(start, vel, acc, goal, 0) up to getSamples.  points [FUELGPU_MAX_PTS-2][3], derivs [4][3], dt [1]
 * as the device writes them; nodes [node_max][12] (state, input, duration, g, f of the path root .. end) and shot [3][4]
 * (coef_shot_, row = axis) or NULL.  map_size is the map's size (getRegion).  Returns 0, -1 when out of memory. */
int orc_kino_replan(const OrcAstarMap* m, const double map_size[3], const OrcKinoParams* p, int32_t math,
                    const double start[3], const double vel[3], const double acc[3], const double goal[3],
                    OrcKinoInfo* info, double* points, double* derivs, double* dt, int32_t node_max, double* nodes,
                    double* shot);

/* how many heuristic evaluations took cubic()'s D < 0 branch since the last reset (reset != 0 zeroes the count) */
long long orc_kino_three_root_count(int32_t reset);

/* the host build of fuel_b200/csrc/kino_math.cuh, for its tests: out[i] = f(in[i]), f = 0 cbrt, 1 cube, 2 acos_cr,
 * 3 cos_cr, 4 libm cbrt */
void orc_kino_math(int32_t f, int64_t n, const double* in, double* out);
