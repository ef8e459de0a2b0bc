// bspline.cu -- batched B-spline cost/gradient (BsplineOptimizer::combineCost) on sm_90a.
//
// Replaces bspline_opt/src/bspline_optimizer.cpp:518-647 (combineCost) and the calc*Cost
// functions it calls (:255-516), evaluated for a batch of trajectories against one ESDF
// (EDTEnvironment::evaluateEDTWithGrad -> SDFMap::getDistWithGrad, sdf_map.cpp:497-536).
// fp64 throughout; products and sums are kept in the reference's order and are not
// contracted into FMAs (-fmad=false for this file), so results agree with the host
// arithmetic to rounding of the fp32 ESDF samples.
#include "common.cuh"
#include "bspline_eval.cuh"

namespace {

constexpr int MAXP = FUELGPU_MAX_PTS;

struct Terms {
  double f;
  double gt;
};

// One trajectory's full combineCost, sequential restatement.  q/g live in local memory
// (thread-per-trajectory variant) -- the warp-cooperative kernel below is the fast path.
__device__ void combine_cost_thread(const Geom& g, const float* __restrict__ dist,
                                    const FuelOptParams& p, const FuelTrajConst& tc, int n, int mask,
                                    const double* __restrict__ x, double* __restrict__ fout,
                                    double* __restrict__ grad) {
  const bool opt_time = (mask & FUELGPU_MINTIME) != 0;
  const int nvar = opt_time ? 3 * n + 1 : 3 * n;
  const double dt = opt_time ? x[nvar - 1] : tc.knot_span;
  double q[MAXP][3];
  double gq[MAXP][3];
  for (int i = 0; i < n; ++i)
    for (int k = 0; k < 3; ++k) q[i][k] = x[3 * i + k];
  for (int i = 0; i < nvar; ++i) grad[i] = 0.0;
  double f_combine = 0.0;

  if (mask & FUELGPU_SMOOTHNESS) {  // calcSmoothnessCost :255-282
    double cost = 0.0;
    for (int i = 0; i < n; ++i) gq[i][0] = gq[i][1] = gq[i][2] = 0.0;
    for (int i = 0; i < n - 3; i++) {
      double ji[3], tj[3];
      for (int k = 0; k < 3; ++k)
        ji[k] = (q[i + 3][k] - 3 * q[i + 2][k] + 3 * q[i + 1][k] - q[i][k]) / tc.pt_dist;
      cost += ji[0] * ji[0] + ji[1] * ji[1] + ji[2] * ji[2];
      for (int k = 0; k < 3; ++k) tj[k] = 2 * ji[k] / tc.pt_dist;
      for (int k = 0; k < 3; ++k) {
        gq[i + 0][k] += -tj[k];
        gq[i + 1][k] += 3.0 * tj[k];
        gq[i + 2][k] += -3.0 * tj[k];
        gq[i + 3][k] += tj[k];
      }
    }
    f_combine += p.ld_smooth * cost;
    for (int i = 0; i < n; i++)
      for (int k = 0; k < 3; k++) grad[3 * i + k] += p.ld_smooth * gq[i][k];
    if (opt_time) grad[nvar - 1] += p.ld_smooth * 0.0;
  }
  if (mask & FUELGPU_DISTANCE) {  // calcDistanceCost :284-306
    double cost = 0.0;
    for (int i = 0; i < n; i++) {
      double dg[3];
      const double d = dev_dist_with_grad(g, dist, q[i], dg);
      const double nrm = sqrt(dg[0] * dg[0] + dg[1] * dg[1] + dg[2] * dg[2]);
      if (nrm > 1e-4) {
        dg[0] /= nrm;
        dg[1] /= nrm;
        dg[2] /= nrm;
      }
      gq[i][0] = gq[i][1] = gq[i][2] = 0.0;
      if (d < p.dist0) {
        cost += (d - p.dist0) * (d - p.dist0);
        for (int k = 0; k < 3; ++k) gq[i][k] += 2.0 * (d - p.dist0) * dg[k];
      }
    }
    f_combine += p.ld_dist * cost;
    for (int i = 0; i < n; i++)
      for (int k = 0; k < 3; k++) grad[3 * i + k] += p.ld_dist * gq[i][k];
  }
  if (mask & FUELGPU_FEASIBILITY) {  // calcFeasibilityCost :308-353
    double cost = 0.0, gt = 0.0;
    for (int i = 0; i < n; ++i) gq[i][0] = gq[i][1] = gq[i][2] = 0.0;
    const double dt_inv = 1 / dt;
    const double dt_inv2 = dt_inv * dt_inv;
    for (int i = 0; i < n - 1; ++i)
      for (int k = 0; k < 3; ++k) {
        const double vi = (q[i + 1][k] - q[i][k]) * dt_inv;
        const double vd = fabs(vi) - p.max_vel;
        if (vd > 0.0) {
          cost += vd * vd;
          const double sign = vi > 0 ? 1.0 : -1.0;
          const double tmp = 2 * vd * sign * dt_inv;
          gq[i][k] += -tmp;
          gq[i + 1][k] += tmp;
          if (opt_time) gt += tmp * (-vi);
        }
      }
    for (int i = 0; i < n - 2; ++i)
      for (int k = 0; k < 3; ++k) {
        const double ai = (q[i + 2][k] - 2 * q[i + 1][k] + q[i][k]) * dt_inv2;
        const double ad = fabs(ai) - p.max_acc;
        if (ad > 0.0) {
          cost += ad * ad;
          const double sign = ai > 0 ? 1.0 : -1.0;
          const double tmp = 2 * ad * sign * dt_inv2;
          gq[i][k] += tmp;
          gq[i + 1][k] += -2 * tmp;
          gq[i + 2][k] += tmp;
          if (opt_time) gt += tmp * ai * (-2) * dt;
        }
      }
    f_combine += p.ld_feasi * cost;
    for (int i = 0; i < n; i++)
      for (int k = 0; k < 3; k++) grad[3 * i + k] += p.ld_feasi * gq[i][k];
    if (opt_time) grad[nvar - 1] += p.ld_feasi * gt;
  }
  if (mask & FUELGPU_START) {  // calcStartCost :355-391
    double cost = 0.0, gt = 0.0;
    for (int i = 0; i < 3; ++i) gq[i][0] = gq[i][1] = gq[i][2] = 0.0;
    const double w_pos = 10.0;
    double dq[3];
    for (int k = 0; k < 3; ++k) dq[k] = 1 / 6.0 * (q[0][k] + 4 * q[1][k] + q[2][k]) - tc.start[0][k];
    cost += w_pos * (dq[0] * dq[0] + dq[1] * dq[1] + dq[2] * dq[2]);
    for (int k = 0; k < 3; ++k) {
      gq[0][k] += w_pos * 2 * dq[k] * (1 / 6.0);
      gq[1][k] += w_pos * 2 * dq[k] * (4 / 6.0);
      gq[2][k] += w_pos * 2 * dq[k] * (1 / 6.0);
    }
    for (int k = 0; k < 3; ++k) dq[k] = 1 / (2 * dt) * (q[2][k] - q[0][k]) - tc.start[1][k];
    cost += dq[0] * dq[0] + dq[1] * dq[1] + dq[2] * dq[2];
    for (int k = 0; k < 3; ++k) {
      gq[0][k] += 2 * dq[k] * (-1.0) / (2 * dt);
      gq[2][k] += 2 * dq[k] * 1.0 / (2 * dt);
    }
    if (opt_time) {
      double d = 0;
      for (int k = 0; k < 3; ++k) d += dq[k] * (q[2][k] - q[0][k]);
      gt += d / (-dt * dt);
    }
    for (int k = 0; k < 3; ++k) dq[k] = 1 / (dt * dt) * (q[0][k] - 2 * q[1][k] + q[2][k]) - tc.start[2][k];
    cost += dq[0] * dq[0] + dq[1] * dq[1] + dq[2] * dq[2];
    for (int k = 0; k < 3; ++k) {
      gq[0][k] += 2 * dq[k] * 1.0 / (dt * dt);
      gq[1][k] += 2 * dq[k] * (-2.0) / (dt * dt);
      gq[2][k] += 2 * dq[k] * 1.0 / (dt * dt);
    }
    if (opt_time) {
      double d = 0;
      for (int k = 0; k < 3; ++k) d += dq[k] * (q[0][k] - 2 * q[1][k] + q[2][k]);
      gt += d / (-dt * dt * dt);
    }
    f_combine += p.ld_start * cost;
    for (int i = 0; i < 3; i++)
      for (int k = 0; k < 3; k++) grad[3 * i + k] += p.ld_start * gq[i][k];
    if (opt_time) grad[nvar - 1] += p.ld_start * gt;
  }
  if (mask & FUELGPU_END) {  // calcEndCost :393-431
    double cost = 0.0, gt = 0.0;
    for (int i = n - 3; i < n; ++i) gq[i][0] = gq[i][1] = gq[i][2] = 0.0;
    const double* q_3 = q[n - 3];
    const double* q_2 = q[n - 2];
    const double* q_1 = q[n - 1];
    double dq[3];
    for (int k = 0; k < 3; ++k) dq[k] = 1 / 6.0 * (q_1[k] + 4 * q_2[k] + q_3[k]) - tc.end[0][k];
    cost += dq[0] * dq[0] + dq[1] * dq[1] + dq[2] * dq[2];
    for (int k = 0; k < 3; ++k) {
      gq[n - 1][k] += 2 * dq[k] * (1 / 6.0);
      gq[n - 2][k] += 2 * dq[k] * (4 / 6.0);
      gq[n - 3][k] += 2 * dq[k] * (1 / 6.0);
    }
    if (tc.n_end >= 2) {
      for (int k = 0; k < 3; ++k) dq[k] = 1 / (2 * dt) * (q_1[k] - q_3[k]) - tc.end[1][k];
      cost += dq[0] * dq[0] + dq[1] * dq[1] + dq[2] * dq[2];
      for (int k = 0; k < 3; ++k) {
        gq[n - 1][k] += 2 * dq[k] * 1.0 / (2 * dt);
        gq[n - 3][k] += 2 * dq[k] * (-1.0) / (2 * dt);
      }
      if (opt_time) {
        double d = 0;
        for (int k = 0; k < 3; ++k) d += dq[k] * (q_1[k] - q_3[k]);
        gt += d / (-dt * dt);
      }
    }
    if (tc.n_end == 3) {
      for (int k = 0; k < 3; ++k) dq[k] = 1 / (dt * dt) * (q_1[k] - 2 * q_2[k] + q_3[k]) - tc.end[2][k];
      cost += dq[0] * dq[0] + dq[1] * dq[1] + dq[2] * dq[2];
      for (int k = 0; k < 3; ++k) {
        gq[n - 1][k] += 2 * dq[k] * 1.0 / (dt * dt);
        gq[n - 2][k] += 2 * dq[k] * (-2.0) / (dt * dt);
        gq[n - 3][k] += 2 * dq[k] * 1.0 / (dt * dt);
      }
      if (opt_time) {
        double d = 0;
        for (int k = 0; k < 3; ++k) d += dq[k] * (q_1[k] - 2 * q_2[k] + q_3[k]);
        gt += d / (-dt * dt * dt);
      }
    }
    f_combine += p.ld_end * cost;
    for (int i = n - 3; i < n; i++)
      for (int k = 0; k < 3; k++) grad[3 * i + k] += p.ld_end * gq[i][k];
    if (opt_time) grad[nvar - 1] += p.ld_end * gt;
  }
  if (mask & FUELGPU_GUIDE) {  // calcGuideCost :462-475
    double cost = 0.0;
    for (int i = 0; i < n; ++i) gq[i][0] = gq[i][1] = gq[i][2] = 0.0;
    const int end_idx = n - p.order;
    for (int i = p.order; i < end_idx; i++) {
      double d[3];
      for (int k = 0; k < 3; ++k) d[k] = q[i][k] - tc.guide[i - p.order][k];
      cost += d[0] * d[0] + d[1] * d[1] + d[2] * d[2];
      for (int k = 0; k < 3; ++k) gq[i][k] += 2 * d[k];
    }
    f_combine += p.ld_guide * cost;
    for (int i = 0; i < n; i++)
      for (int k = 0; k < 3; k++) grad[3 * i + k] += p.ld_guide * gq[i][k];
  }
  if (mask & FUELGPU_WAYPOINTS) {  // calcWaypointsCost :433-457
    double cost = 0.0;
    for (int i = 0; i < n; ++i) gq[i][0] = gq[i][1] = gq[i][2] = 0.0;
    for (int i = 0; i < tc.n_waypt; ++i) {
      const int idx = tc.waypt_idx[i];
      double dq[3];
      for (int k = 0; k < 3; ++k)
        dq[k] = 1 / 6.0 * (q[idx][k] + 4 * q[idx + 1][k] + q[idx + 2][k]) - tc.waypt[i][k];
      cost += dq[0] * dq[0] + dq[1] * dq[1] + dq[2] * dq[2];
      for (int k = 0; k < 3; ++k) {
        gq[idx][k] += dq[k] * (2.0 / 6.0);
        gq[idx + 1][k] += dq[k] * (8.0 / 6.0);
        gq[idx + 2][k] += dq[k] * (2.0 / 6.0);
      }
    }
    f_combine += p.ld_waypt * cost;
    for (int i = 0; i < n; i++)
      for (int k = 0; k < 3; k++) grad[3 * i + k] += p.ld_waypt * gq[i][k];
  }
  if (mask & FUELGPU_VIEWCONS) {  // calcViewCost :477-502
    const int idx = tc.view_idx;
    if (idx >= 0 && idx < n) {
      double gv[3];
      const double c = view_cost_point(q[idx], tc.view_pt, tc.view_dir, p.wnl, gv);
      f_combine += p.ld_view * c;
      for (int k = 0; k < 3; k++) grad[3 * idx + k] += p.ld_view * gv[k];
    }
  }
  if (mask & FUELGPU_MINTIME) {  // calcTimeCost :504-516
    const double duration = (n - p.order) * dt;
    double cost = duration;
    double gt = (double)(n - p.order);
    if (tc.time_lb > 0 && duration < tc.time_lb) {
      const double w_lb = 10;
      cost += w_lb * (duration - tc.time_lb) * (duration - tc.time_lb);
      gt += w_lb * 2 * (duration - tc.time_lb) * (n - p.order);
    }
    f_combine += p.ld_time * cost;
    grad[nvar - 1] += p.ld_time * gt;
  }
  *fout = f_combine;
}

__global__ void __launch_bounds__(64) cost_batch_thread_kernel(Geom g, const float* __restrict__ dist,
                                                               FuelOptParams p,
                                                               const FuelTrajConst* __restrict__ tc,
                                                               int n, int mask, int B,
                                                               const double* __restrict__ x,
                                                               double* __restrict__ f,
                                                               double* __restrict__ grad) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  const int nvar = (mask & FUELGPU_MINTIME) ? 3 * n + 1 : 3 * n;
  combine_cost_thread(g, dist, p, tc[b], n, mask, x + (int64_t)b * nvar, f + b, grad + (int64_t)b * nvar);
}



// FAST = the evaluator instantiation the solver loop runs (fp32 lerps, reciprocals, one merged reduction);
// reachable through FUELGPU_COST_FAST_EVAL so that the parity tests cover exactly what the benchmark times.
template <bool FAST>
__global__ void __launch_bounds__(WPB * 32) cost_batch_warp_kernel(
    Geom g, const float* __restrict__ dist, FuelOptParams p, const FuelTrajConst* __restrict__ tc, int n,
    int mask, int B, const double* __restrict__ x, double* __restrict__ f, double* __restrict__ grad) {
  const int lane = threadIdx.x & 31;
  const int b = blockIdx.x * WPB + (threadIdx.x >> 5);
  if (b >= B) return;
  const bool opt_time = (mask & FUELGPU_MINTIME) != 0;
  const int nvar = opt_time ? 3 * n + 1 : 3 * n;
  const double* xb = x + (int64_t)b * nvar;
  TrajRegs t;
  load_traj(tc + b, t);
  double q[3] = { 0.0, 0.0, 0.0 };
  if (lane < n) {
    q[0] = xb[3 * lane];
    q[1] = xb[3 * lane + 1];
    q[2] = xb[3 * lane + 2];
  }
  const double dt = opt_time ? xb[nvar - 1] : t.knot_span;
  double fo, gr[3], gdt;
  if constexpr (FAST) {
    TrajFast tf;
    load_traj_fast(tc + b, tf);
    eval_warp_fast(g, dist, p, tf, tc + b, n, mask, q, dt, lane, fo, gr, gdt);
  } else {
    eval_warp(g, dist, p, t, tc + b, n, mask, q, dt, lane, fo, gr, gdt);
  }
  double* gb = grad + (int64_t)b * nvar;
  if (lane < n) {
    gb[3 * lane] = gr[0];
    gb[3 * lane + 1] = gr[1];
    gb[3 * lane + 2] = gr[2];
  }
  if (lane == 0) {
    f[b] = fo;
    if (opt_time) gb[nvar - 1] = gdt;
  }
}

// FUELGPU_COST_FAST_EVAL for 32 < n <= 64: the two-points-per-lane evaluator of the long-trajectory solver
__global__ void __launch_bounds__(WPB * 32) cost_batch_warp2_kernel(
    Geom g, const float* __restrict__ dist, FuelOptParams p, const FuelTrajConst* __restrict__ tc, int n,
    int mask, int B, const double* __restrict__ x, double* __restrict__ f, double* __restrict__ grad) {
  const int lane = threadIdx.x & 31;
  const int b = blockIdx.x * WPB + (threadIdx.x >> 5);
  if (b >= B) return;
  const bool opt_time = (mask & FUELGPU_MINTIME) != 0;
  const int nvar = opt_time ? 3 * n + 1 : 3 * n;
  const double* xb = x + (int64_t)b * nvar;
  double q[2][3];
#pragma unroll
  for (int s = 0; s < 2; ++s) {
    const int i = 32 * s + lane;
#pragma unroll
    for (int k = 0; k < 3; ++k) q[s][k] = i < n ? xb[3 * i + k] : 0.0;
  }
  const double dt = opt_time ? xb[nvar - 1] : tc[b].knot_span;
  TrajFast tf;
  load_traj_fast(tc + b, tf);
  double fo, gr[2][3], gdt;
  eval_warp_fast2(g, dist, p, tf, tc + b, n, mask, q, dt, lane, fo, gr, gdt);
  double* gb = grad + (int64_t)b * nvar;
#pragma unroll
  for (int s = 0; s < 2; ++s) {
    const int i = 32 * s + lane;
    if (i < n) {
#pragma unroll
      for (int k = 0; k < 3; ++k) gb[3 * i + k] = gr[s][k];
    }
  }
  if (lane == 0) {
    f[b] = fo;
    if (opt_time) gb[nvar - 1] = gdt;
  }
}

}  // namespace

int bspline_cost_batch_dev_impl(FuelMap* m, int B, int n_pts, int mask, const FuelOptParams* p,
                                const FuelTrajConst* tc_dev, const double* x_dev, double* f_dev,
                                double* grad_dev) {
  if (B <= 0) return 0;
  const bool fast = (mask & FUELGPU_COST_FAST_EVAL) != 0;
  mask &= ~FUELGPU_COST_FAST_EVAL;
  if (fast && n_pts > 32) {
    cost_batch_warp2_kernel<<<(B + WPB - 1) / WPB, WPB * 32, 0, m->stream>>>(m->g, m->dist, *p, tc_dev, n_pts, mask, B,
                                                                            x_dev, f_dev, grad_dev);
  } else if (fast) {
    cost_batch_warp_kernel<true><<<(B + WPB - 1) / WPB, WPB * 32, 0, m->stream>>>(m->g, m->dist, *p, tc_dev, n_pts,
                                                                              mask, B, x_dev, f_dev, grad_dev);
  } else if (n_pts <= 32) {
    cost_batch_warp_kernel<false><<<(B + WPB - 1) / WPB, WPB * 32, 0, m->stream>>>(m->g, m->dist, *p, tc_dev, n_pts,
                                                                               mask, B, x_dev, f_dev, grad_dev);
  } else {
    cost_batch_thread_kernel<<<(B + 63) / 64, 64, 0, m->stream>>>(m->g, m->dist, *p, tc_dev, n_pts, mask, B,
                                                                  x_dev, f_dev, grad_dev);
  }
  FUEL_LAUNCHES(m, 1);
  FUEL_CUDA(m, cudaGetLastError());
  return 0;
}
