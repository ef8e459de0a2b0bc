// bspline_eval.cuh -- warp-cooperative evaluation of combineCost shared by the cost kernel
// (bspline.cu, compiled with -fmad=false: the reference's rounding sequence) and the solver
// kernel (bspline_solve.cu, FMA contraction allowed).
#pragma once
#include "common.cuh"

namespace {

constexpr int WPB = 4;  // warps (trajectories) per CTA

// getDistWithGrad for the solver: the ESDF samples are fp32, so the 7 lerps and the gradient are
// evaluated in fp32 (the voxel index and the fractional offsets still come from fp64 positions).
// "No site" samples are +inf: d is then inf/NaN, `d < dist0` is false and the gradient is unused,
// which is what the reference's 1.34e153 sentinel does to the cost as well.
__device__ __forceinline__ double dev_dist_with_grad_fast(const Geom& g, const float* __restrict__ dist,
                                                          const double pos[3], double grad[3]) {
  if (pos[0] < g.origin[0] + 1e-4 || pos[1] < g.origin[1] + 1e-4 || pos[2] < g.origin[2] + 1e-4 ||
      pos[0] > g.map_max[0] - 1e-4 || pos[1] > g.map_max[1] - 1e-4 || pos[2] > g.map_max[2] - 1e-4) {
    grad[0] = grad[1] = grad[2] = 0.0;
    return 0.0;
  }
  int idx[3];
  float t[3];
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    const double u = (pos[i] - 0.5 * g.res - g.origin[i]) * g.res_inv;
    const double fl = floor(u);
    idx[i] = (int)fl;
    t[i] = (float)(u - fl);  // = (pos - indexToPos(idx)) * res_inv
  }
  float v[2][2][2];
#pragma unroll
  for (int x = 0; x < 2; x++)
#pragma unroll
    for (int y = 0; y < 2; y++)
#pragma unroll
      for (int z = 0; z < 2; z++) {
        const int X = idx[0] + x, Y = idx[1] + y, Z = idx[2] + z;
        const bool in = !(X < 0 || Y < 0 || Z < 0 || X > g.nx - 1 || Y > g.ny - 1 || Z > g.nz - 1);
        v[x][y][z] = in ? __ldg(dist + addr_of(g, X, Y, Z)) : -1.0f;  // getDistance(): -1 outside
      }
  const float ri = (float)g.res_inv;
  const float v00 = (1 - t[0]) * v[0][0][0] + t[0] * v[1][0][0];
  const float v01 = (1 - t[0]) * v[0][0][1] + t[0] * v[1][0][1];
  const float v10 = (1 - t[0]) * v[0][1][0] + t[0] * v[1][1][0];
  const float v11 = (1 - t[0]) * v[0][1][1] + t[0] * v[1][1][1];
  const float v0 = (1 - t[1]) * v00 + t[1] * v10;
  const float v1 = (1 - t[1]) * v01 + t[1] * v11;
  const float d = (1 - t[2]) * v0 + t[2] * v1;
  grad[2] = (double)((v1 - v0) * ri);
  grad[1] = (double)(((1 - t[2]) * (v10 - v00) + t[2] * (v11 - v01)) * ri);
  float g0 = (1 - t[2]) * (1 - t[1]) * (v[1][0][0] - v[0][0][0]);
  g0 += (1 - t[2]) * t[1] * (v[1][1][0] - v[0][1][0]);
  g0 += t[2] * (1 - t[1]) * (v[1][0][1] - v[0][0][1]);
  g0 += t[2] * t[1] * (v[1][1][1] - v[0][1][1]);
  grad[0] = (double)(g0 * ri);
  return (double)d;
}

// =========================================================================================
// Warp-cooperative evaluation: lane i <-> control point i (n <= 32; with MINTIME n <= 31 in
// the optimiser, where lane n carries dt).  Control points stay in registers; neighbours
// come from warp shuffles; the 8 ESDF samples of every control point are gathered by its
// own lane, so one warp has 8*n independent loads in flight (L2-resident map).
// The accumulation order of every gradient row is the reference's loop order, so a row is
// bit-identical to the sequential restatement; only the scalar sums (costs, dt-gradient)
// are warp reductions and may differ in the last bits.
// =========================================================================================
__device__ __forceinline__ double wsum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
  return __shfl_sync(0xffffffffu, v, 0);
}
__device__ __forceinline__ double up(double v, int d, int lane) {
  const double r = __shfl_up_sync(0xffffffffu, v, d);
  return lane >= d ? r : 0.0;
}


// calcViewCost (bspline_optimizer.cpp:477-502) for the constrained control point qi = q[view_idx]: returns the
// cost and the gradient row of that point (all other rows are zero).  Eigen's expressions evaluated element-wise
// in written order (v = dir/sqrt(dir.dir); dn = qp - (qp.v) v; g = (2 (I - v vT)) dn; dl = (qp.v) v; if |dl| < |dir|:
// cost += wnl (|dl| - |dir|)^2, g += ((wnl 2 (|dl| - |dir|)) v vT) dl / |dl|).
__device__ __forceinline__ double view_cost_point(const double qi[3], const double* __restrict__ pt,
                                                  const double* __restrict__ dir, double wnl, double g[3]) {
  const double zz = dir[0] * dir[0] + dir[1] * dir[1] + dir[2] * dir[2];
  double v[3] = { dir[0], dir[1], dir[2] };
  if (zz > 0) {
    const double nrm = sqrt(zz);
#pragma unroll
    for (int k = 0; k < 3; ++k) v[k] = dir[k] / nrm;
  }
  const double qp[3] = { qi[0] - pt[0], qi[1] - pt[1], qi[2] - pt[2] };
  const double s = qp[0] * v[0] + qp[1] * v[1] + qp[2] * v[2];
  double dn[3], dl[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    dl[k] = s * v[k];
    dn[k] = qp[k] - dl[k];
  }
  double cost = dn[0] * dn[0] + dn[1] * dn[1] + dn[2] * dn[2];
#pragma unroll
  for (int r = 0; r < 3; ++r) {
    double acc = 0.0;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const double ivv = (r == c ? 1.0 : 0.0) - v[r] * v[c];
      const double term = (2 * ivv) * dn[c];
      acc = c == 0 ? term : acc + term;
    }
    g[r] = acc;
  }
  const double norm_dl = sqrt(dl[0] * dl[0] + dl[1] * dl[1] + dl[2] * dl[2]);
  const double safe_dist = sqrt(zz);
  if (norm_dl < safe_dist) {
    const double e = norm_dl - safe_dist;
    cost += wnl * (e * e);
    const double cc = wnl * 2 * e;
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      double acc = 0.0;
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const double term = (cc * (v[r] * v[c])) * dl[c];
        acc = c == 0 ? term : acc + term;
      }
      g[r] += acc / norm_dl;
    }
  }
  return cost;
}

struct TrajRegs {  // loop-invariant per-trajectory constants, loaded once
  double pt_dist, knot_span, time_lb;
  double start[3][3];
  double end[3][3];
  int n_end, n_guide, n_waypt;
};

__device__ __forceinline__ void load_traj(const FuelTrajConst* __restrict__ tc, TrajRegs& r) {
  r.pt_dist = tc->pt_dist;
  r.knot_span = tc->knot_span;
  r.time_lb = tc->time_lb;
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      r.start[i][k] = tc->start[i][k];
      r.end[i][k] = tc->end[i][k];
    }
  r.n_end = tc->n_end;
  r.n_guide = tc->n_guide;
  r.n_waypt = tc->n_waypt;
}

// calcWaypointsCost, calcViewCost and calcTimeCost, the last terms of combineCost: warp-uniform costs (added to f in
// every lane) and gradient rows of single lanes, evaluated the same way by both evaluators.
__device__ __forceinline__ void tail_terms(const FuelOptParams& p, const FuelTrajConst* __restrict__ tc, int n, int mask,
                                           const double q[3], double dt, int lane, int n_waypt, double time_lb,
                                           double& f, double gr[3], double& gdt) {
  if (mask & FUELGPU_WAYPOINTS) {  // calcWaypointsCost :433-457
    double cost = 0.0, gq[3] = { 0.0, 0.0, 0.0 };
    for (int w = 0; w < n_waypt; ++w) {
      const int idx = tc->waypt_idx[w];
      double dq[3];
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        const double a = __shfl_sync(0xffffffffu, q[k], idx);
        const double b = __shfl_sync(0xffffffffu, q[k], idx + 1);
        const double c = __shfl_sync(0xffffffffu, q[k], idx + 2);
        dq[k] = 1 / 6.0 * (a + 4 * b + c) - tc->waypt[w][k];
      }
      cost += dq[0] * dq[0] + dq[1] * dq[1] + dq[2] * dq[2];
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        if (lane == idx) gq[k] += dq[k] * (2.0 / 6.0);
        if (lane == idx + 1) gq[k] += dq[k] * (8.0 / 6.0);
        if (lane == idx + 2) gq[k] += dq[k] * (2.0 / 6.0);
      }
    }
    f += p.ld_waypt * cost;
#pragma unroll
    for (int k = 0; k < 3; ++k) gr[k] += p.ld_waypt * gq[k];
  }
  if (mask & FUELGPU_VIEWCONS) {  // calcViewCost :477-502: one control point, every lane evaluates it (no reduction)
    const int idx = tc->view_idx;
    if (idx >= 0 && idx < n) {
      double qi[3], gv[3];
#pragma unroll
      for (int k = 0; k < 3; ++k) qi[k] = __shfl_sync(0xffffffffu, q[k], idx);
      const double c = view_cost_point(qi, tc->view_pt, tc->view_dir, p.wnl, gv);
      f += p.ld_view * c;
      if (lane == idx) {
#pragma unroll
        for (int k = 0; k < 3; ++k) gr[k] += p.ld_view * gv[k];
      }
    }
  }
  if (mask & FUELGPU_MINTIME) {  // calcTimeCost :504-516
    const double duration = (n - p.order) * dt;
    double cost = duration;
    double gt = (double)(n - p.order);
    if (time_lb > 0 && duration < time_lb) {
      const double w_lb = 10;
      cost += w_lb * (duration - time_lb) * (duration - time_lb);
      gt += w_lb * 2 * (duration - time_lb) * (n - p.order);
    }
    f += p.ld_time * cost;
    gdt += p.ld_time * gt;
  }
}

// q[3]: this lane's control point (lanes >= n hold anything finite).  Returns f in every
// lane, this lane's gradient row in gr[3] (zero for lanes >= n) and the dt-gradient in gdt.
// The faithful evaluator (cost_batch, and min_cost_ at the solver's returned x); the solver
// loop runs eval_warp_fast below.
__device__ __forceinline__ void eval_warp(const Geom& g, const float* __restrict__ dist,
                                          const FuelOptParams& p, const TrajRegs& t,
                                          const FuelTrajConst* __restrict__ tc, int n, int mask,
                                          const double q[3], double dt, int lane, double& f_out,
                                          double gr[3], double& gdt) {
  const bool opt_time = (mask & FUELGPU_MINTIME) != 0;
  const bool act = lane < n;
  double f = 0.0;
  gr[0] = gr[1] = gr[2] = 0.0;
  gdt = 0.0;

  // neighbours i+1..i+3
  double q1[3], q2[3], q3[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    q1[k] = __shfl_down_sync(0xffffffffu, q[k], 1);
    q2[k] = __shfl_down_sync(0xffffffffu, q[k], 2);
    q3[k] = __shfl_down_sync(0xffffffffu, q[k], 3);
  }

  if (mask & FUELGPU_SMOOTHNESS) {  // calcSmoothnessCost :255-282
    const bool v = lane <= n - 4;
    double tj[3], c = 0.0;
    {
      double ji[3];
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        const double num = q3[k] - 3 * q2[k] + 3 * q1[k] - q[k];
        ji[k] = num / t.pt_dist;
      }
      c = ji[0] * ji[0] + ji[1] * ji[1] + ji[2] * ji[2];
#pragma unroll
      for (int k = 0; k < 3; ++k) tj[k] = v ? 2 * ji[k] / t.pt_dist : 0.0;
      if (!v) c = 0.0;
    }
    f += p.ld_smooth * wsum(c);
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const double t1 = up(tj[k], 1, lane), t2 = up(tj[k], 2, lane), t3 = up(tj[k], 3, lane);
      double gq = 0.0;
      gq += t3;          // i = p-3: gq[i+3] +=  tj
      gq += -3.0 * t2;   // i = p-2: gq[i+2] += -3 tj
      gq += 3.0 * t1;    // i = p-1: gq[i+1] +=  3 tj
      gq += -tj[k];      // i = p  : gq[i]   += -tj
      gr[k] += p.ld_smooth * gq;
    }
  }
  if (mask & FUELGPU_DISTANCE) {  // calcDistanceCost :284-306
    double c = 0.0, gq[3] = { 0.0, 0.0, 0.0 };
    if (act) {
      double dg[3];
      const double d = dev_dist_with_grad(g, dist, q, dg);
      const double nrm = sqrt(dg[0] * dg[0] + dg[1] * dg[1] + dg[2] * dg[2]);
      if (nrm > 1e-4) {
        dg[0] /= nrm;
        dg[1] /= nrm;
        dg[2] /= nrm;
      }
      if (d < p.dist0) {
        c = (d - p.dist0) * (d - p.dist0);
#pragma unroll
        for (int k = 0; k < 3; ++k) gq[k] += 2.0 * (d - p.dist0) * dg[k];
      }
    }
    f += p.ld_dist * wsum(c);
#pragma unroll
    for (int k = 0; k < 3; ++k) gr[k] += p.ld_dist * gq[k];
  }
  if (mask & FUELGPU_FEASIBILITY) {  // calcFeasibilityCost :308-353
    const double dt_inv = 1 / dt;
    const double dt_inv2 = dt_inv * dt_inv;
    double c = 0.0, gtl = 0.0;
    double tv[3], ta[3];
    const bool vv = lane <= n - 2, va = lane <= n - 3;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      tv[k] = 0.0;
      const double vi = (q1[k] - q[k]) * dt_inv;
      const double vd = fabs(vi) - p.max_vel;
      if (vv && vd > 0.0) {
        c += vd * vd;
        const double sign = vi > 0 ? 1.0 : -1.0;
        tv[k] = 2 * vd * sign * dt_inv;
        if (opt_time) gtl += tv[k] * (-vi);
      }
    }
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      ta[k] = 0.0;
      const double ai = (q2[k] - 2 * q1[k] + q[k]) * dt_inv2;
      const double ad = fabs(ai) - p.max_acc;
      if (va && ad > 0.0) {
        c += ad * ad;
        const double sign = ai > 0 ? 1.0 : -1.0;
        ta[k] = 2 * ad * sign * dt_inv2;
        if (opt_time) gtl += ta[k] * ai * (-2) * dt;
      }
    }
    f += p.ld_feasi * wsum(c);
    const double gt = wsum(gtl);
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const double v1 = up(tv[k], 1, lane);
      const double a1 = up(ta[k], 1, lane), a2 = up(ta[k], 2, lane);
      double gq = 0.0;
      gq += v1;          // velocity loop, i = p-1: gq[i+1] += tmp
      gq += -tv[k];      //                i = p  : gq[i]   += -tmp
      gq += a2;          // acceleration loop, i = p-2: gq[i+2] += tmp
      gq += -2 * a1;     //                    i = p-1: gq[i+1] += -2 tmp
      gq += ta[k];       //                    i = p  : gq[i]   += tmp
      gr[k] += p.ld_feasi * gq;
    }
    if (opt_time) gdt += p.ld_feasi * gt;
  }
  if (mask & FUELGPU_START) {  // calcStartCost :355-391
    double a[3], b[3], c3[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      a[k] = __shfl_sync(0xffffffffu, q[k], 0);
      b[k] = __shfl_sync(0xffffffffu, q[k], 1);
      c3[k] = __shfl_sync(0xffffffffu, q[k], 2);
    }
    const double w_pos = 10.0;
    double cost = 0.0, gt = 0.0, row[3] = { 0.0, 0.0, 0.0 };
    double dq[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) dq[k] = 1 / 6.0 * (a[k] + 4 * b[k] + c3[k]) - t.start[0][k];
    cost += w_pos * (dq[0] * dq[0] + dq[1] * dq[1] + dq[2] * dq[2]);
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      if (lane == 0) row[k] += w_pos * 2 * dq[k] * (1 / 6.0);
      if (lane == 1) row[k] += w_pos * 2 * dq[k] * (4 / 6.0);
      if (lane == 2) row[k] += w_pos * 2 * dq[k] * (1 / 6.0);
    }
#pragma unroll
    for (int k = 0; k < 3; ++k) dq[k] = 1 / (2 * dt) * (c3[k] - a[k]) - t.start[1][k];
    cost += dq[0] * dq[0] + dq[1] * dq[1] + dq[2] * dq[2];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      if (lane == 0) row[k] += 2 * dq[k] * (-1.0) / (2 * dt);
      if (lane == 2) row[k] += 2 * dq[k] * 1.0 / (2 * dt);
    }
    if (opt_time) {
      double d = 0;
#pragma unroll
      for (int k = 0; k < 3; ++k) d += dq[k] * (c3[k] - a[k]);
      gt += d / (-dt * dt);
    }
#pragma unroll
    for (int k = 0; k < 3; ++k) dq[k] = 1 / (dt * dt) * (a[k] - 2 * b[k] + c3[k]) - t.start[2][k];
    cost += dq[0] * dq[0] + dq[1] * dq[1] + dq[2] * dq[2];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      if (lane == 0) row[k] += 2 * dq[k] * 1.0 / (dt * dt);
      if (lane == 1) row[k] += 2 * dq[k] * (-2.0) / (dt * dt);
      if (lane == 2) row[k] += 2 * dq[k] * 1.0 / (dt * dt);
    }
    if (opt_time) {
      double d = 0;
#pragma unroll
      for (int k = 0; k < 3; ++k) d += dq[k] * (a[k] - 2 * b[k] + c3[k]);
      gt += d / (-dt * dt * dt);
    }
    f += p.ld_start * cost;
    if (lane < 3) {
#pragma unroll
      for (int k = 0; k < 3; ++k) gr[k] += p.ld_start * row[k];
    }
    if (opt_time) gdt += p.ld_start * gt;
  }
  if (mask & FUELGPU_END) {  // calcEndCost :393-431
    double q_3[3], q_2[3], q_1[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      q_3[k] = __shfl_sync(0xffffffffu, q[k], n - 3);
      q_2[k] = __shfl_sync(0xffffffffu, q[k], n - 2);
      q_1[k] = __shfl_sync(0xffffffffu, q[k], n - 1);
    }
    double cost = 0.0, gt = 0.0, row[3] = { 0.0, 0.0, 0.0 };
    double dq[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) dq[k] = 1 / 6.0 * (q_1[k] + 4 * q_2[k] + q_3[k]) - t.end[0][k];
    cost += dq[0] * dq[0] + dq[1] * dq[1] + dq[2] * dq[2];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      if (lane == n - 1) row[k] += 2 * dq[k] * (1 / 6.0);
      if (lane == n - 2) row[k] += 2 * dq[k] * (4 / 6.0);
      if (lane == n - 3) row[k] += 2 * dq[k] * (1 / 6.0);
    }
    if (t.n_end >= 2) {
#pragma unroll
      for (int k = 0; k < 3; ++k) dq[k] = 1 / (2 * dt) * (q_1[k] - q_3[k]) - t.end[1][k];
      cost += dq[0] * dq[0] + dq[1] * dq[1] + dq[2] * dq[2];
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        if (lane == n - 1) row[k] += 2 * dq[k] * 1.0 / (2 * dt);
        if (lane == n - 3) row[k] += 2 * dq[k] * (-1.0) / (2 * dt);
      }
      if (opt_time) {
        double d = 0;
#pragma unroll
        for (int k = 0; k < 3; ++k) d += dq[k] * (q_1[k] - q_3[k]);
        gt += d / (-dt * dt);
      }
    }
    if (t.n_end == 3) {
#pragma unroll
      for (int k = 0; k < 3; ++k) dq[k] = 1 / (dt * dt) * (q_1[k] - 2 * q_2[k] + q_3[k]) - t.end[2][k];
      cost += dq[0] * dq[0] + dq[1] * dq[1] + dq[2] * dq[2];
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        if (lane == n - 1) row[k] += 2 * dq[k] * 1.0 / (dt * dt);
        if (lane == n - 2) row[k] += 2 * dq[k] * (-2.0) / (dt * dt);
        if (lane == n - 3) row[k] += 2 * dq[k] * 1.0 / (dt * dt);
      }
      if (opt_time) {
        double d = 0;
#pragma unroll
        for (int k = 0; k < 3; ++k) d += dq[k] * (q_1[k] - 2 * q_2[k] + q_3[k]);
        gt += d / (-dt * dt * dt);
      }
    }
    f += p.ld_end * cost;
    if (lane >= n - 3 && lane < n) {
#pragma unroll
      for (int k = 0; k < 3; ++k) gr[k] += p.ld_end * row[k];
    }
    if (opt_time) gdt += p.ld_end * gt;
  }
  if (mask & FUELGPU_GUIDE) {  // calcGuideCost :462-475
    double c = 0.0, gq[3] = { 0.0, 0.0, 0.0 };
    if (lane >= p.order && lane < n - p.order) {
      double d[3];
#pragma unroll
      for (int k = 0; k < 3; ++k) d[k] = q[k] - tc->guide[lane - p.order][k];
      c = d[0] * d[0] + d[1] * d[1] + d[2] * d[2];
#pragma unroll
      for (int k = 0; k < 3; ++k) gq[k] += 2 * d[k];
    }
    f += p.ld_guide * wsum(c);
#pragma unroll
    for (int k = 0; k < 3; ++k) gr[k] += p.ld_guide * gq[k];
  }
  tail_terms(p, tc, n, mask, q, dt, lane, t.n_waypt, t.time_lb, f, gr, gdt);
  if (!act) gr[0] = gr[1] = gr[2] = 0.0;
  f_out = f;
}

// What the FAST evaluator keeps in registers across a solve; the boundary states are read from the trajectory's
// constants by the two lanes that use them.
struct TrajFast {
  double inv_pt, time_lb;
  int n_end, n_waypt;
};

__device__ __forceinline__ void load_traj_fast(const FuelTrajConst* __restrict__ tc, TrajFast& r) {
  r.inv_pt = 1.0 / tc->pt_dist;
  r.time_lb = tc->time_lb;
  r.n_end = tc->n_end;
  r.n_waypt = tc->n_waypt;
}

// The evaluator of the solver loop (and of FUELGPU_COST_FAST_EVAL): same terms and mathematics as eval_warp, same
// outputs, but written for a short dependent chain per evaluation.
//  * Divisions by loop-invariant scalars are multiplications by reciprocals, the ESDF samples are lerped in fp32
//    and the ESDF gradient is normalised with rsqrt.
//  * Every term adds what it owes to the rows of lanes i+1, i+2, i+3 into one vector per offset (o1, o2, o3), and each
//    vector goes up the warp with ONE shuffle: 9 fp64 shuffles for all terms together.
//  * calcStartCost runs on lane 0 and calcEndCost on lane n-3 (n >= 4): each holds its three points in q, q1, q2
//    already, so neither needs a broadcast, and both run in the same pass.
//  * Every cost and dt-gradient term is a per-lane partial; one merged butterfly reduces both at the end.
// Rounding differs from eval_warp in the last bits.
__device__ __forceinline__ void eval_warp_fast(const Geom& g, const float* __restrict__ dist, const FuelOptParams& p,
                                               const TrajFast& t, const FuelTrajConst* __restrict__ tc, int n,
                                               int mask, const double q[3], double dt, int lane, double& f_out,
                                               double gr[3], double& gdt) {
  const bool opt_time = (mask & FUELGPU_MINTIME) != 0;
  const bool act = lane < n;
  double f = 0.0;                       // warp-uniform terms
  double f_lane = 0.0, gdt_lane = 0.0;  // per-lane partial sums, reduced once at the end
  gdt = 0.0;
  const double dt_inv = 1.0 / dt;
  const double dt_inv2 = dt_inv * dt_inv, inv2dt = 0.5 * dt_inv;

  // neighbours i+1..i+3
  double q1[3], q2[3], q3[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    q1[k] = __shfl_down_sync(0xffffffffu, q[k], 1);
    q2[k] = __shfl_down_sync(0xffffffffu, q[k], 2);
    q3[k] = __shfl_down_sync(0xffffffffu, q[k], 3);
  }
  // this lane's own gradient row, and what its terms add to the rows of lanes i+1, i+2, i+3
  double own[3] = { 0.0, 0.0, 0.0 }, o1[3] = { 0.0, 0.0, 0.0 }, o2[3] = { 0.0, 0.0, 0.0 }, o3[3] = { 0.0, 0.0, 0.0 };

  if ((mask & FUELGPU_SMOOTHNESS) && lane <= n - 4) {  // calcSmoothnessCost :255-282
    double ji[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) ji[k] = (q3[k] - 3 * q2[k] + 3 * q1[k] - q[k]) * t.inv_pt;
    f_lane += p.ld_smooth * (ji[0] * ji[0] + ji[1] * ji[1] + ji[2] * ji[2]);
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const double tj = p.ld_smooth * 2 * ji[k] * t.inv_pt;
      own[k] -= tj;
      o1[k] += 3.0 * tj;
      o2[k] -= 3.0 * tj;
      o3[k] += tj;
    }
  }
  if ((mask & FUELGPU_DISTANCE) && act) {  // calcDistanceCost :284-306
    double dg[3];
    const double d = dev_dist_with_grad_fast(g, dist, q, dg);
    const double n2 = dg[0] * dg[0] + dg[1] * dg[1] + dg[2] * dg[2];
    if (n2 > 1e-8) {
      const double rn = rsqrt(n2);
      dg[0] *= rn;
      dg[1] *= rn;
      dg[2] *= rn;
    }
    if (d < p.dist0) {
      f_lane += p.ld_dist * ((d - p.dist0) * (d - p.dist0));
#pragma unroll
      for (int k = 0; k < 3; ++k) own[k] += p.ld_dist * (2.0 * (d - p.dist0) * dg[k]);
    }
  }
  if (mask & FUELGPU_FEASIBILITY) {  // calcFeasibilityCost :308-353
    double c = 0.0, gtl = 0.0;
    const bool vv = lane <= n - 2, va = lane <= n - 3;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const double vi = (q1[k] - q[k]) * dt_inv;
      const double vd = fabs(vi) - p.max_vel;
      if (vv && vd > 0.0) {
        c += vd * vd;
        const double tv = 2 * vd * (vi > 0 ? 1.0 : -1.0) * dt_inv;
        if (opt_time) gtl += tv * (-vi);
        own[k] -= p.ld_feasi * tv;
        o1[k] += p.ld_feasi * tv;
      }
    }
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const double ai = (q2[k] - 2 * q1[k] + q[k]) * dt_inv2;
      const double ad = fabs(ai) - p.max_acc;
      if (va && ad > 0.0) {
        c += ad * ad;
        const double ta = 2 * ad * (ai > 0 ? 1.0 : -1.0) * dt_inv2;
        if (opt_time) gtl += ta * ai * (-2) * dt;
        own[k] += p.ld_feasi * ta;
        o1[k] -= 2.0 * p.ld_feasi * ta;
        o2[k] += p.ld_feasi * ta;
      }
    }
    f_lane += p.ld_feasi * c;
    gdt_lane += p.ld_feasi * gtl;
  }
  // calcStartCost :355-391 (lane 0: points 0, 1, 2) and calcEndCost :393-431 (lane n-3: points n-3, n-2, n-1)
  const bool do_start = (mask & FUELGPU_START) && lane == 0, do_end = (mask & FUELGPU_END) && lane == n - 3;
  if (do_start || do_end) {
    const double(*st)[3] = do_start ? tc->start : tc->end;
    const double w_pos = do_start ? 10.0 : 1.0, ld = do_start ? p.ld_start : p.ld_end;
    const bool use_v = do_start || t.n_end >= 2, use_a = do_start || t.n_end == 3;
    double cost = 0.0, gt = 0.0;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const double dv = q2[k] - q[k], da = q[k] - 2 * q1[k] + q2[k];
      const double dqp = 1 / 6.0 * (q[k] + 4 * q1[k] + q2[k]) - __ldg(&st[0][k]);
      const double dqv = use_v ? inv2dt * dv - __ldg(&st[1][k]) : 0.0;
      const double dqa = use_a ? dt_inv2 * da - __ldg(&st[2][k]) : 0.0;
      cost += w_pos * dqp * dqp + dqv * dqv + dqa * dqa;
      gt -= dqv * dv * dt_inv2 + dqa * da * dt_inv2 * dt_inv;
      const double ep = ld * 2.0 * w_pos * dqp, ev = ld * 2.0 * dqv, ea = ld * 2.0 * dqa;
      own[k] += ep * (1 / 6.0) - ev * inv2dt + ea * dt_inv2;
      o1[k] += ep * (4 / 6.0) - 2.0 * ea * dt_inv2;
      o2[k] += ep * (1 / 6.0) + ev * inv2dt + ea * dt_inv2;
    }
    f_lane += ld * cost;
    if (opt_time) gdt_lane += ld * gt;
  }
#pragma unroll
  for (int k = 0; k < 3; ++k) gr[k] = own[k] + up(o1[k], 1, lane) + up(o2[k], 2, lane) + up(o3[k], 3, lane);

  if (mask & FUELGPU_GUIDE) {  // calcGuideCost :462-475
    if (lane >= p.order && lane < n - p.order) {
      double d[3];
#pragma unroll
      for (int k = 0; k < 3; ++k) d[k] = q[k] - tc->guide[lane - p.order][k];
      f_lane += p.ld_guide * (d[0] * d[0] + d[1] * d[1] + d[2] * d[2]);
#pragma unroll
      for (int k = 0; k < 3; ++k) gr[k] += p.ld_guide * (2 * d[k]);
    }
  }
  tail_terms(p, tc, n, mask, q, dt, lane, t.n_waypt, t.time_lb, f, gr, gdt);
  // one butterfly for both scalars (the two chains interleave)
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    f_lane += __shfl_down_sync(0xffffffffu, f_lane, o);
    gdt_lane += __shfl_down_sync(0xffffffffu, gdt_lane, o);
  }
  f += __shfl_sync(0xffffffffu, f_lane, 0);
  if (opt_time) gdt += __shfl_sync(0xffffffffu, gdt_lane, 0);
  if (!act) gr[0] = gr[1] = gr[2] = 0.0;
  f_out = f;
}

}  // namespace
