// bspline_solve_long.cu -- the persistent per-trajectory solver for 32 < n_pts + dt lanes (up to 64 control points).
// Compiled with FMA contraction enabled, like bspline_solve.cu; min_cost_ comes from the faithful cost kernel of
// bspline.cu at the returned x.
#include "bspline_eval.cuh"

namespace {

// =========================================================================================
// The contract of optimize_gram_kernel (bspline_solve.cu) -- clamp to the box shrunk by 0.1 m (:175-204), bounds
// q0 +- 10 m clipped to that box and dt in [0,5] (:206-217), maxeval and xtol_rel stops (:170-173), best-x tracking
// of costFunction (:693-706), projected L-BFGS with Armijo backtracking -- with two control points per lane: point i
// lives on lane i % 32, slot i / 32 (eval_warp_fast2), and dt is a warp-uniform scalar held by every lane.  One warp
// per trajectory; the iterate, gradient and direction stay in registers, the (s, y) history in shared memory (vector
// form of the two-loop recursion, fp32 storage).
// =========================================================================================
constexpr int LMAXM = 8;
constexpr int LONG_WPB = 2;  // warps (trajectories) per CTA

struct V6 {
  double v[2][3];  // [slot][component]
};

// Solver-internal inner products: each lane adds its two slots (dt on lane 0 only) in fp64, the 32-lane sum runs as
// an fp32 xor butterfly that lands in every lane (as wsum_x of bspline_solve.cu).  They only steer the direction;
// the cost that decides acceptance and best-x stays fp64.
__device__ __forceinline__ double dot6(const V6& a, double adt, const V6& b, double bdt, int lane) {
  double v = 0.0;
#pragma unroll
  for (int s = 0; s < 2; ++s)
#pragma unroll
    for (int k = 0; k < 3; ++k) v += a.v[s][k] * b.v[s][k];
  if (lane == 0) v += adt * bdt;
  float f = (float)v;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) f += __shfl_xor_sync(0xffffffffu, f, o);
  return (double)f;
}

// Shared memory per warp: box bounds LB, UB [2][3][32] doubles; the history S, Y [m][2][3][32] floats (ring order,
// conflict-free: lane fastest); the dt components of the history Sdt, Ydt [LMAXM] floats.
#define LONG_SMEM_BYTES(M) (2 * 192 * 8 + 2 * (M) * 192 * 4 + 2 * LMAXM * 4)
#define BIDX(s, k) (((s) * 3 + (k)) * 32 + lane)
#define HIDX2(slot, s, k) ((((slot) * 2 + (s)) * 3 + (k)) * 32 + lane)

__global__ void __launch_bounds__(LONG_WPB * 32) optimize_long_kernel(
    Geom g, const float* __restrict__ dist, FuelOptParams p, const FuelTrajConst* __restrict__ tc, int n,
    int mask, int B, FuelSolveParams sp, double* __restrict__ x, int* __restrict__ neval_out) {
  extern __shared__ double lsm[];
  const int lane = threadIdx.x & 31;
  const int w = threadIdx.x >> 5;
  const int b = blockIdx.x * LONG_WPB + w;
  if (b >= B) return;
  const bool opt_time = (mask & FUELGPU_MINTIME) != 0;
  const int nvar = opt_time ? 3 * n + 1 : 3 * n;
  const int m = sp.lbfgs_m;
  double* LB = lsm + (size_t)w * (LONG_SMEM_BYTES(m) / 8);
  double* UB = LB + 192;
  float* S = reinterpret_cast<float*>(UB + 192);
  float* Y = S + m * 192;
  float* Sdt = Y + m * 192;
  float* Ydt = Sdt + LMAXM;
  double* xb = x + (int64_t)b * nvar;
  TrajFast t;
  load_traj_fast(tc + b, t);
  const double knot_span = tc[b].knot_span;

  V6 X;
#pragma unroll
  for (int s = 0; s < 2; ++s) {
    const int i = 32 * s + lane;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      double c = 0.0, lo = 0.0, hi = 0.0;  // inactive points: pinned at 0 with a zero gradient
      if (i < n) {
        const double bmin = g.box_mind[k] + 0.1, bmax = g.box_maxd[k] - 0.1;
        c = fmax(fmin(xb[3 * i + k], bmax), bmin);  // :199-203
        lo = fmax(c - 10.0, bmin);                  // :208-214
        hi = fmin(c + 10.0, bmax);
      }
      X.v[s][k] = c;
      LB[BIDX(s, k)] = lo;
      UB[BIDX(s, k)] = hi;
    }
  }
  double Xdt = opt_time ? xb[nvar - 1] : 0.0;  // bounds [0, 5] (:215-218)
  __syncwarp();

  auto evaluate = [&](const V6& xx, double xdt, double& fo, V6& go, double& godt) {
    double gdt;
    eval_warp_fast2(g, dist, p, t, tc + b, n, mask, xx.v, opt_time ? xdt : knot_span, lane, fo, go.v, gdt);
    godt = opt_time ? gdt : 0.0;
  };
  auto store_best = [&](const V6& xx, double xdt) {
#pragma unroll
    for (int s = 0; s < 2; ++s) {
      const int i = 32 * s + lane;
      if (i < n) {
#pragma unroll
        for (int k = 0; k < 3; ++k) xb[3 * i + k] = xx.v[s][k];
      }
    }
    if (opt_time && lane == 0) xb[nvar - 1] = xdt;
  };

  double F, Gdt;
  V6 G;
  evaluate(X, Xdt, F, G, Gdt);
  int neval = 1;
  double best = F;
  store_best(X, Xdt);
  if (!(best == best)) best = 1.7976931348623157e308;  // a NaN start cannot be improved on by comparison

  const bool exact = (sp.flags & FUELGPU_SOLVE_EXACT_EVALS) != 0;
  int cnt = 0, head = 0;  // history ring: newest at (head-1) mod m
  double gamma_new = 1.0;
  double rho[LMAXM];  // rho[j] belongs to the j-th newest pair (static indices: stays in registers)
#pragma unroll
  for (int j = 0; j < LMAXM; ++j) rho[j] = 0.0;

  while (neval < sp.max_eval) {
    // projected gradient
    V6 PG, D;
    bool actv[2][3];
#pragma unroll
    for (int s = 0; s < 2; ++s)
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        const double xv = X.v[s][k], gv = G.v[s][k];
        actv[s][k] = (xv <= LB[BIDX(s, k)] && gv > 0.0) || (xv >= UB[BIDX(s, k)] && gv < 0.0);
        PG.v[s][k] = actv[s][k] ? 0.0 : gv;
      }
    const bool actv_dt = (Xdt <= 0.0 && Gdt > 0.0) || (Xdt >= 5.0 && Gdt < 0.0);
    const double PGdt = actv_dt ? 0.0 : Gdt;
    const double pgn2 = dot6(PG, PGdt, PG, PGdt, lane);
    if (!(pgn2 > 1e-24)) {
      if (!exact) break;
      while (neval < sp.max_eval) {  // benchmark mode: the objective is still evaluated max_eval times
        evaluate(X, Xdt, F, G, Gdt);
        ++neval;
      }
      break;
    }
    // two-loop recursion
    V6 Q = PG;
    double Qdt = PGdt;
    double alpha[LMAXM];
#pragma unroll
    for (int j = 0; j < LMAXM; ++j) {
      alpha[j] = 0.0;
      if (j < cnt) {
        int slot = head - 1 - j;  // j < cnt <= m: one wrap at most
        if (slot < 0) slot += m;
        V6 sv;
#pragma unroll
        for (int s = 0; s < 2; ++s)
#pragma unroll
          for (int k = 0; k < 3; ++k) sv.v[s][k] = S[HIDX2(slot, s, k)];
        alpha[j] = rho[j] * dot6(sv, Sdt[slot], Q, Qdt, lane);
#pragma unroll
        for (int s = 0; s < 2; ++s)
#pragma unroll
          for (int k = 0; k < 3; ++k) Q.v[s][k] -= alpha[j] * Y[HIDX2(slot, s, k)];
        Qdt -= alpha[j] * Ydt[slot];
      }
    }
    if (cnt > 0) {  // gamma = s.y / y.y of the newest pair
#pragma unroll
      for (int s = 0; s < 2; ++s)
#pragma unroll
        for (int k = 0; k < 3; ++k) Q.v[s][k] *= gamma_new;
      Qdt *= gamma_new;
    }
#pragma unroll
    for (int j = LMAXM - 1; j >= 0; --j) {
      if (j < cnt) {
        int slot = head - 1 - j;
        if (slot < 0) slot += m;
        V6 yv;
#pragma unroll
        for (int s = 0; s < 2; ++s)
#pragma unroll
          for (int k = 0; k < 3; ++k) yv.v[s][k] = Y[HIDX2(slot, s, k)];
        const double beta = rho[j] * dot6(yv, Ydt[slot], Q, Qdt, lane);
#pragma unroll
        for (int s = 0; s < 2; ++s)
#pragma unroll
          for (int k = 0; k < 3; ++k) Q.v[s][k] += S[HIDX2(slot, s, k)] * (alpha[j] - beta);
        Qdt += Sdt[slot] * (alpha[j] - beta);
      }
    }
#pragma unroll
    for (int s = 0; s < 2; ++s)
#pragma unroll
      for (int k = 0; k < 3; ++k) D.v[s][k] = actv[s][k] ? 0.0 : -Q.v[s][k];
    double Ddt = actv_dt ? 0.0 : -Qdt;
    double gd = dot6(G, Gdt, D, Ddt, lane);
    if (!(gd < 0.0)) {  // not a descent direction: restart from steepest descent
#pragma unroll
      for (int s = 0; s < 2; ++s)
#pragma unroll
        for (int k = 0; k < 3; ++k) D.v[s][k] = -PG.v[s][k];
      Ddt = -PGdt;
      gd = -pgn2;
      cnt = 0;
    }
    double step = cnt == 0 ? fmin(1.0, 1.0 / sqrt(pgn2)) : 1.0;

    // Armijo backtracking on the projected path
    bool accepted = false;
    V6 XN, GN;
    double XNdt = Xdt, GNdt = 0.0, FN = 0.0;
    while (neval < sp.max_eval) {
      bool clipped = false;
#pragma unroll
      for (int s = 0; s < 2; ++s)
#pragma unroll
        for (int k = 0; k < 3; ++k) {
          const double xt = X.v[s][k] + step * D.v[s][k], lo = LB[BIDX(s, k)], hi = UB[BIDX(s, k)];
          clipped = clipped || xt > hi || xt < lo;
          XN.v[s][k] = fmax(fmin(xt, hi), lo);
        }
      {
        const double xt = Xdt + step * Ddt;
        clipped = clipped || xt > 5.0 || xt < 0.0;
        XNdt = opt_time ? fmax(fmin(xt, 5.0), 0.0) : 0.0;
      }
      evaluate(XN, XNdt, FN, GN, GNdt);
      ++neval;
      if (FN < best) {  // costFunction :698-704
        best = FN;
        store_best(XN, XNdt);
      }
      double dec = step * gd;  // = G.(XN - X) as long as no component hit a bound
      if (__any_sync(0xffffffffu, clipped)) {
        V6 dx;
#pragma unroll
        for (int s = 0; s < 2; ++s)
#pragma unroll
          for (int k = 0; k < 3; ++k) dx.v[s][k] = XN.v[s][k] - X.v[s][k];
        dec = dot6(G, Gdt, dx, XNdt - Xdt, lane);
      }
      if (FN <= F + 1e-4 * dec) {
        accepted = true;
        break;
      }
      step *= 0.5;
      if (step < 1e-12) break;
    }
    if (!accepted) {
      if (!exact) break;
      cnt = 0;  // benchmark mode: drop the history and go on from steepest descent
      continue;
    }
    V6 sv, yv;
    bool small = true;
#pragma unroll
    for (int s = 0; s < 2; ++s)
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        sv.v[s][k] = XN.v[s][k] - X.v[s][k];
        yv.v[s][k] = GN.v[s][k] - G.v[s][k];
        small = small && (fabs(sv.v[s][k]) <= sp.xtol_rel * fabs(XN.v[s][k]));
      }
    const double sdt = XNdt - Xdt, ydt = GNdt - Gdt;
    small = small && (fabs(sdt) <= sp.xtol_rel * fabs(XNdt));
    const double sy = dot6(sv, sdt, yv, ydt, lane);
    const double ss = dot6(sv, sdt, sv, sdt, lane), yy = dot6(yv, ydt, yv, ydt, lane);
    if (sy > 1e-10 * sqrt(ss * yy)) {
      const int slot = head;
#pragma unroll
      for (int s = 0; s < 2; ++s)
#pragma unroll
        for (int k = 0; k < 3; ++k) {
          S[HIDX2(slot, s, k)] = (float)sv.v[s][k];
          Y[HIDX2(slot, s, k)] = (float)yv.v[s][k];
        }
      if (lane == 0) {
        Sdt[slot] = (float)sdt;
        Ydt[slot] = (float)ydt;
      }
      __syncwarp();
#pragma unroll
      for (int j = LMAXM - 1; j > 0; --j) rho[j] = rho[j - 1];
      rho[0] = 1.0 / sy;
      gamma_new = sy / yy;
      head = head + 1 == m ? 0 : head + 1;
      if (cnt < m) ++cnt;
    }
    X = XN;
    Xdt = XNdt;
    F = FN;
    G = GN;
    Gdt = GNdt;
    if (!exact && __all_sync(0xffffffffu, small)) break;  // xtol_rel, :173
  }
  if (lane == 0) neval_out[b] = neval;
}

int ensure_bs_grad(FuelMap* m, size_t bytes) {  // freed with the map (fuelgpu_map_destroy)
  if (bytes <= m->bs_grad_bytes) return 0;
  if (m->bs_grad) cudaFree(m->bs_grad);
  m->bs_grad = nullptr;
  m->bs_grad_bytes = 0;
  FUEL_CUDA(m, cudaMalloc(&m->bs_grad, bytes));
  m->bs_grad_bytes = bytes;
  return 0;
}

}  // namespace

// n_pts + dt > 32 lanes: the solver above, then min_cost_ at the returned best_variable_ from the faithful evaluator
// (bspline.cu, cost_batch_thread_kernel for these sizes) on the same stream, so that f_best is exactly what
// fuelgpu_bspline_cost_batch returns for that x.
int bspline_optimize_long_impl(FuelMap* m, int B, int n_pts, int mask, const FuelOptParams* p,
                               const FuelTrajConst* tc_dev, const FuelSolveParams* sp, double* x_dev,
                               double* fbest_dev, int32_t* neval_dev) {
  const int nvar = (mask & FUELGPU_MINTIME) ? 3 * n_pts + 1 : 3 * n_pts;
  int rc = ensure_bs_grad(m, sizeof(double) * (size_t)B * nvar);
  if (rc) return rc;
  const size_t smem = (size_t)LONG_WPB * LONG_SMEM_BYTES(sp->lbfgs_m);
  FUEL_CUDA(m, cudaFuncSetAttribute(optimize_long_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  optimize_long_kernel<<<(B + LONG_WPB - 1) / LONG_WPB, LONG_WPB * 32, smem, m->stream>>>(m->g, m->dist, *p, tc_dev, n_pts,
                                                                                     mask, B, *sp, x_dev, neval_dev);
  FUEL_LAUNCHES(m, 1);
  FUEL_CUDA(m, cudaGetLastError());
  return bspline_cost_batch_dev_impl(m, B, n_pts, mask & ~FUELGPU_COST_FAST_EVAL, p, tc_dev, x_dev, fbest_dev,
                                     (double*)m->bs_grad);
}
