// poly_traj.cu -- the head of FastPlannerManager::planExploreTraj (plan_manage/src/planner_manager.cpp:270-297) for a
// batch of tours, on the map's main stream: the segment times of :276-278, PolynomialTraj::waypointsTraj
// (poly_traj/src/polynomial_traj.cpp:5-175), getTotalTime / getLength (polynomial_traj.h:83-124), seg_num and dt
// (:285-288), and the samples and boundary derivatives handed to parameterizeToBspline (:292-297).
//
// The solve.  waypointsTraj minimizes the jerk integral over a piecewise quintic through the waypoints, with the start
// and end velocity / acceleration fixed.  Its free unknowns are (v_i, a_i) at the S - 1 inner waypoints; with each
// segment's cost written in its endpoint derivatives, d^T (A^-T Q A^-1) d, whose entries are integers
// (720, 360, 192, 168, 60, 36, 24, 9, 3) over powers of T, the normal equations are block tridiagonal with SPD 2x2
// diagonal blocks.  The reference forms the 6S x 6S matrices and takes three dense inverses; this file never forms them.
// Lane i builds node i's blocks, lane 0 factors the system once (block LDL^T, a 2x2 Cholesky per pivot), lanes 0..2
// substitute one axis each, and lane k maps segment k's endpoint derivatives back to its six monomial coefficients.
// The minimizer is unique, so the result agrees with the reference's to the conditioning of the problem (DESIGN.md 4.8).
//
// Built with -fmad=false.  Bit for bit the reference's fp64 arithmetic, because they come from the inputs by additions
// and comparisons only: getTotalTime (the times summed in order), dt = duration / seg_num, the sample grid (ts = 0,
// += dt while ts <= duration + 1e-4; getLength's eval_t = 0, += 0.01 while eval_t < total_t) and the segment search of
// PolynomialTraj::evaluate (while (times_[idx] + 1e-4 < ts) ts -= times_[idx++]; it may evaluate a segment up to 1e-4 s
// past its end).  Computed segment times are sqrt((dx*dx + dy*dy) + dz*dz) / (max_vel * 0.5); Eigen's order of that norm
// is unpinned.  Polynomial::evaluate uses pow() like the reference, whose libm it does not share: the length, samples
// and derivatives agree to rounding, and seg_num = (int)(length / ctrl_pt_dist) to within that rounding.
// One warp per trajectory; the waypoints, times, coefficients and the system sit in shared memory.
#include "common.cuh"

#include <math.h>

namespace {

constexpr int PT_WPB = 4;  // warps per CTA
constexpr int PT_MAXS = FUELGPU_MAX_WAYPTS - 1;
constexpr int PT_MAXK = FUELGPU_MAX_PTS - 2;
constexpr int PT_MAX_LEN_STEPS = (1 << 20) / 32;  // getLength: 2^20 samples (2.9 h of flight) at most
constexpr unsigned FULL = 0xffffffffu;

struct PolySmem {
  double P[FUELGPU_MAX_WAYPTS][3];  // waypoints
  double T[PT_MAXS];                // segment times
  double C[PT_MAXS][3][6];          // coefficients, cx[j] multiplies t^j
  double V[FUELGPU_MAX_WAYPTS][3];  // velocity at each waypoint
  double A[FUELGPU_MAX_WAYPTS][3];  // acceleration at each waypoint
  double D[PT_MAXS][3];             // node i's diagonal block (d00, d01, d11), then its Cholesky factor (l00, l10, l11)
  double L[PT_MAXS][4];             // node i's coupling to node i - 1 (rows v_i, a_i; columns v_i-1, a_i-1), then W_i
  double R[PT_MAXS][2][3];          // node i's right-hand side per axis, then the forward-substituted one
};

// PolynomialTraj::evaluate(t, k) (polynomial_traj.h:83-91) and the segment's Polynomial::evaluate (:35-45): tv[i] =
// getTBasis(t, i, k), then tv.dot(c) in written order per axis.  The reference does not bound idx; it cannot pass S - 1
// for the t the planner evaluates (t <= duration + 1e-4), and the bound keeps any other t inside the table.
__device__ __forceinline__ void traj_eval(const PolySmem& s, int S, double t, int k, double out[3]) {
  int idx = 0;
  double ts = t;
  while (idx < S - 1 && s.T[idx] + 1e-4 < ts) ts -= s.T[idx++];
  double tv[6];
#pragma unroll
  for (int i = 0; i < 6; ++i) {
    int coeff = 1;
    for (int j = i; j >= i - k + 1; --j) coeff *= j;
    tv[i] = i < k ? 0.0 : coeff * pow(ts, (double)(i - k));
  }
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    const double* c = s.C[idx][j];
    double v = tv[0] * c[0];
#pragma unroll
    for (int i = 1; i < 6; ++i) v = v + tv[i] * c[i];
    out[j] = v;
  }
}

__device__ __forceinline__ bool finite_pos(double v) { return v > 0.0 && v <= 1.7976931348623157e308; }

__global__ void __launch_bounds__(PT_WPB * 32) poly_waypoints_kernel(
    int B, int w_max, const int32_t* __restrict__ n_wp, const double* __restrict__ wp, const double* __restrict__ sv,
    const double* __restrict__ sa, const double* __restrict__ ev, const double* __restrict__ ea,
    const double* __restrict__ times, FuelPolyParams prm, FuelPolyInfo* __restrict__ info, double* __restrict__ coeffs,
    double* __restrict__ points, double* __restrict__ derivs) {
  __shared__ PolySmem smem[PT_WPB];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int b = blockIdx.x * PT_WPB + warp;
  if (b >= B) return;
  PolySmem& s = smem[warp];
  const int W = n_wp[b];
  const int S = W - 1;
  double* pts_b = points + (size_t)b * PT_MAXK * 3;
  double* der_b = derivs + (size_t)b * 12;
  double* cof_b = coeffs ? coeffs + (size_t)b * (w_max - 1) * 18 : nullptr;

  bool bad = W < 3 || W > FUELGPU_MAX_WAYPTS || W > w_max;
  if (!bad) {
    if (lane < W)
      for (int j = 0; j < 3; ++j) s.P[lane][j] = wp[((size_t)b * w_max + lane) * 3 + j];
    __syncwarp();
    bool ok = true;
    if (lane < S) {
      double t;
      if (times) {
        t = times[(size_t)b * (w_max - 1) + lane];
      } else {  // planner_manager.cpp:276-278
        const double dx = s.P[lane + 1][0] - s.P[lane][0], dy = s.P[lane + 1][1] - s.P[lane][1],
                     dz = s.P[lane + 1][2] - s.P[lane][2];
        t = sqrt((dx * dx + dy * dy) + dz * dz) / (prm.max_vel * 0.5);
      }
      s.T[lane] = t;
      ok = finite_pos(t);
    }
    bad = !__all_sync(FULL, ok);
  }
  if (bad) {  // FUELGPU_POLY_BAD_INPUT: NaN outputs, the other trajectories are unaffected
    const double nan = __longlong_as_double(0x7ff8000000000000ll);
    for (int e = lane; e < PT_MAXK * 3; e += 32) pts_b[e] = nan;
    if (lane < 12) der_b[lane] = nan;
    if (cof_b)
      for (int e = lane; e < (w_max - 1) * 18; e += 32) cof_b[e] = nan;
    if (lane == 0) {
      FuelPolyInfo r;
      r.duration = r.length = r.dt = nan;
      r.seg_num = r.n_pts = 0;
      r.status = FUELGPU_POLY_BAD_INPUT;
      r.reserved = 0;
      info[b] = r;
    }
    return;
  }

  // ---- the system: node i = lane + 1 (1..S-1), between segment L = i - 1 and segment R = i ----
  if (lane < S - 1) {
    const int i = lane + 1;
    const double iL = 1.0 / s.T[i - 1], iR = 1.0 / s.T[i];
    const double iL2 = iL * iL, iL3 = iL2 * iL, iL4 = iL3 * iL;
    const double iR2 = iR * iR, iR3 = iR2 * iR, iR4 = iR3 * iR;
    s.D[lane][0] = 192.0 * iL3 + 192.0 * iR3;
    s.D[lane][1] = 36.0 * iR2 - 36.0 * iL2;
    s.D[lane][2] = 9.0 * iL + 9.0 * iR;
    const double l00 = 168.0 * iL3, l01 = 24.0 * iL2, l10 = -24.0 * iL2, l11 = -3.0 * iL;
    s.L[lane][0] = l00, s.L[lane][1] = l01, s.L[lane][2] = l10, s.L[lane][3] = l11;
    for (int j = 0; j < 3; ++j) {
      const double dL = s.P[i][j] - s.P[i - 1][j], dR = s.P[i + 1][j] - s.P[i][j];
      double rv = 360.0 * dL * iL4 + 360.0 * dR * iR4;
      double ra = 60.0 * dR * iR3 - 60.0 * dL * iL3;
      if (i == 1) {  // the known start state moves to the right-hand side
        const double v0 = sv[(size_t)b * 3 + j], a0 = sa[(size_t)b * 3 + j];
        rv -= l00 * v0 + l01 * a0;
        ra -= l10 * v0 + l11 * a0;
      }
      if (i == S - 1) {  // and the known end state: node S's coupling is (168/T^3, -24/T^2; 24/T^2, -3/T)
        const double vS = ev ? ev[(size_t)b * 3 + j] : 0.0, aS = ea ? ea[(size_t)b * 3 + j] : 0.0;
        rv -= 168.0 * iR3 * vS - 24.0 * iR2 * aS;
        ra -= 24.0 * iR2 * vS - 3.0 * iR * aS;
      }
      s.R[lane][0][j] = rv;
      s.R[lane][1][j] = ra;
    }
  }
  if (lane < 3) {
    s.V[0][lane] = sv[(size_t)b * 3 + lane];
    s.A[0][lane] = sa[(size_t)b * 3 + lane];
    s.V[S][lane] = ev ? ev[(size_t)b * 3 + lane] : 0.0;
    s.A[S][lane] = ea ? ea[(size_t)b * 3 + lane] : 0.0;
  }
  __syncwarp();
  // block LDL^T, once for the three axes: D'_i = D_i - W_i U_i-1 with W_i = L_i D'_i-1^-1 and U_i-1 = L_i^T;
  // D'_i is kept as its 2x2 Cholesky factor, L_i is overwritten by W_i
  if (lane == 0) {
    for (int n = 0; n < S - 1; ++n) {
      double d00 = s.D[n][0], d01 = s.D[n][1], d11 = s.D[n][2];
      if (n > 0) {
        const double c00 = s.D[n - 1][0], c10 = s.D[n - 1][1], c11 = s.D[n - 1][2];
        // inverse of D'_n-1 = C C^T: (C^-T C^-1)
        const double i00 = 1.0 / c00, i11 = 1.0 / c11, i10 = -c10 * i00 * i11;  // C^-1 (lower)
        const double m00 = i00 * i00 + i10 * i10, m01 = i10 * i11, m11 = i11 * i11;
        const double l00 = s.L[n][0], l01 = s.L[n][1], l10 = s.L[n][2], l11 = s.L[n][3];
        const double w00 = l00 * m00 + l01 * m01, w01 = l00 * m01 + l01 * m11;
        const double w10 = l10 * m00 + l11 * m01, w11 = l10 * m01 + l11 * m11;
        d00 -= w00 * l00 + w01 * l01;  // W L^T
        d01 -= w00 * l10 + w01 * l11;
        d11 -= w10 * l10 + w11 * l11;
        s.L[n][0] = w00, s.L[n][1] = w01, s.L[n][2] = w10, s.L[n][3] = w11;
      }
      const double c00 = sqrt(d00), c10 = d01 / c00;
      s.D[n][0] = c00, s.D[n][1] = c10, s.D[n][2] = sqrt(d11 - c10 * c10);
    }
  }
  __syncwarp();
  if (lane < 3) {  // one axis per lane: forward, then back substitution
    const int j = lane;
    for (int n = 1; n < S - 1; ++n) {
      const double r0 = s.R[n - 1][0][j], r1 = s.R[n - 1][1][j];
      s.R[n][0][j] -= s.L[n][0] * r0 + s.L[n][1] * r1;
      s.R[n][1][j] -= s.L[n][2] * r0 + s.L[n][3] * r1;
    }
    double u0 = 0.0, u1 = 0.0;  // u_n+1
    for (int n = S - 2; n >= 0; --n) {
      double r0 = s.R[n][0][j], r1 = s.R[n][1][j];
      if (n < S - 2) {  // U_n u_n+1 with U_n = L_n+1^T (the original coupling: rebuild it from the times)
        const double iT = 1.0 / s.T[n + 1], iT2 = iT * iT;
        r0 -= 168.0 * iT2 * iT * u0 - 24.0 * iT2 * u1;
        r1 -= 24.0 * iT2 * u0 - 3.0 * iT * u1;
      }
      const double c00 = s.D[n][0], c10 = s.D[n][1], c11 = s.D[n][2];
      const double y0 = r0 / c00, y1 = (r1 - c10 * y0) / c11;  // C y = r, C^T u = y
      u1 = y1 / c11;
      u0 = (y0 - c10 * u1) / c00;
      s.V[n + 1][j] = u0;
      s.A[n + 1][j] = u1;
    }
  }
  __syncwarp();
  if (lane < S) {  // segment k's coefficients from its endpoint derivatives (A_k^-1 in closed form)
    const int k = lane;
    const double iT = 1.0 / s.T[k], iT2 = iT * iT, iT3 = iT2 * iT, iT4 = iT3 * iT, iT5 = iT4 * iT;
    for (int j = 0; j < 3; ++j) {
      const double d = s.P[k + 1][j] - s.P[k][j];
      const double v0 = s.V[k][j], v1 = s.V[k + 1][j], a0 = s.A[k][j], a1 = s.A[k + 1][j];
      double* c = s.C[k][j];
      c[0] = s.P[k][j];
      c[1] = v0;
      c[2] = 0.5 * a0;
      c[3] = 10.0 * d * iT3 - (6.0 * v0 + 4.0 * v1) * iT2 - (1.5 * a0 - 0.5 * a1) * iT;
      c[4] = (8.0 * v0 + 7.0 * v1) * iT3 - 15.0 * d * iT4 + (1.5 * a0 - a1) * iT2;
      c[5] = 6.0 * d * iT5 - 3.0 * (v0 + v1) * iT4 - 0.5 * (a0 - a1) * iT3;
    }
  }
  __syncwarp();
  if (cof_b) {
    for (int e = lane; e < (w_max - 1) * 18; e += 32) cof_b[e] = e < S * 18 ? (&s.C[0][0][0])[e] : 0.0;
  }

  // ---- getTotalTime: the times summed in order ----
  double duration = 0.0;
  for (int k = 0; k < S; ++k) duration += s.T[k];

  // ---- getLength: samples at eval_t = 0, 0.01, ... (running sum) while eval_t < total_t, 32 per step ----
  double length = 0.0, e_base = 0.0, prev[3] = {0.0, 0.0, 0.0};
  for (int step = 0; step < PT_MAX_LEN_STEPS; ++step) {
    double e = e_base, mine = 0.0;
#pragma unroll
    for (int i = 0; i < 32; ++i) {
      mine = i == lane ? e : mine;
      e = e + 0.01;
    }
    const bool in = mine < duration;
    double p[3] = {0.0, 0.0, 0.0};
    if (in) traj_eval(s, S, mine, 0, p);
    double q[3], nrm = 0.0;
    for (int j = 0; j < 3; ++j) {
      q[j] = __shfl_up_sync(FULL, p[j], 1);
      if (lane == 0) q[j] = prev[j];
    }
    const bool first = step == 0 && lane == 0;
    if (in && !first) {
      const double dx = p[0] - q[0], dy = p[1] - q[1], dz = p[2] - q[2];
      nrm = sqrt((dx * dx + dy * dy) + dz * dz);
    }
    const unsigned bal = __ballot_sync(FULL, in);
    for (int i = 0; i < 32; ++i) {  // length_ += |p_cur - p_prev| in the reference's order
      const double v = __shfl_sync(FULL, nrm, i);
      if (((bal >> i) & 1u) && !(step == 0 && i == 0)) length += v;
    }
    if (bal != FULL) break;
    for (int j = 0; j < 3; ++j) prev[j] = __shfl_sync(FULL, p[j], 31);
    e_base = e;
  }

  // ---- planExploreTraj :285-288 ----
  const int sn = (int)(length / prm.ctrl_pt_dist);
  const int seg_num = sn > prm.min_seg_num ? sn : prm.min_seg_num;
  const double dt = duration / (double)seg_num;
  const double lim = duration + 1e-4;

  // ---- the samples: ts = 0, += dt while ts <= duration + 1e-4 (:292-293) ----
  int K = 0;
  double t_base = 0.0;
  for (int step = 0; step < PT_MAX_LEN_STEPS; ++step) {
    double e = t_base, mine = 0.0;
#pragma unroll
    for (int i = 0; i < 32; ++i) {
      mine = i == lane ? e : mine;
      e = e + dt;
    }
    const bool in = mine <= lim;
    const int idx = step * 32 + lane;
    if (in && idx < PT_MAXK) {
      double p[3];
      traj_eval(s, S, mine, 0, p);
      for (int j = 0; j < 3; ++j) pts_b[idx * 3 + j] = p[j];
    }
    const unsigned bal = __ballot_sync(FULL, in);
    K += __popc(bal);
    if (bal != FULL) break;
    t_base = e;
  }
  const int status = K + 2 > FUELGPU_MAX_PTS ? FUELGPU_POLY_TOO_LONG : 0;
  if (status) {  // no samples
    for (int e = lane; e < PT_MAXK * 3; e += 32) pts_b[e] = 0.0;
  } else {
    for (int e = K * 3 + lane; e < PT_MAXK * 3; e += 32) pts_b[e] = 0.0;
  }
  // boundary_deri (:294-297): evaluate(0, 1), evaluate(duration, 1), evaluate(0, 2), evaluate(duration, 2)
  if (lane < 4) {
    double d[3];
    traj_eval(s, S, (lane & 1) ? duration : 0.0, 1 + (lane >> 1), d);
    for (int j = 0; j < 3; ++j) der_b[lane * 3 + j] = d[j];
  }
  if (lane == 0) {
    FuelPolyInfo r;
    r.duration = duration;
    r.length = length;
    r.dt = dt;
    r.seg_num = seg_num;
    r.n_pts = K + 2;
    r.status = status;
    r.reserved = 0;
    info[b] = r;
  }
}

}  // namespace

int poly_waypoints_impl(FuelMap* m, int B, int w_max, const int32_t* n_wp_dev, const double* wp_dev,
                        const double* sv_dev, const double* sa_dev, const double* ev_dev, const double* ea_dev,
                        const double* times_dev, const FuelPolyParams* p, FuelPolyInfo* info_dev, double* coeffs_dev,
                        double* points_dev, double* derivs_dev) {
  if (B == 0) return 0;
  const int grid = (B + PT_WPB - 1) / PT_WPB;
  poly_waypoints_kernel<<<grid, PT_WPB * 32, 0, m->stream>>>(B, w_max, n_wp_dev, wp_dev, sv_dev, sa_dev, ev_dev, ea_dev,
                                                              times_dev, *p, info_dev, coeffs_dev, points_dev,
                                                              derivs_dev);
  FUEL_CUDA(m, cudaGetLastError());
  FUEL_LAUNCHES(m, 1);
  return 0;
}
