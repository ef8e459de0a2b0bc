// traj_check.cu -- verdicts on a batch of uniform cubic B-splines, on the map's main stream behind the solver:
// NonUniformBspline::evaluateDeBoorT / getDerivative / getTimeSum / getJerk / checkFeasibility / checkRatio
// (bspline/src/non_uniform_bspline.cpp), FastPlannerManager::checkTrajCollision (planner_manager.cpp:96-118) and
// selectBestTraj (:476-482); and, ahead of the solver, parameterizeToBspline (:178-265) with the boundary states and
// pt_dist_ that BsplineOptimizer::optimize() freezes from its result.
//
// Built with -fmad=false: every output equals the reference's fp64 arithmetic bit for bit (for the parameterization:
// given the control points it returns; their least-squares solve is this file's own, see traj_param_kernel).
//  - knots are the running sum of setUniformBspline (:16-32), u[i] = u[i-1] + dt, not i*dt;
//  - derivative control points are (p * (P[i+1] - P[i])) / (u[i+p+1] - u[i+1]) per element (:77-86), the derivative
//    spline keeps the parent's knots minus the first and last (:97-106);
//  - getJerk sums (dt_i * c) * c sequentially, i outer, axis inner (:283-298);
//  - the collision scan's fut_t is the running sum 0.02, 0.04, ... of the reference's loop; a warp evaluates 32
//    samples at a time and a ballot finds the first one at which the sequential loop stops.
// One warp per trajectory; its control points, knots and derivative control points sit in shared memory.
#include "common.cuh"

namespace {

constexpr int TC_WPB = 4;                       // warps per CTA
constexpr int TC_KNOTS = FUELGPU_MAX_PTS + 4;   // knots of a cubic with n_pts control points
constexpr unsigned FULL = 0xffffffffu;

struct SplineSmem {
  double P[FUELGPU_MAX_PTS][3];  // control points
  double Q[FUELGPU_MAX_PTS][3];  // getDerivative() control points (n - 1)
  double R[FUELGPU_MAX_PTS][3];  // getDerivative().getDerivative() control points (n - 2)
  double U[TC_KNOTS];            // knots u_[0..n+3]
  double J[FUELGPU_MAX_PTS][3];  // getJerk's terms (n - 3 rows)
};

// The spline of warp `b`: control points from x [B][nvar] (dt in x[b][3n] when nvar == 3n + 1, else dt[b]), the
// knot vector, and the control points of the first and second derivative.
__device__ void load_spline(SplineSmem& s, int b, int n, int nvar, const double* __restrict__ x,
                            const double* __restrict__ dtv, int lane) {
  const double* xb = x + (size_t)b * nvar;
  for (int e = lane; e < 3 * n; e += 32) s.P[e / 3][e % 3] = xb[e];
  if (lane == 0) {
    const double dt = nvar == 3 * n + 1 ? xb[3 * n] : dtv[b];
    const int m = n + 3;  // m_ = n_ + p_ + 1 with n_ = n - 1
    for (int i = 0; i <= m; ++i) s.U[i] = i <= 3 ? (double)(-3 + i) * dt : s.U[i - 1] + dt;
  }
  __syncwarp();
  for (int e = lane; e < 3 * (n - 1); e += 32) {
    const int i = e / 3, j = e % 3;
    s.Q[i][j] = (3.0 * (s.P[i + 1][j] - s.P[i][j])) / (s.U[i + 4] - s.U[i + 1]);
  }
  __syncwarp();
  for (int e = lane; e < 3 * (n - 2); e += 32) {  // derivative knots u'[k] = u[k + 1], p' = 2
    const int i = e / 3, j = e % 3;
    s.R[i][j] = (2.0 * (s.Q[i + 1][j] - s.Q[i][j])) / (s.U[i + 4] - s.U[i + 2]);
  }
  __syncwarp();
}

// evaluateDeBoor (:51-71) of a degree-p spline with nc control points C and knots Uk (m = nc + p), at u; the knot
// search starts at *k (>= p), which is exact whenever every knot below it is < the clamped u, and returns its stop.
template <int p>
__device__ __forceinline__ void deboor(const double (*C)[3], const double* Uk, int nc, double u, int* kio,
                                       double out[3]) {
  const int m = nc + p;
  const double lo = Uk[p], hi = Uk[m - p];
  double ub = lo < u ? u : lo;  // std::max(u_(p_), u)
  ub = hi < ub ? hi : ub;       // std::min(.., u_(m_ - p_))
  int k = *kio;
  while (k < m - p - 1 && Uk[k + 1] < ub) ++k;
  *kio = k;
  double d[p + 1][3];
#pragma unroll
  for (int i = 0; i <= p; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) d[i][j] = C[k - p + i][j];
#pragma unroll
  for (int r = 1; r <= p; ++r)
#pragma unroll
    for (int i = p; i >= r; --i) {
      const double alpha = (ub - Uk[i + k - p]) / (Uk[i + 1 + k - r] - Uk[i + k - p]);
#pragma unroll
      for (int j = 0; j < 3; ++j) d[i][j] = (1 - alpha) * d[i - 1][j] + alpha * d[i][j];
    }
#pragma unroll
  for (int j = 0; j < 3; ++j) out[j] = d[p][j];
}

// SDFMap::getInflateOccupancy(pos) == 1 (sdf_map.h:217-226): posToIndex then isInMap(idx); outside the map is -1,
// not a hit.  Comparing the floored doubles with [0, n-1] is the int conversion plus the bounds test of the
// reference for every value (an out-of-range or NaN conversion lands outside the map on x86-64 as well).
__device__ __forceinline__ bool inflate_hit(const Geom& g, const uint8_t* __restrict__ occ, const double pt[3]) {
  const double fx = floor((pt[0] - g.origin[0]) * g.res_inv);
  const double fy = floor((pt[1] - g.origin[1]) * g.res_inv);
  const double fz = floor((pt[2] - g.origin[2]) * g.res_inv);
  if (!(fx >= 0.0 && fy >= 0.0 && fz >= 0.0 && fx <= g.nx - 1 && fy <= g.ny - 1 && fz <= g.nz - 1)) return false;
  return (__ldg(occ + addr_of(g, (int)fx, (int)fy, (int)fz)) & 4) != 0;
}

__device__ __forceinline__ double warp_max_ref(double v) {  // std::max reduction of non-NaN partials
#pragma unroll
  for (int o = 16; o; o >>= 1) {
    const double w = __shfl_xor_sync(FULL, v, o);
    v = v < w ? w : v;
  }
  return v;
}

__global__ void __launch_bounds__(TC_WPB * 32) traj_check_kernel(Geom g, const uint8_t* __restrict__ occ, int B, int n,
                                                                 int nvar, const double* __restrict__ x,
                                                                 const double* __restrict__ dtv, FuelTrajCheckParams prm,
                                                                 FuelTrajReport* __restrict__ rep) {
  __shared__ SplineSmem sm[TC_WPB];
  const int lane = threadIdx.x & 31;
  const int b = blockIdx.x * TC_WPB + (threadIdx.x >> 5);
  if (b >= B) return;
  SplineSmem& s = sm[threadIdx.x >> 5];
  load_spline(s, b, n, nvar, x, dtv, lane);

  // checkRatio / checkFeasibility (:135-160, :443-487): the velocity rows are the derivative control points
  const double lim_v = prm.max_vel + 1e-4, lim_a = prm.max_acc + 1e-4;
  double mv = -1.0, ma = -1.0;
  bool fea = true;
  for (int e = lane; e < 3 * (n - 1); e += 32) {
    const double v = fabs(s.Q[e / 3][e % 3]);
    fea = fea && !(v > lim_v);
    mv = mv < v ? v : mv;
  }
  for (int e = lane; e < 3 * (n - 2); e += 32) {
    const int i = e / 3, j = e % 3;
    const double a = (6.0 * ((s.P[i + 2][j] - s.P[i + 1][j]) / (s.U[i + 5] - s.U[i + 2]) -
                             (s.P[i + 1][j] - s.P[i][j]) / (s.U[i + 4] - s.U[i + 1]))) /
                     (s.U[i + 4] - s.U[i + 2]);
    const double v = fabs(a);
    fea = fea && !(v > lim_a);
    ma = ma < v ? v : ma;
  }
  // getJerk's terms: third-derivative control points (knots u''[k] = u[k + 2], p'' = 1) times their knot interval
  for (int e = lane; e < 3 * (n - 3); e += 32) {
    const int i = e / 3, j = e % 3;
    const double w = s.U[i + 4] - s.U[i + 3];
    const double c = (1.0 * (s.R[i + 1][j] - s.R[i][j])) / w;
    s.J[i][j] = w * c * c;
  }
  mv = warp_max_ref(mv);
  ma = warp_max_ref(ma);
  fea = __all_sync(FULL, fea);
  __syncwarp();

  // checkTrajCollision's loop (planner_manager.cpp:96-118), 32 samples per step
  const double duration = s.U[n] - s.U[3];
  const double t_now = prm.t_now;
  double cur[3];
  int k0 = 3;
  deboor<3>(s.P, s.U, n, t_now + s.U[3], &k0, cur);
  int kstart = 3;
  double ft_base = 0.0, r_carry = 0.0;  // fut_t of the sample before this step (0 + 0.02 = 0.02 exactly), its radius
  int n_checked = 0, safe = 1;
  double distance = -1.0;
  for (int base = 0;; base += 32) {
    double ft = ft_base, mine = 0.0;
#pragma unroll
    for (int i = 0; i < 32; ++i) {
      ft = ft + 0.02;
      mine = i == lane ? ft : mine;
    }
    const double ts = t_now + mine;
    const bool in_time = ts < duration;
    bool hit = false;
    double radius = 0.0;
    int k = kstart;
    if (in_time) {
      double pt[3];
      deboor<3>(s.P, s.U, n, ts + s.U[3], &k, pt);
      hit = inflate_hit(g, occ, pt);
      const double dx = pt[0] - cur[0], dy = pt[1] - cur[1], dz = pt[2] - cur[2];
      radius = sqrt(dx * dx + dy * dy + dz * dz);
    }
    const bool stop = !in_time || hit || !(radius < 6.0);
    const unsigned bal = __ballot_sync(FULL, stop);
    double r_prev = __shfl_up_sync(FULL, radius, 1);
    if (lane == 0) r_prev = r_carry;
    if (bal) {
      const int f = __ffs(bal) - 1;
      const bool f_in = __shfl_sync(FULL, in_time, f), f_hit = __shfl_sync(FULL, hit, f);
      const double f_rprev = __shfl_sync(FULL, r_prev, f);
      n_checked = base + f + (f_in ? 1 : 0);
      if (f_in && f_hit) {
        safe = 0;
        distance = f_rprev;
      }
      break;
    }
    if (base + 32 >= FUELGPU_CHECK_MAX_SAMPLES) {  // a scan the reference would not finish in practice
      n_checked = base + 32;
      break;
    }
    ft_base = ft;
    r_carry = __shfl_sync(FULL, radius, 31);
    kstart = __shfl_sync(FULL, k, 31);
  }

  if (lane == 0) {
    double jerk = 0.0;
    for (int i = 0; i < n - 3; ++i)
      for (int j = 0; j < 3; ++j) jerk += s.J[i][j];
    const double vr = mv / prm.max_vel, ar = sqrt(fabs(ma) / prm.max_acc);
    FuelTrajReport r;
    r.duration = duration;
    r.jerk = jerk;
    r.ratio = vr < ar ? ar : vr;  // std::max(max_vel / limit_vel_, sqrt(fabs(max_acc) / limit_acc_))
    r.distance = distance;
    r.safe = safe;
    r.feasible = fea ? 1 : 0;
    r.n_checked = n_checked;
    r.reserved = 0;
    rep[b] = r;
  }
}

// selectBestTraj: least jerk, lowest index on ties, NaN never wins; [1] the same among safe && feasible
__device__ __forceinline__ bool better(double j, int i, double jc, int ic) {
  return i >= 0 && (ic < 0 || j < jc || (j == jc && i < ic));
}

__global__ void __launch_bounds__(1024) traj_best_kernel(const FuelTrajReport* __restrict__ rep, int B, int32_t* best) {
  __shared__ double sj[2][32];
  __shared__ int si[2][32];
  double j0 = 0.0, j1 = 0.0;
  int i0 = -1, i1 = -1;
  for (int b = threadIdx.x; b < B; b += blockDim.x) {
    const FuelTrajReport r = rep[b];
    if (isnan(r.jerk)) continue;
    if (better(r.jerk, b, j0, i0)) j0 = r.jerk, i0 = b;
    if (r.safe && r.feasible && better(r.jerk, b, j1, i1)) j1 = r.jerk, i1 = b;
  }
#pragma unroll
  for (int o = 16; o; o >>= 1) {
    const double a0 = __shfl_xor_sync(FULL, j0, o), a1 = __shfl_xor_sync(FULL, j1, o);
    const int b0 = __shfl_xor_sync(FULL, i0, o), b1 = __shfl_xor_sync(FULL, i1, o);
    if (better(a0, b0, j0, i0)) j0 = a0, i0 = b0;
    if (better(a1, b1, j1, i1)) j1 = a1, i1 = b1;
  }
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  if (lane == 0) sj[0][w] = j0, si[0][w] = i0, sj[1][w] = j1, si[1][w] = i1;
  __syncthreads();
  if (w == 0) {
    j0 = lane < nw ? sj[0][lane] : 0.0, i0 = lane < nw ? si[0][lane] : -1;
    j1 = lane < nw ? sj[1][lane] : 0.0, i1 = lane < nw ? si[1][lane] : -1;
#pragma unroll
    for (int o = 16; o; o >>= 1) {
      const double a0 = __shfl_xor_sync(FULL, j0, o), a1 = __shfl_xor_sync(FULL, j1, o);
      const int b0 = __shfl_xor_sync(FULL, i0, o), b1 = __shfl_xor_sync(FULL, i1, o);
      if (better(a0, b0, j0, i0)) j0 = a0, i0 = b0;
      if (better(a1, b1, j1, i1)) j1 = a1, i1 = b1;
    }
    if (lane == 0) best[0] = i0, best[1] = i1;
  }
}

// evaluateDeBoorT (:73-75) of the spline or of its first / second derivative at t [B][n_t] -> out [B][n_t][3]
__global__ void __launch_bounds__(TC_WPB * 32) traj_evaluate_kernel(int B, int n, int nvar, const double* __restrict__ x,
                                                                    const double* __restrict__ dtv, int n_t,
                                                                    const double* __restrict__ t, int deriv,
                                                                    double* __restrict__ out) {
  __shared__ SplineSmem sm[TC_WPB];
  const int lane = threadIdx.x & 31;
  const int b = blockIdx.x * TC_WPB + (threadIdx.x >> 5);
  if (b >= B) return;
  SplineSmem& s = sm[threadIdx.x >> 5];
  load_spline(s, b, n, nvar, x, dtv, lane);
  for (int q = lane; q < n_t; q += 32) {
    const size_t o = (size_t)b * n_t + q;
    const double tq = t[o];
    double v[3];
    int k;
    if (deriv == 0) {
      k = 3;
      deboor<3>(s.P, s.U, n, tq + s.U[3], &k, v);
    } else if (deriv == 1) {
      k = 2;
      deboor<2>(s.Q, s.U + 1, n - 1, tq + s.U[3], &k, v);
    } else {
      k = 1;
      deboor<1>(s.R, s.U + 2, n - 2, tq + s.U[3], &k, v);
    }
    out[3 * o] = v[0], out[3 * o + 1] = v[1], out[3 * o + 2] = v[2];
  }
}

// ---- parameterizeToBspline (:178-265), degree 3, and what optimize() freezes from its control points ------------------
struct ParamSmem {
  SplineSmem s;
  double Rb[FUELGPU_MAX_PTS][3];  // band of the triangular factor: Rb[i][k] = R(i, i + k)
  double D[FUELGPU_MAX_PTS][3];   // Q^T b per axis, rows of R
  double seg[FUELGPU_MAX_PTS];    // |P[i+1] - P[i]| for pt_dist_
};

// Row r of the system in column order (start vel, start acc, positions 0..K-1, end vel, end acc): its first column and
// its three coefficients, with the reference's entries (1/6.0)*(1,4,1), (1/(2*ts))*(-1,0,1), (1/(ts*ts))*(1,-2,1).
__device__ __forceinline__ int param_row(int r, int K, double ts, const double* __restrict__ pts,
                                         const double* __restrict__ der, double w[3], double e[3]) {
  const double to_pos = 1 / 6.0, to_vel = 1 / (2 * ts), to_acc = 1 / (ts * ts);
  int c, src;  // src: index into der (0 start vel, 1 end vel, 2 start acc, 3 end acc), or -1 for a position
  if (r == 0) c = 0, src = 0;
  else if (r == 1) c = 0, src = 2;
  else if (r < K + 2) c = r - 2, src = -1;
  else c = K - 1, src = r == K + 2 ? 1 : 3;
  if (src < 0) {
    w[0] = to_pos * 1, w[1] = to_pos * 4, w[2] = to_pos * 1;
  } else if (src == 0 || src == 1) {
    w[0] = to_vel * -1, w[1] = to_vel * 0, w[2] = to_vel * 1;
  } else {
    w[0] = to_acc * 1, w[1] = to_acc * -2, w[2] = to_acc * 1;
  }
  const double* bsrc = src < 0 ? pts + 3 * c : der + 3 * src;
#pragma unroll
  for (int a = 0; a < 3; ++a) e[a] = bsrc[a];
  return c;
}

// One warp per trajectory.  Lane 0 solves the (K+4) x (K+2) least-squares system with Givens rotations, row by row in
// column order, so that the triangular factor keeps the band of A (three entries per row); the three axes share the
// rotations.  The warp then loads the returned spline with load_spline and evaluates getBoundaryStates(2, 0) with the
// check kernels' deboor, and sums pt_dist_ in the reference's order.  A knot span that is not finite and positive
// gives NaN in every output of its trajectory.
__global__ void __launch_bounds__(TC_WPB * 32) traj_param_kernel(int B, int n, int nvar, const double* __restrict__ pts,
                                                                 const double* __restrict__ der,
                                                                 const double* __restrict__ dtv,
                                                                 const double* __restrict__ tlb, double* x,
                                                                 FuelTrajConst* __restrict__ tc) {
  __shared__ ParamSmem sm[TC_WPB];
  const int lane = threadIdx.x & 31;
  const int b = blockIdx.x * TC_WPB + (threadIdx.x >> 5);
  if (b >= B) return;
  ParamSmem& q = sm[threadIdx.x >> 5];
  const int K = n - 2;
  const double raw = dtv[b];
  const double dt = isfinite(raw) && raw > 0.0 ? raw : __longlong_as_double(0x7ff8000000000000ll);
  double* xb = x + (size_t)b * nvar;

  if (lane == 0) {
    const double* pb = pts + (size_t)b * K * 3;
    const double* db = der + (size_t)b * 12;
    int nfill = 0;  // rows of R filled so far: rows arrive in column order, so R fills top down
    for (int r = 0; r < K + 4; ++r) {
      double w[3], e[3];
      const int c = param_row(r, K, dt, pb, db, w, e);
      for (int j = c; j < c + 3; ++j) {
        if (j == nfill) {
#pragma unroll
          for (int k = 0; k < 3; ++k) q.Rb[j][k] = w[k], q.D[j][k] = e[k];
          ++nfill;
          break;
        }
        // the rotation that zeroes w[0] against R(j, j); one reciprocal square root instead of a square root and two
        // divisions on the dependent chain (it rounds the rotation by a few ulp, far below the solve's cond(A) * eps)
        const double rj = q.Rb[j][0], hh = rj * rj + w[0] * w[0];
        const double inv = hh != 0.0 ? rsqrt(hh) : 0.0;
        const double h = hh * inv;
        const double cs = hh != 0.0 ? rj * inv : 1.0, sn = w[0] * inv;
        const double r1 = q.Rb[j][1], r2 = q.Rb[j][2];
        q.Rb[j][0] = h;
        q.Rb[j][1] = cs * r1 + sn * w[1];
        q.Rb[j][2] = cs * r2 + sn * w[2];
        w[0] = cs * w[1] - sn * r1;
        w[1] = cs * w[2] - sn * r2;
        w[2] = 0.0;
#pragma unroll
        for (int a = 0; a < 3; ++a) {
          const double dj = q.D[j][a];
          q.D[j][a] = cs * dj + sn * e[a];
          e[a] = cs * e[a] - sn * dj;
        }
      }
    }
    double x1[3] = {0.0, 0.0, 0.0}, x2[3] = {0.0, 0.0, 0.0};  // solution rows i + 1, i + 2
    for (int i = n - 1; i >= 0; --i) {
#pragma unroll
      for (int a = 0; a < 3; ++a) {
        const double v = (q.D[i][a] - q.Rb[i][1] * x1[a] - q.Rb[i][2] * x2[a]) / q.Rb[i][0];
        xb[3 * i + a] = v;
        x2[a] = x1[a];
        x1[a] = v;
      }
    }
    if (nvar == 3 * n + 1) xb[3 * n] = dt;
  }
  __syncwarp();
  // setUniformBspline(ctrl, 3, dt) of the returned control points; with nvar == 3n, dt comes from the input array
  load_spline(q.s, b, n, nvar, x, dtv, lane);
  SplineSmem& s = q.s;
  for (int i = lane; i < n - 1; i += 32) {
    const double a0 = s.P[i + 1][0] - s.P[i][0], a1 = s.P[i + 1][1] - s.P[i][1], a2 = s.P[i + 1][2] - s.P[i][2];
    q.seg[i] = sqrt(a0 * a0 + a1 * a1 + a2 * a2);
  }
  FuelTrajConst* t = tc + b;
  uint64_t* tw = reinterpret_cast<uint64_t*>(t);
  for (int i = lane; i < (int)(sizeof(FuelTrajConst) / 8); i += 32) tw[i] = 0;
  __syncwarp();
  // getBoundaryStates(2, 0) (:108-123): pos, vel, acc at t = 0 on lanes 0-2, the end position at getTimeSum() on lane 3
  double v[3];
  int k;
  if (lane == 0) {
    k = 3;
    deboor<3>(s.P, s.U, n, 0.0 + s.U[3], &k, v);
  } else if (lane == 1) {
    k = 2;
    deboor<2>(s.Q, s.U + 1, n - 1, 0.0 + s.U[3], &k, v);
  } else if (lane == 2) {
    k = 1;
    deboor<1>(s.R, s.U + 2, n - 2, 0.0 + s.U[3], &k, v);
  } else if (lane == 3) {
    k = 3;
    deboor<3>(s.P, s.U, n, (s.U[n] - s.U[3]) + s.U[3], &k, v);
  }
  if (lane < 3) {
    for (int a = 0; a < 3; ++a) t->start[lane][a] = v[a];
  } else if (lane == 3) {
    for (int a = 0; a < 3; ++a) t->end[0][a] = v[a];
  }
  if (lane == 0) {
    double d = 0.0;  // pt_dist_ (bspline_optimizer.cpp:136-140): sequential sum over the segments, over the point count
    for (int i = 0; i < n - 1; ++i) d += q.seg[i];
    t->pt_dist = d / (double)n;
    t->knot_span = dt;
    t->n_end = 1;
    t->time_lb = tlb ? tlb[b] : -1.0;
    t->view_idx = -1;
  }
}

// ---- planYawExplore (planner_manager.cpp:774-865) with lookfwd, on each trajectory of the batch -----------------------
constexpr int YS = FUELGPU_YAW_SEG_NUM, YP = FUELGPU_YAW_PTS, YW = FUELGPU_YAW_MAX_WAYPT;
constexpr double YAW_PI = 3.141592653589793;  // M_PI

struct YawSmem {
  SplineSmem s;
  double wp[YW];     // atan2 of look-ahead difference i + 1 (NaN where |pd| <= 1e-6), then waypoint i + 1
  double Hb[YP][4];  // normal equations, Hb[i][d] = H(i, i - d); the Cholesky factor in place
  double r[YP];      // right-hand side, then the solution
};

// calcNextYaw (:867-885)
__device__ __forceinline__ double next_yaw(double last_yaw, double yaw) {
  double round_last = last_yaw;
  while (round_last < -YAW_PI) round_last += 2 * YAW_PI;
  while (round_last > YAW_PI) round_last -= 2 * YAW_PI;
  const double diff = yaw - round_last;
  if (fabs(diff) <= YAW_PI) return last_yaw + diff;
  if (diff > YAW_PI) return last_yaw + diff - 2 * YAW_PI;
  return last_yaw + diff + 2 * YAW_PI;
}

// w * (a . q - t)^2 over control points o .. o + L - 1, added to H (band Hb[i][d] = H(i, i - d)) and r (the objective's
// Hessian and gradient at 0, both halved)
template <int L>
__device__ __forceinline__ void yaw_term(double (*Hb)[4], double* r, int o, const double (&a)[L], double w, double t) {
#pragma unroll
  for (int u = 0; u < L; ++u) {
#pragma unroll
    for (int v = 0; v <= u; ++v) Hb[o + u][u - v] += (w * a[u]) * a[v];
    r[o + u] += (w * a[u]) * t;
  }
}

// H q = r for the n x n band of half-bandwidth 3 in Hb: banded Cholesky H = L L^T in place (L(i, k) in Hb[i][i - k]),
// then the two triangular solves, q in r.  False on a pivot that is not finite and positive or a non-finite solution.
__device__ __forceinline__ bool band_solve(double (*Hb)[4], double* r, int n) {
  for (int j = 0; j < n; ++j) {
    double dj = Hb[j][0];
    for (int k = j < 3 ? 0 : j - 3; k < j; ++k) dj -= Hb[j][j - k] * Hb[j][j - k];
    if (!(dj > 0.0 && dj <= 1.7976931348623157e308)) return false;
    const double ljj = sqrt(dj);
    Hb[j][0] = ljj;
    for (int i = j + 1; i <= j + 3 && i < n; ++i) {
      double s = Hb[i][i - j];
      for (int k = i - 3; k < j; ++k)
        if (k >= 0) s -= Hb[i][i - k] * Hb[j][j - k];
      Hb[i][i - j] = s / ljj;
    }
  }
  for (int j = 0; j < n; ++j) {  // L z = r
    double s = r[j];
    for (int k = j < 3 ? 0 : j - 3; k < j; ++k) s -= Hb[j][j - k] * r[k];
    r[j] = s / Hb[j][0];
  }
  for (int j = n - 1; j >= 0; --j) {  // L^T q = z
    double s = r[j];
    for (int i = j + 1; i <= j + 3 && i < n; ++i) s -= Hb[i][i - j] * r[i];
    r[j] = s / Hb[j][0];
  }
  bool fin = true;
  for (int j = 0; j < n; ++j) fin = fin && isfinite(r[j]);
  return fin;
}

// One warp per trajectory.  Lanes 0..10 evaluate the look-ahead differences of waypoints 1..11 with the check kernels'
// deboor; lane 0 then chains calcNextYaw in the reference's order, builds the initial guess and pt_dist_, assembles the
// normal equations of combineCost's SMOOTHNESS | START | END | WAYPOINTS terms (dim_ == 1) and solves them by banded
// Cholesky.  Each term is stored as w * (a . q - t)^2 with integer a: 1/6 (1, 4, 1) becomes (1, 4, 1) over w / 36 and
// 6 t, 1/(2 dt) (-1, 0, 1) becomes (-1, 0, 1) over w / (4 dt^2) and 2 dt t, 1/dt^2 (1, -2, 1) likewise.
__global__ void __launch_bounds__(TC_WPB * 32) yaw_explore_kernel(int B, int n, int nvar, const double* __restrict__ x,
                                                                  const double* __restrict__ dtv,
                                                                  const double* __restrict__ syaw,
                                                                  const double* __restrict__ eyaw, FuelOptParams prm,
                                                                  FuelYawParams yprm, double* __restrict__ yaw,
                                                                  FuelYawInfo* __restrict__ info,
                                                                  double* __restrict__ wpt) {
  __shared__ YawSmem sm[TC_WPB];
  const int lane = threadIdx.x & 31;
  const int b = blockIdx.x * TC_WPB + (threadIdx.x >> 5);
  if (b >= B) return;
  YawSmem& y = sm[threadIdx.x >> 5];
  const double nan = __longlong_as_double(0x7ff8000000000000ll);

  const double dt = nvar == 3 * n + 1 ? x[(size_t)b * nvar + 3 * n] : dtv[b];
  double y0 = syaw[3 * b];
  const double y1 = syaw[3 * b + 1], y2 = syaw[3 * b + 2];
  double ye = eyaw[b];
  bool bad = !(dt > 0.0 && dt <= 1.7976931348623157e308) || !isfinite(y1) || !isfinite(y2) || !isfinite(ye) ||
             !(fabs(y0) <= FUELGPU_YAW_MAX_START);
  double dt_yaw = nan, duration = nan;
  if (!bad) {
    load_spline(y.s, b, n, nvar, x, dtv, lane);
    duration = y.s.U[n] - y.s.U[3];  // getTimeSum
    dt_yaw = duration / YS;
    bad = !(dt_yaw > 0.0 && dt_yaw <= 1.7976931348623157e308);
  }
  int status = 0, nw = 0;
  if (bad) {
    status = FUELGPU_YAW_BAD_INPUT;
    dt_yaw = nan;
  } else if (yprm.lookfwd) {
    // (int)(relax_time / dt_yaw): any quotient >= 11 leaves no waypoint; from 2^31 on the conversion is undefined
    const double qr = yprm.relax_time / dt_yaw;
    if (qr >= 2147483648.0) status = FUELGPU_YAW_RELAX_OVERFLOW;
    else nw = qr >= (double)YW ? 0 : YW - (int)qr;
  }
  // waypoint i = l + 1: lane l evaluates pc at tc, lane l + 16 pf at min(duration, tc + forward_t)
  const int l = lane & 15;
  double p[3] = {0.0, 0.0, 0.0};
  if (l < nw) {
    const double tc = (double)(l + 1) * dt_yaw;
    const double tf2 = tc + 2.0;
    const double t = lane < 16 ? tc : tf2 < duration ? tf2 : duration;
    int k = 3;
    deboor<3>(y.s.P, y.s.U, n, t + y.s.U[3], &k, p);
  }
  const double dx = __shfl_down_sync(FULL, p[0], 16) - p[0], dy = __shfl_down_sync(FULL, p[1], 16) - p[1],
               dz = __shfl_down_sync(FULL, p[2], 16) - p[2];
  if (lane < nw) y.wp[lane] = sqrt((dx * dx + dy * dy) + dz * dz) > 1e-6 ? atan2(dy, dx) : nan;
  __syncwarp();
  if (lane != 0) return;

  // the start wrap (|y0| <= FUELGPU_YAW_MAX_START bounds it) and the calcNextYaw chain (:782-821)
  if (!bad) {
    while (y0 < -YAW_PI) y0 += 2 * YAW_PI;
    while (y0 > YAW_PI) y0 -= 2 * YAW_PI;
  }
  double last_yaw = y0;
  for (int i = 0; i < nw; ++i) {
    double w = y.wp[i];
    if (w != w) {  // waypt = waypts.back()
      if (i == 0) {
        status = FUELGPU_YAW_NO_LOOKAHEAD;
        break;
      }
      w = y.wp[i - 1];
    } else {
      w = next_yaw(last_yaw, w);
    }
    last_yaw = w;
    y.wp[i] = w;
  }
  double pt_dist = nan;
  if (status == 0) {
    ye = next_yaw(last_yaw, ye);
    // the initial guess: states2pts * start_yaw3d in rows 0-2, states2pts * (end, 0, 0) in rows 12-14
    const double c13 = ((1 / 3.0) * dt_yaw) * dt_yaw, c16 = ((-(1 / 6.0)) * dt_yaw) * dt_yaw;
    double g[YP];
#pragma unroll
    for (int i = 0; i < YP; ++i) g[i] = 0.0;
    g[0] = (1.0 * y0 + -dt_yaw * y1) + c13 * y2;
    g[1] = (1.0 * y0 + 0.0 * y1) + c16 * y2;
    g[2] = (1.0 * y0 + dt_yaw * y1) + c13 * y2;
    g[YS] = (1.0 * ye + -dt_yaw * 0.0) + c13 * 0.0;
    g[YS + 1] = (1.0 * ye + 0.0 * 0.0) + c16 * 0.0;
    g[YS + 2] = (1.0 * ye + dt_yaw * 0.0) + c13 * 0.0;
    double d = 0.0;  // pt_dist_ (bspline_optimizer.cpp:136-140): |row(i + 1) - row(i)| of a one-column matrix
#pragma unroll
    for (int i = 0; i < YP - 1; ++i) {
      const double e = g[i + 1] - g[i];
      d += sqrt(e * e);
    }
    pt_dist = d / (double)YP;
    if (pt_dist == 0.0) status = FUELGPU_YAW_ZERO_PT_DIST;
  }

  if (status == 0) {
#pragma unroll
    for (int i = 0; i < YP; ++i) {
      y.r[i] = 0.0;
#pragma unroll
      for (int k = 0; k < 4; ++k) y.Hb[i][k] = 0.0;
    }
    const double jerk[4] = {-1.0, 3.0, -3.0, 1.0}, pos[3] = {1.0, 4.0, 1.0}, vel[3] = {-1.0, 0.0, 1.0},
                 acc[3] = {1.0, -2.0, 1.0};
    const double ws = prm.ld_smooth / (pt_dist * pt_dist), dt2 = dt_yaw * dt_yaw;
    for (int i = 0; i + 3 < YP; ++i) yaw_term<4>(y.Hb, y.r, i, jerk, ws, 0.0);
    yaw_term<3>(y.Hb, y.r, 0, pos, prm.ld_start * 10.0 / 36.0, 6.0 * y0);
    yaw_term<3>(y.Hb, y.r, 0, vel, prm.ld_start / (4.0 * dt2), 2.0 * dt_yaw * y1);
    yaw_term<3>(y.Hb, y.r, 0, acc, prm.ld_start / (dt2 * dt2), dt2 * y2);
    yaw_term<3>(y.Hb, y.r, YS, pos, prm.ld_end / 36.0, 6.0 * ye);
    yaw_term<3>(y.Hb, y.r, YS, vel, prm.ld_end / (4.0 * dt2), 0.0);
    for (int i = 0; i < nw; ++i) yaw_term<3>(y.Hb, y.r, i + 1, pos, prm.ld_waypt / 36.0, 6.0 * y.wp[i]);
    if (!band_solve(y.Hb, y.r, YP)) status = FUELGPU_YAW_NOT_SPD;
  }

  // what the reference defined before a failure is written, the rest is NaN
  const bool have_wp = status == 0 || status == FUELGPU_YAW_ZERO_PT_DIST || status == FUELGPU_YAW_NOT_SPD;
  double* yb = yaw + (size_t)b * YP;
  for (int j = 0; j < YP; ++j) yb[j] = status == 0 ? y.r[j] : nan;
  if (wpt) {
    double* wb = wpt + (size_t)b * YW;
    for (int i = 0; i < YW; ++i) wb[i] = !have_wp ? nan : i < nw ? y.wp[i] : 0.0;
  }
  FuelYawInfo o;
  o.dt_yaw = dt_yaw;
  o.pt_dist = have_wp ? pt_dist : nan;
  o.n_waypt = have_wp ? nw : 0;
  o.status = status;
  info[b] = o;
}

// ---- planYaw (planner_manager.cpp:695-772) on each trajectory of the batch ---------------------------------------------
constexpr int PYS = FUELGPU_PLANYAW_MAX_SEG, PYP = FUELGPU_PLANYAW_MAX_PTS;
constexpr int PY_WPB = 2;  // warps per CTA: 2 x sizeof(PlanYawSmem) stays under the 48 KB of static shared memory

struct PlanYawSmem {
  SplineSmem s;
  double wp[PYS];     // atan2 of look-ahead difference i (NaN where |pd| <= 1e-6), then waypoint i
  double Hb[PYP][4];  // normal equations, Hb[i][d] = H(i, i - d); the Cholesky factor in place
  double r[PYP];      // right-hand side, then the solution
};

// One warp per trajectory.  Lanes l and l + 16 evaluate pc and pf of waypoints l, l + 16, ... with the check kernels'
// deboor, lane 0 the velocity spline at duration - 0.1; lane 0 then chains calcNextYaw in the reference's order, builds
// the initial guess and pt_dist_, assembles the normal equations of SMOOTHNESS | START | END (3 states) | WAYPOINTS
// (dim_ == 1; the integer-coefficient form of yaw_explore_kernel) and solves them with band_solve.
__global__ void __launch_bounds__(PY_WPB * 32) plan_yaw_kernel(int B, int n, int nvar, const double* __restrict__ x,
                                                               const double* __restrict__ dtv,
                                                               const double* __restrict__ syaw, FuelOptParams prm,
                                                               double* __restrict__ yaw,
                                                               FuelPlanYawInfo* __restrict__ info,
                                                               double* __restrict__ wpt) {
  __shared__ PlanYawSmem sm[PY_WPB];
  const int lane = threadIdx.x & 31;
  const int b = blockIdx.x * PY_WPB + (threadIdx.x >> 5);
  if (b >= B) return;
  PlanYawSmem& y = sm[threadIdx.x >> 5];
  const double nan = __longlong_as_double(0x7ff8000000000000ll);

  const double dt = nvar == 3 * n + 1 ? x[(size_t)b * nvar + 3 * n] : dtv[b];
  const double y0 = syaw[3 * b], y1 = syaw[3 * b + 1], y2 = syaw[3 * b + 2];
  int status = 0, seg = 0;
  double duration = nan, dt_yaw = nan;
  if (!(dt > 0.0 && dt <= 1.7976931348623157e308) || !isfinite(y1) || !isfinite(y2) ||
      !(fabs(y0) <= FUELGPU_YAW_MAX_START)) {
    status = FUELGPU_YAW_BAD_INPUT;
  } else {
    load_spline(y.s, b, n, nvar, x, dtv, lane);
    duration = y.s.U[n] - y.s.U[3];  // getTimeSum
    const double q = duration / 0.3;
    if (!(duration > 0.0 && duration <= 1.7976931348623157e308)) status = FUELGPU_YAW_BAD_INPUT;
    else if (!(q <= (double)PYS)) status = FUELGPU_YAW_TOO_LONG;
    else {
      seg = (int)ceil(q);
      dt_yaw = duration / seg;
    }
  }
  // waypoint i = base + l: lane l evaluates pc at tc, lane l + 16 pf at min(duration, tc + forward_t)
  const int l = lane & 15;
  for (int base = 0; base < seg; base += 16) {
    const int i = base + l;
    double p[3] = {0.0, 0.0, 0.0};
    if (i < seg) {
      const double tc = i * dt_yaw;
      const double tf2 = tc + 2.0;
      const double t = lane < 16 ? tc : tf2 < duration ? tf2 : duration;
      int k = 3;
      deboor<3>(y.s.P, y.s.U, n, t + y.s.U[3], &k, p);
    }
    const double dx = __shfl_down_sync(FULL, p[0], 16) - p[0], dy = __shfl_down_sync(FULL, p[1], 16) - p[1],
                 dz = __shfl_down_sync(FULL, p[2], 16) - p[2];
    if (lane < 16 && i < seg) y.wp[i] = sqrt((dx * dx + dy * dy) + dz * dz) > 1e-6 ? atan2(dy, dx) : nan;
  }
  __syncwarp();
  if (lane != 0) return;

  // the calcNextYaw chain from the unwrapped start yaw (:707-730)
  double last_yaw = y0;
  for (int i = 0; i < seg; ++i) {
    double w = y.wp[i];
    if (w != w) {  // waypt = waypts.back()
      if (i == 0) {
        status = FUELGPU_YAW_NO_LOOKAHEAD;
        break;
      }
      w = y.wp[i - 1];
    } else {
      w = next_yaw(last_yaw, w);
    }
    last_yaw = w;
    y.wp[i] = w;
  }
  const int np = seg + 3;
  double pt_dist = nan, ye = nan;
  if (status == 0) {
    // velocity_traj_.evaluateDeBoorT(duration - 0.1); evaluateDeBoor clamps it to the first knot when duration < 0.1.
    // CUDA's atan2 has C99's signed-zero cases, so atan2(+-0, -0) = +-pi as in glibc.
    double v[3];
    int k = 2;
    deboor<2>(y.s.Q, y.s.U + 1, n - 1, (duration - 0.1) + y.s.U[3], &k, v);
    ye = next_yaw(last_yaw, atan2(v[1], v[0]));
    // the initial guess: states2pts * start_yaw in rows 0-2, then states2pts * (end, 0, 0) in rows seg..seg+2
    const double c13 = ((1 / 3.0) * dt_yaw) * dt_yaw, c16 = ((-(1 / 6.0)) * dt_yaw) * dt_yaw;
    const double gs[3] = {(1.0 * y0 + -dt_yaw * y1) + c13 * y2, (1.0 * y0 + 0.0 * y1) + c16 * y2,
                          (1.0 * y0 + dt_yaw * y1) + c13 * y2};
    const double ge[3] = {(1.0 * ye + -dt_yaw * 0.0) + c13 * 0.0, (1.0 * ye + 0.0 * 0.0) + c16 * 0.0,
                          (1.0 * ye + dt_yaw * 0.0) + c13 * 0.0};
    auto pick = [](const double (&v)[3], int k) { return k == 0 ? v[0] : k == 1 ? v[1] : v[2]; };  // no local memory
    auto g = [&](int i) { return i >= seg ? pick(ge, i - seg) : i < 3 ? pick(gs, i) : 0.0; };
    double d = 0.0;  // pt_dist_ (bspline_optimizer.cpp:136-140) over the seg + 3 rows
    for (int i = 0; i + 1 < np; ++i) {
      const double e = g(i + 1) - g(i);
      d += sqrt(e * e);
    }
    pt_dist = d / (double)np;
    if (pt_dist == 0.0) status = FUELGPU_YAW_ZERO_PT_DIST;
  }

  if (status == 0) {
    for (int i = 0; i < np; ++i) {
      y.r[i] = 0.0;
#pragma unroll
      for (int k = 0; k < 4; ++k) y.Hb[i][k] = 0.0;
    }
    const double jerk[4] = {-1.0, 3.0, -3.0, 1.0}, pos[3] = {1.0, 4.0, 1.0}, vel[3] = {-1.0, 0.0, 1.0},
                 acc[3] = {1.0, -2.0, 1.0};
    const double ws = prm.ld_smooth / (pt_dist * pt_dist), dt2 = dt_yaw * dt_yaw;
    for (int i = 0; i + 3 < np; ++i) yaw_term<4>(y.Hb, y.r, i, jerk, ws, 0.0);
    yaw_term<3>(y.Hb, y.r, 0, pos, prm.ld_start * 10.0 / 36.0, 6.0 * y0);
    yaw_term<3>(y.Hb, y.r, 0, vel, prm.ld_start / (4.0 * dt2), 2.0 * dt_yaw * y1);
    yaw_term<3>(y.Hb, y.r, 0, acc, prm.ld_start / (dt2 * dt2), dt2 * y2);
    yaw_term<3>(y.Hb, y.r, seg, pos, prm.ld_end / 36.0, 6.0 * ye);
    yaw_term<3>(y.Hb, y.r, seg, vel, prm.ld_end / (4.0 * dt2), 0.0);
    yaw_term<3>(y.Hb, y.r, seg, acc, prm.ld_end / (dt2 * dt2), 0.0);
    for (int i = 0; i < seg; ++i) yaw_term<3>(y.Hb, y.r, i, pos, prm.ld_waypt / 36.0, 6.0 * y.wp[i]);
    if (!band_solve(y.Hb, y.r, np)) status = FUELGPU_YAW_NOT_SPD;
  }

  // what the reference defined before a failure is written, the rest is NaN
  const bool have_seg = status == 0 || status == FUELGPU_YAW_NO_LOOKAHEAD || status == FUELGPU_YAW_ZERO_PT_DIST ||
                        status == FUELGPU_YAW_NOT_SPD;
  const bool have_wp = status == 0 || status == FUELGPU_YAW_ZERO_PT_DIST || status == FUELGPU_YAW_NOT_SPD;
  double* yb = yaw + (size_t)b * PYP;
  for (int j = 0; j < PYP; ++j) yb[j] = status == 0 && j < np ? y.r[j] : nan;
  if (wpt) {
    double* wb = wpt + (size_t)b * PYS;
    for (int i = 0; i < PYS; ++i) wb[i] = !have_wp ? nan : i < seg ? y.wp[i] : 0.0;
  }
  FuelPlanYawInfo o;
  o.dt_yaw = have_seg ? dt_yaw : nan;
  o.pt_dist = have_wp ? pt_dist : nan;
  o.seg_num = have_seg ? seg : 0;
  o.n_waypt = have_wp ? seg : 0;
  o.status = status;
  o.reserved = 0;
  info[b] = o;
}

}  // namespace

int traj_check_impl(FuelMap* m, int B, int n_pts, int nvar, const double* x_dev, const double* dt_dev,
                    const FuelTrajCheckParams* p, FuelTrajReport* rep_dev, int32_t* best_dev) {
  if (B == 0) {
    FUEL_CUDA(m, cudaMemsetAsync(best_dev, 0xff, 2 * sizeof(int32_t), m->stream));  // -1, -1
    return 0;
  }
  const int grid = (B + TC_WPB - 1) / TC_WPB;
  traj_check_kernel<<<grid, TC_WPB * 32, 0, m->stream>>>(m->g, m->occ, B, n_pts, nvar, x_dev, dt_dev, *p, rep_dev);
  FUEL_CUDA(m, cudaGetLastError());
  traj_best_kernel<<<1, 1024, 0, m->stream>>>(rep_dev, B, best_dev);
  FUEL_CUDA(m, cudaGetLastError());
  FUEL_LAUNCHES(m, 2);
  return 0;
}

int traj_evaluate_impl(FuelMap* m, int B, int n_pts, int nvar, const double* x_dev, const double* dt_dev, int n_t,
                       const double* t_dev, int deriv, double* out_dev) {
  if (B == 0 || n_t == 0) return 0;
  const int grid = (B + TC_WPB - 1) / TC_WPB;
  traj_evaluate_kernel<<<grid, TC_WPB * 32, 0, m->stream>>>(B, n_pts, nvar, x_dev, dt_dev, n_t, t_dev, deriv, out_dev);
  FUEL_CUDA(m, cudaGetLastError());
  FUEL_LAUNCHES(m, 1);
  return 0;
}

int traj_param_impl(FuelMap* m, int B, int n_pts, int nvar, const double* pts_dev, const double* der_dev,
                    const double* dt_dev, const double* tlb_dev, double* x_dev, FuelTrajConst* tc_dev) {
  if (B == 0) return 0;
  const int grid = (B + TC_WPB - 1) / TC_WPB;
  traj_param_kernel<<<grid, TC_WPB * 32, 0, m->stream>>>(B, n_pts, nvar, pts_dev, der_dev, dt_dev, tlb_dev, x_dev, tc_dev);
  FUEL_CUDA(m, cudaGetLastError());
  FUEL_LAUNCHES(m, 1);
  return 0;
}

int yaw_explore_impl(FuelMap* m, int B, int n_pts, int nvar, const double* x_dev, const double* dt_dev,
                     const double* syaw_dev, const double* eyaw_dev, const FuelOptParams* p, const FuelYawParams* yp,
                     double* yaw_dev, FuelYawInfo* info_dev, double* wpt_dev) {
  if (B == 0) return 0;
  const int grid = (B + TC_WPB - 1) / TC_WPB;
  yaw_explore_kernel<<<grid, TC_WPB * 32, 0, m->stream>>>(B, n_pts, nvar, x_dev, dt_dev, syaw_dev, eyaw_dev, *p, *yp,
                                                          yaw_dev, info_dev, wpt_dev);
  FUEL_CUDA(m, cudaGetLastError());
  FUEL_LAUNCHES(m, 1);
  return 0;
}

int plan_yaw_impl(FuelMap* m, int B, int n_pts, int nvar, const double* x_dev, const double* dt_dev,
                  const double* syaw_dev, const FuelOptParams* p, double* yaw_dev, FuelPlanYawInfo* info_dev,
                  double* wpt_dev) {
  if (B == 0) return 0;
  const int grid = (B + PY_WPB - 1) / PY_WPB;
  plan_yaw_kernel<<<grid, PY_WPB * 32, 0, m->stream>>>(B, n_pts, nvar, x_dev, dt_dev, syaw_dev, *p, yaw_dev, info_dev,
                                                       wpt_dev);
  FUEL_CUDA(m, cudaGetLastError());
  FUEL_LAUNCHES(m, 1);
  return 0;
}
