/* fuel_oracle_poly.c -- see fuel_oracle_poly.h.  Line-faithful: the same matrices, products in the order the reference
 * writes them, the same sums.  Compiled with -O3 -ffp-contract=off -fno-builtin-pow (poly.mk): pow() is libm's. */
#include "fuel_oracle_poly.h"

#include <math.h>
#include <stdlib.h>
#include <string.h>

int32_t orc_lu_inverse(int32_t n, const double* M, double* Minv) {
  double* LU = (double*)malloc(sizeof(double) * n * n);
  int32_t* perm = (int32_t*)malloc(sizeof(int32_t) * n);
  double* y = (double*)malloc(sizeof(double) * n);
  int32_t rc = 0;
  memcpy(LU, M, sizeof(double) * n * n);
  for (int i = 0; i < n; ++i) perm[i] = i;
  for (int k = 0; k < n && rc == 0; ++k) {
    int p = k;
    for (int i = k + 1; i < n; ++i)
      if (fabs(LU[i * n + k]) > fabs(LU[p * n + k])) p = i;
    if (LU[p * n + k] == 0.0) {
      rc = -1;
      break;
    }
    if (p != k) {
      for (int j = 0; j < n; ++j) {
        const double t = LU[k * n + j];
        LU[k * n + j] = LU[p * n + j];
        LU[p * n + j] = t;
      }
      const int32_t t = perm[k];
      perm[k] = perm[p];
      perm[p] = t;
    }
    for (int i = k + 1; i < n; ++i) {
      const double l = LU[i * n + k] / LU[k * n + k];
      LU[i * n + k] = l;
      for (int j = k + 1; j < n; ++j) LU[i * n + j] -= l * LU[k * n + j];
    }
  }
  for (int c = 0; c < n && rc == 0; ++c) {  /* column c of the inverse: L U x = P e_c */
    for (int i = 0; i < n; ++i) {
      double s = perm[i] == c ? 1.0 : 0.0;
      for (int j = 0; j < i; ++j) s -= LU[i * n + j] * y[j];
      y[i] = s;
    }
    for (int i = n - 1; i >= 0; --i) {
      double s = y[i];
      for (int j = i + 1; j < n; ++j) s -= LU[i * n + j] * Minv[j * n + c];
      Minv[i * n + c] = s / LU[i * n + i];
    }
  }
  free(LU);
  free(perm);
  free(y);
  return rc;
}

void orc_matmul(int32_t n, int32_t m, int32_t p, const double* A, const double* B, double* C) {
  for (int i = 0; i < n; ++i)
    for (int j = 0; j < p; ++j) {
      double s = A[i * m] * B[j];
      for (int k = 1; k < m; ++k) s = s + A[i * m + k] * B[k * p + j];
      C[i * p + j] = s;
    }
}

static double* mat(int r, int c) { return (double*)calloc((size_t)r * c, sizeof(double)); }

static void transpose(int r, int c, const double* M, double* T) {
  for (int i = 0; i < r; ++i)
    for (int j = 0; j < c; ++j) T[j * r + i] = M[i * c + j];
}

static int factorial(int x) {
  int fac = 1;
  for (int i = x; i > 0; i--) fac = fac * i;
  return fac;
}

int32_t orc_poly_waypoints(int32_t S, const double* waypts, const double* start_vel, const double* end_vel,
                           const double* start_acc, const double* end_acc, const double* times, double* coeffs,
                           double* A_out, double* Q_out, double* Ct_out, double* D_out) {
  if (S < 2) return -1;
  const int nd = 6 * S, nf = 2 * S + 4, np = 2 * S - 2, nc = nf + np;
  double* Dv = mat(3, nd); /* Dx, Dy, Dz */
  for (int k = 0; k < S; k++) {
    for (int a = 0; a < 3; ++a) {
      Dv[a * nd + k * 6] = waypts[3 * k + a];
      Dv[a * nd + k * 6 + 1] = waypts[3 * (k + 1) + a];
    }
    if (k == 0) {
      for (int a = 0; a < 3; ++a) Dv[a * nd + k * 6 + 2] = start_vel[a];
      for (int a = 0; a < 3; ++a) Dv[a * nd + k * 6 + 4] = start_acc[a];
    } else if (k == S - 1) {
      for (int a = 0; a < 3; ++a) Dv[a * nd + k * 6 + 3] = end_vel[a];
      for (int a = 0; a < 3; ++a) Dv[a * nd + k * 6 + 5] = end_acc[a];
    }
  }
  double* A = mat(nd, nd);
  for (int k = 0; k < S; k++) {
    double Ab[36] = { 0 };
    for (int i = 0; i < 3; i++) {
      Ab[(2 * i) * 6 + i] = factorial(i);
      for (int j = i; j < 6; j++) Ab[(2 * i + 1) * 6 + j] = factorial(j) / factorial(j - i) * pow(times[k], j - i);
    }
    for (int i = 0; i < 6; ++i)
      for (int j = 0; j < 6; ++j) A[(k * 6 + i) * nd + k * 6 + j] = Ab[i * 6 + j];
  }
  double* Ct = mat(nd, nc);
#define CT(r, c) Ct[(r) * nc + (c)]
  CT(0, 0) = 1;
  CT(2, 1) = 1;
  CT(4, 2) = 1;
  CT(1, 3) = 1;
  CT(3, 2 * S + 4) = 1;
  CT(5, 2 * S + 5) = 1;
  CT(6 * (S - 1) + 0, 2 * S + 0) = 1;
  CT(6 * (S - 1) + 1, 2 * S + 1) = 1;
  CT(6 * (S - 1) + 2, 4 * S + 0) = 1;
  CT(6 * (S - 1) + 3, 2 * S + 2) = 1;
  CT(6 * (S - 1) + 4, 4 * S + 1) = 1;
  CT(6 * (S - 1) + 5, 2 * S + 3) = 1;
  for (int j = 2; j < S; j++) {
    CT(6 * (j - 1) + 0, 2 + 2 * (j - 1) + 0) = 1;
    CT(6 * (j - 1) + 1, 2 + 2 * (j - 1) + 1) = 1;
    CT(6 * (j - 1) + 2, 2 * S + 4 + 2 * (j - 2) + 0) = 1;
    CT(6 * (j - 1) + 3, 2 * S + 4 + 2 * (j - 1) + 0) = 1;
    CT(6 * (j - 1) + 4, 2 * S + 4 + 2 * (j - 2) + 1) = 1;
    CT(6 * (j - 1) + 5, 2 * S + 4 + 2 * (j - 1) + 1) = 1;
  }
#undef CT
  double* Cm = mat(nc, nd);
  transpose(nd, nc, Ct, Cm);
  double* D1 = mat(3, nc); /* Dx1 = C * Dx, ... */
  for (int a = 0; a < 3; ++a) orc_matmul(nc, nd, 1, Cm, Dv + a * nd, D1 + a * nc);
  double* Q = mat(nd, nd);
  for (int k = 0; k < S; k++)
    for (int i = 3; i < 6; i++)
      for (int j = 3; j < 6; j++)
        Q[(k * 6 + i) * nd + k * 6 + j] =
            i * (i - 1) * (i - 2) * j * (j - 1) * (j - 2) / (i + j - 5) * pow(times[k], (i + j - 5));
  /* R = C * A.transpose().inverse() * Q * A.inverse() * Ct, left to right */
  double *At = mat(nd, nd), *AtI = mat(nd, nd), *AI = mat(nd, nd);
  double *T1 = mat(nc, nd), *T2 = mat(nc, nd), *T3 = mat(nc, nd), *R = mat(nc, nc);
  int32_t rc = 0;
  transpose(nd, nd, A, At);
  rc |= orc_lu_inverse(nd, At, AtI);
  rc |= orc_lu_inverse(nd, A, AI);
  orc_matmul(nc, nd, nd, Cm, AtI, T1);
  orc_matmul(nc, nd, nd, T1, Q, T2);
  orc_matmul(nc, nd, nd, T2, AI, T3);
  orc_matmul(nc, nd, nc, T3, Ct, R);
  /* Rfp = R.block(0, nf, nf, np), Rpp = R.block(nf, nf, np, np); Dp = -(Rpp.inverse() * Rfp.transpose()) * Df */
  double *Rfp = mat(nf, np), *RfpT = mat(np, nf), *Rpp = mat(np, np), *RppI = mat(np, np), *M = mat(np, nf);
  for (int i = 0; i < nf; ++i)
    for (int j = 0; j < np; ++j) Rfp[i * np + j] = R[i * nc + nf + j];
  for (int i = 0; i < np; ++i)
    for (int j = 0; j < np; ++j) Rpp[i * np + j] = R[(nf + i) * nc + nf + j];
  transpose(nf, np, Rfp, RfpT);
  rc |= orc_lu_inverse(np, Rpp, RppI);
  orc_matmul(np, np, nf, RppI, RfpT, M);
  for (int i = 0; i < np * nf; ++i) M[i] = -M[i];
  double* Dp = mat(1, np);
  for (int a = 0; a < 3; ++a) {
    orc_matmul(np, nf, 1, M, D1 + a * nc, Dp); /* Dxf = Dx1.segment(0, nf) */
    for (int i = 0; i < np; ++i) D1[a * nc + nf + i] = Dp[i];
  }
  /* P = (A.inverse() * Ct) * D1 */
  double *AC = mat(nd, nc), *P = mat(1, nd);
  orc_matmul(nd, nd, nc, AI, Ct, AC);
  for (int a = 0; a < 3; ++a) {
    orc_matmul(nd, nc, 1, AC, D1 + a * nc, P);
    for (int k = 0; k < S; ++k)
      for (int i = 0; i < 6; ++i) coeffs[(k * 3 + a) * 6 + i] = P[k * 6 + i];
  }
  if (A_out) memcpy(A_out, A, sizeof(double) * nd * nd);
  if (Q_out) memcpy(Q_out, Q, sizeof(double) * nd * nd);
  if (Ct_out) memcpy(Ct_out, Ct, sizeof(double) * nd * nc);
  if (D_out) memcpy(D_out, Dv, sizeof(double) * 3 * nd);
  free(Dv), free(A), free(Ct), free(Cm), free(D1), free(Q), free(At), free(AtI), free(AI), free(T1), free(T2);
  free(T3), free(R), free(Rfp), free(RfpT), free(Rpp), free(RppI), free(M), free(Dp), free(AC), free(P);
  return rc ? -1 : 0;
}

/* Polynomial::getTBasis / evaluate (polynomial_traj.h:27-45) */
static double tbasis(double t, int n, int k) {
  int coeff = 1;
  for (int i = n; i >= n - k + 1; --i) coeff *= i;
  return coeff * pow(t, n - k);
}

void orc_poly_evaluate(int32_t S, const double* coeffs, const double* times, double t, int32_t k, double* out) {
  int idx = 0;
  double ts = t;
  while (times[idx] + 1e-4 < ts) ts -= times[idx++];
  (void)S;
  double tv[6] = { 0 };
  for (int i = k; i < 6; ++i) tv[i] = tbasis(ts, i, k);
  for (int a = 0; a < 3; ++a) {
    const double* c = coeffs + (idx * 3 + a) * 6;
    double s = tv[0] * c[0];
    for (int i = 1; i < 6; ++i) s = s + tv[i] * c[i];
    out[a] = s;
  }
}

double orc_poly_total_time(int32_t S, const double* times) {
  double s = 0.0;
  for (int i = 0; i < S; ++i) s += times[i];
  return s;
}

double orc_poly_length(int32_t S, const double* coeffs, const double* times, int32_t* n_samples) {
  const double total_t = orc_poly_total_time(S, times);
  double eval_t = 0.0, length = 0.0, prev[3], cur[3];
  int n = 0;
  while (eval_t < total_t) {
    orc_poly_evaluate(S, coeffs, times, eval_t, 0, cur);
    if (n > 0) {
      const double dx = cur[0] - prev[0], dy = cur[1] - prev[1], dz = cur[2] - prev[2];
      length += sqrt((dx * dx + dy * dy) + dz * dz);
    }
    memcpy(prev, cur, sizeof(prev));
    ++n;
    eval_t += 0.01;
  }
  if (n_samples) *n_samples = n;
  return length;
}

int32_t orc_explore_samples(int32_t W, const double* waypts, const double* cur_vel, const double* cur_acc, double max_vel,
                            double ctrl_pt_dist, int32_t min_seg_num, int32_t max_k, double* times_out, double* coeffs,
                            double* points, double* derivs, double* out_d, int32_t* out_i) {
  const int S = W - 1;
  if (S < 2) return -1;
  double* times = (double*)malloc(sizeof(double) * S);
  double* cf = (double*)malloc(sizeof(double) * S * 18);
  for (int i = 0; i < S; ++i) {
    const double dx = waypts[3 * i + 3] - waypts[3 * i], dy = waypts[3 * i + 4] - waypts[3 * i + 1],
                 dz = waypts[3 * i + 5] - waypts[3 * i + 2];
    times[i] = sqrt((dx * dx + dy * dy) + dz * dz) / (max_vel * 0.5);
  }
  const double zero[3] = { 0, 0, 0 };
  int32_t rc = orc_poly_waypoints(S, waypts, cur_vel, zero, cur_acc, zero, times, cf, NULL, NULL, NULL, NULL);
  const double duration = orc_poly_total_time(S, times);
  const double length = orc_poly_length(S, cf, times, NULL);
  int seg_num = (int)(length / ctrl_pt_dist);
  seg_num = seg_num > min_seg_num ? seg_num : min_seg_num;
  const double dt = duration / (double)seg_num;
  int K = 0;
  for (double ts = 0.0; ts <= duration + 1e-4; ts += dt) {
    if (K < max_k) orc_poly_evaluate(S, cf, times, ts, 0, points + 3 * K);
    ++K;
  }
  orc_poly_evaluate(S, cf, times, 0.0, 1, derivs);
  orc_poly_evaluate(S, cf, times, duration, 1, derivs + 3);
  orc_poly_evaluate(S, cf, times, 0.0, 2, derivs + 6);
  orc_poly_evaluate(S, cf, times, duration, 2, derivs + 9);
  out_d[0] = duration, out_d[1] = length, out_d[2] = dt;
  out_i[0] = seg_num, out_i[1] = K;
  if (times_out) memcpy(times_out, times, sizeof(double) * S);
  if (coeffs) memcpy(coeffs, cf, sizeof(double) * S * 18);
  free(times);
  free(cf);
  return rc;
}
