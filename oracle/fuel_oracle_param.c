/* fuel_oracle_param.c -- CPU restatement of NonUniformBspline::parameterizeToBspline (bspline/src/non_uniform_bspline.cpp
 * :178-265, degree 3) with getBoundaryStates(2, 0) (:108-123) and the pt_dist_ of BsplineOptimizer::optimize()
 * (bspline_optimizer.cpp:136-140).  TEST INFRASTRUCTURE ONLY (see fuel_oracle.h).  Sequential fp64, no FMA contraction:
 * the system and the boundary states in the reference's arithmetic, what the device parameterization
 * (fuel_b200/csrc/traj_check.cu) must equal bit for bit given its control points.  Declared in fuel_oracle_param.h. */
#include <math.h>
#include <stdlib.h>
#include <string.h>

#include "fuel_oracle_param.h"
#include "fuel_oracle_traj.h"

#define ORC_PARAM_MAX_PTS 64

/* A and the three b of :199-258, in the reference's arithmetic: 1 / 6.0 * (1, 4, 1), 1 / (2 * ts) * (-1, 0, 1),
 * 1 / (ts * ts) * (1, -2, 1), scalar times vector element by element; rows: K positions, start vel, end vel, start acc,
 * end acc */
void orc_bspline_param_system(int32_t K, double ts, const double* points, const double* derivs, double* A, double* b) {
  const int rows = K + 4, cols = K + 2;
  const double pos[3] = { 1 / 6.0 * 1, 1 / 6.0 * 4, 1 / 6.0 * 1 };
  const double vel[3] = { 1 / (2 * ts) * -1, 1 / (2 * ts) * 0, 1 / (2 * ts) * 1 };
  const double acc[3] = { 1 / (ts * ts) * 1, 1 / (ts * ts) * -2, 1 / (ts * ts) * 1 };
  for (int i = 0; i < rows * cols; ++i) A[i] = 0.0;
  for (int k = 0; k < 3; ++k) {
    for (int i = 0; i < K; ++i) A[i * cols + i + k] = pos[k];
    A[K * cols + k] = vel[k];
    A[(K + 1) * cols + K - 1 + k] = vel[k];
    A[(K + 2) * cols + k] = acc[k];
    A[(K + 3) * cols + K - 1 + k] = acc[k];
  }
  for (int j = 0; j < 3; ++j) {
    for (int i = 0; i < K; ++i) b[j * rows + i] = points[3 * i + j];
    for (int i = 0; i < 4; ++i) b[j * rows + K + i] = derivs[3 * i + j];
  }
}

/* min |A x - b| for each of nrhs right-hand sides by a column-pivoted Householder QR (Businger & Golub 1965; the
 * algorithm Eigen's ColPivHouseholderQR names, restated from its published description, not from Eigen's code):
 * at step k the remaining column of largest norm is swapped in (the first on ties), a reflector zeroes it below the
 * diagonal and is applied to the remaining columns and to every b; R x = Q^T b is back-substituted for the leading
 * rank columns, the others are 0.  The rank stops at the first pivot |R(k,k)| <= 1e-16 * max(rows, cols) * |R(0,0)|.
 * A [rows][cols] row-major with rows >= cols <= 128, b [nrhs][rows] -> x [nrhs][cols]; returns the rank. */
#define ORC_QR_MAX 128
int32_t orc_lstsq_colpiv_qr(int32_t rows, int32_t cols, const double* A, int32_t nrhs, const double* b, double* x) {
  if (rows < cols || cols > ORC_QR_MAX || rows > ORC_QR_MAX + 4) return -1;
  double* R = (double*)malloc(sizeof(double) * rows * cols);
  double* y = (double*)malloc(sizeof(double) * nrhs * rows);
  double v[ORC_QR_MAX + 4];
  int perm[ORC_QR_MAX];
  for (int i = 0; i < rows * cols; ++i) R[i] = A[i];
  for (int i = 0; i < nrhs * rows; ++i) y[i] = b[i];
  for (int j = 0; j < cols; ++j) perm[j] = j;
  int rank = cols;
  double r00 = 0.0;
  for (int k = 0; k < cols; ++k) {
    int p = k;
    double best = -1.0;
    for (int j = k; j < cols; ++j) {
      double s = 0.0;
      for (int i = k; i < rows; ++i) s += R[i * cols + j] * R[i * cols + j];
      if (s > best) best = s, p = j;
    }
    if (p != k) {
      for (int i = 0; i < rows; ++i) {
        const double t = R[i * cols + k];
        R[i * cols + k] = R[i * cols + p];
        R[i * cols + p] = t;
      }
      const int t = perm[k];
      perm[k] = perm[p];
      perm[p] = t;
    }
    const double norm = sqrt(best);
    if (k == 0) r00 = norm;
    if (!(norm > 1e-16 * (rows > cols ? rows : cols) * r00)) {
      rank = k;
      break;
    }
    const double alpha = R[k * cols + k] > 0 ? -norm : norm;
    double vv = 0.0;
    for (int i = k; i < rows; ++i) {
      v[i] = R[i * cols + k];
      if (i == k) v[i] -= alpha;
      vv += v[i] * v[i];
    }
    R[k * cols + k] = alpha;
    for (int i = k + 1; i < rows; ++i) R[i * cols + k] = 0.0;
    for (int j = k + 1; j < cols; ++j) {
      double s = 0.0;
      for (int i = k; i < rows; ++i) s += v[i] * R[i * cols + j];
      const double f = 2.0 * s / vv;
      for (int i = k; i < rows; ++i) R[i * cols + j] -= f * v[i];
    }
    for (int r = 0; r < nrhs; ++r) {
      double* yr = y + (size_t)r * rows;
      double s = 0.0;
      for (int i = k; i < rows; ++i) s += v[i] * yr[i];
      const double f = 2.0 * s / vv;
      for (int i = k; i < rows; ++i) yr[i] -= f * v[i];
    }
  }
  for (int r = 0; r < nrhs; ++r) {
    const double* yr = y + (size_t)r * rows;
    double z[ORC_QR_MAX];
    for (int k = cols - 1; k >= 0; --k) {
      if (k >= rank) {
        z[k] = 0.0;
        continue;
      }
      double s = yr[k];
      for (int j = k + 1; j < rank; ++j) s -= R[k * cols + j] * z[j];
      z[k] = s / R[k * cols + k];
    }
    for (int k = 0; k < cols; ++k) x[(size_t)r * cols + perm[k]] = z[k];
  }
  free(R);
  free(y);
  return rank;
}

/* getBoundaryStates(2, 0) (:108-123) of trajectory b: start = evaluateDeBoorT(0) of the spline and of its first two
 * derivatives, end = evaluateDeBoorT(getTimeSum()) of the spline, over the trajectory oracle's evaluateDeBoorT
 * (orc_bspline_evaluate); getTimeSum() = u_(n) - u_(3) of setUniformBspline's running-sum knots (:16-32, :267-269) */
static void boundary_states(int b, int n, int nvar, const double* x, const double* dt, double* start, double* end) {
  const double* xb = x + (size_t)b * nvar;
  const double* db = nvar == 3 * n + 1 ? NULL : dt + b;
  const double span = db ? *db : xb[3 * n];
  double u[ORC_PARAM_MAX_PTS + 4];
  for (int i = 0; i <= n + 3; ++i) u[i] = i <= 3 ? (double)(-3 + i) * span : u[i - 1] + span;
  const double t0 = 0.0, duration = u[n] - u[3];
  for (int k = 0; k < 3; ++k) orc_bspline_evaluate(1, n, nvar, xb, db, 1, &t0, k, start + 3 * k);
  orc_bspline_evaluate(1, n, nvar, xb, db, 1, &duration, 0, end);
}

void orc_bspline_boundary_states(int32_t B, int32_t n_pts, int32_t nvar, const double* x, const double* dt, double* start,
                                 double* end) {
  for (int b = 0; b < B; ++b) boundary_states(b, n_pts, nvar, x, dt, start + 9 * (size_t)b, end + 3 * (size_t)b);
}

void orc_bspline_parameterize(int32_t B, int32_t n_pts, int32_t nvar, const double* points, const double* derivs,
                              const double* dt, const double* time_lb, double* x, OrcTrajConst* tc) {
  const int K = n_pts - 2, rows = K + 4, cols = K + 2;
  double* A = (double*)malloc(sizeof(double) * rows * cols);
  double bv[3 * (ORC_PARAM_MAX_PTS + 2)], ctrl[3 * ORC_PARAM_MAX_PTS], sol[3 * ORC_PARAM_MAX_PTS];
  for (int b = 0; b < B; ++b) {
    orc_bspline_param_system(K, dt[b], points + (size_t)b * K * 3, derivs + (size_t)b * 12, A, bv);
    orc_lstsq_colpiv_qr(rows, cols, A, 3, bv, sol);
    double* xb = x + (size_t)b * nvar;
    for (int i = 0; i < n_pts; ++i)
      for (int j = 0; j < 3; ++j) ctrl[3 * i + j] = xb[3 * i + j] = sol[j * cols + i];
    if (nvar == 3 * n_pts + 1) xb[3 * n_pts] = dt[b];
    OrcTrajConst* t = tc + b;
    memset(t, 0, sizeof(*t));
    boundary_states(b, n_pts, nvar, x, dt, &t->start[0][0], t->end[0]);
    t->pt_dist = orc_pt_dist(ctrl, n_pts);
    t->knot_span = dt[b];
    t->n_end = 1;
    t->time_lb = time_lb ? time_lb[b] : -1.0;
    t->view_idx = -1;
  }
  free(A);
}
