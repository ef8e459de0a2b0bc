/* Held-Karp over the integer matrix findGlobalTour writes for LKH (fast_exploration_manager.cpp:357-376).  Clusters
 * are 0 .. n-1 (matrix node k + 1).  h[S][j] is the cheapest path from cluster j through every cluster of S, then back
 * to node 0; cnt[S][j] the number of such paths at that cost.  Subsets are visited in increasing numeric order, so
 * S \ k is always done before S.  TEST INFRASTRUCTURE ONLY. */
#include "fuel_oracle_gtour.h"

#include <stdlib.h>

static int32_t sat_add(int32_t a, int32_t b) {
  const int64_t s = (int64_t)a + b;
  return s > INT32_MAX ? INT32_MAX : (int32_t)s;
}

int orc_global_tour(int32_t d, const double* mat, int64_t* cost, int32_t* n_optimal, int32_t* indices) {
  const int n = d - 1;
  if (n < 1) return -1;
  if (n > ORC_GTOUR_MAX_CLUSTERS) return ORC_GTOUR_TOO_LARGE;
  int32_t* c = malloc(sizeof(int32_t) * (size_t)d * d);
  if (!c) return -1;
  for (int i = 0; i < d; ++i)
    for (int j = 0; j < d; ++j) {
      if (i == j) {
        c[i * d + j] = 0;  /* never read */
        continue;
      }
      const double p = mat[i * d + j] * 100;  /* int int_cost = cost_mat(i, j) * scale */
      if (!(p > -2147483649.0 && p < 2147483648.0)) {
        free(c);
        return ORC_GTOUR_BAD_INPUT;
      }
      c[i * d + j] = (int32_t)p;
    }
  const size_t ns = (size_t)1 << n;
  int64_t* h = malloc(sizeof(int64_t) * ns * n);
  int32_t* cnt = malloc(sizeof(int32_t) * ns * n);
  if (!h || !cnt) {
    free(c), free(h), free(cnt);
    return -1;
  }
  for (size_t S = 0; S < ns; ++S)
    for (int j = 0; j < n; ++j) {
      if ((S >> j) & 1) continue;
      int64_t best = INT64_MAX;
      int32_t ways = 0;
      if (!S) {
        best = c[(j + 1) * d];
        ways = 1;
      }
      for (int k = 0; k < n; ++k) {
        if (!((S >> k) & 1)) continue;
        const size_t q = (S ^ ((size_t)1 << k)) * n + k;
        const int64_t v = c[(j + 1) * d + k + 1] + h[q];
        if (v < best) {
          best = v;
          ways = cnt[q];
        } else if (v == best) {
          ways = sat_add(ways, cnt[q]);
        }
      }
      h[S * n + j] = best;
      cnt[S * n + j] = ways;
    }
  /* from node 0 through every cluster */
  size_t S = ns - 1;
  int64_t best = INT64_MAX;
  int32_t ways = 0;
  for (int k = 0; k < n; ++k) {
    const size_t q = (S ^ ((size_t)1 << k)) * n + k;
    const int64_t v = c[k + 1] + h[q];
    if (v < best) {
      best = v;
      ways = cnt[q];
    } else if (v == best) {
      ways = sat_add(ways, cnt[q]);
    }
  }
  *cost = best;
  *n_optimal = ways;
  /* forwards, the smallest tight cluster at each step */
  int64_t target = best;
  int row = 0;
  for (int step = 0; step < n; ++step) {
    for (int k = 0; k < n; ++k) {
      if (!((S >> k) & 1)) continue;
      const size_t q = (S ^ ((size_t)1 << k)) * n + k;
      if (c[row * d + k + 1] + h[q] == target) {
        indices[step] = k;
        target = h[q];
        S ^= (size_t)1 << k;
        row = k + 1;
        break;
      }
    }
  }
  free(c), free(h), free(cnt);
  return ORC_GTOUR_OK;
}
