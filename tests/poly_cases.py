"""Inputs and an exact ground truth for PolynomialTraj::waypointsTraj (poly_traj/src/polynomial_traj.cpp:5-175), shared
by tests/test_oracle_poly.py (CPU) and tests/test_gpu_poly_traj.py (H100).

The minimum-jerk piecewise quintic through fixed waypoints is unique: its free unknowns are the velocity and
acceleration at the S - 1 inner waypoints, and the cost is a sum of per-segment quadratic forms d_k^T H_k d_k in each
segment's endpoint derivatives d_k.  exact_minjerk() builds H_k = A_k^-T Q_k A_k^-1 in exact rational arithmetic from
the fp64 segment times, eliminates the resulting block-tridiagonal system exactly and maps the solution back to monomial
coefficients with the exact A_k^-1.  Dense rational elimination of the reference's 6S x 6S form is too slow at S = 31."""
from fractions import Fraction

import numpy as np

# the exact-solve grid: segment counts and the range of segment times
GRID_S = (2, 3, 8, 20, 31)
GRID_T = (0.05, 5.0)


def _fact(n):
    f = 1
    for i in range(2, n + 1):
        f *= i
    return f


def _inverse(M):
    """exact inverse of a square list-of-lists of Fractions (Gauss-Jordan with nonzero pivots)"""
    n = len(M)
    a = [list(r) + [Fraction(int(i == j)) for j in range(n)] for i, r in enumerate(M)]
    for k in range(n):
        p = next(i for i in range(k, n) if a[i][k] != 0)
        a[k], a[p] = a[p], a[k]
        pv = a[k][k]
        a[k] = [v / pv for v in a[k]]
        for i in range(n):
            if i != k and a[i][k] != 0:
                f = a[i][k]
                a[i] = [x - f * y for x, y in zip(a[i], a[k])]
    return [r[n:] for r in a]


def segment_forms(T):
    """exact A^-1 (coefficients from d = (p0, p1, v0, v1, a0, a1), the reference's order) and H = A^-T Q A^-1 for one
    segment of fp64 duration T"""
    T = Fraction(float(T))
    A = [[Fraction(0)] * 6 for _ in range(6)]
    for i in range(3):
        A[2 * i][i] = Fraction(_fact(i))
        for j in range(i, 6):
            A[2 * i + 1][j] = Fraction(_fact(j) // _fact(j - i)) * T ** (j - i)
    Q = [[Fraction(0)] * 6 for _ in range(6)]
    for i in range(3, 6):
        for j in range(3, 6):
            Q[i][j] = Fraction(i * (i - 1) * (i - 2) * j * (j - 1) * (j - 2) // (i + j - 5)) * T ** (i + j - 5)
    Ai = _inverse(A)
    QAi = [[sum(Q[i][k] * Ai[k][j] for k in range(6)) for j in range(6)] for i in range(6)]
    H = [[sum(Ai[k][i] * QAi[k][j] for k in range(6)) for j in range(6)] for i in range(6)]
    return Ai, H


def exact_minjerk(waypts, start_vel, start_acc, times, end_vel=(0, 0, 0), end_acc=(0, 0, 0)):
    """the minimizer of waypointsTraj's problem in exact rational arithmetic: waypts [W, 3], times [W - 1] ->
    coefficients [S, 3, 6] (cx[j] multiplies t^j), rounded to fp64"""
    P = [[Fraction(float(v)) for v in p] for p in np.asarray(waypts, dtype=np.float64)]
    S = len(P) - 1
    forms = [segment_forms(t) for t in times]
    # node state x_i = (p_i, v_i, a_i); d of segment k is (p_k, p_k+1, v_k, v_k+1, a_k, a_k+1)
    s_idx, e_idx = (0, 2, 4), (1, 3, 5)  # where the start / end state sits in d
    known = {0: ([Fraction(float(v)) for v in start_vel], [Fraction(float(v)) for v in start_acc]),
             S: ([Fraction(float(v)) for v in end_vel], [Fraction(float(v)) for v in end_acc])}
    coeffs = np.zeros((S, 3, 6))
    for ax in range(3):
        n = S - 1  # unknown pairs (v_i, a_i), i = 1..S-1
        # dense-by-block storage of the tridiagonal system: D[i], Lo[i] (coupling to i-1), rhs[i]
        D = [[[Fraction(0)] * 2 for _ in range(2)] for _ in range(n)]
        Lo = [[[Fraction(0)] * 2 for _ in range(2)] for _ in range(n)]
        rhs = [[Fraction(0)] * 2 for _ in range(n)]

        def state(i):
            if i in known:
                return [P[i][ax], known[i][0][ax], known[i][1][ax]]
            return [P[i][ax], Fraction(0), Fraction(0)]

        for k in range(S):
            H = forms[k][1]
            xs, xe = state(k), state(k + 1)
            for side, node, idx in ((0, k, s_idx), (1, k + 1, e_idx)):
                if not 1 <= node <= S - 1:
                    continue
                r0 = node - 1
                for a in (1, 2):  # rows v, a of this node
                    row = idx[a]
                    # fixed part of grad/2 = H[row, :] . d_fixed
                    g = sum(H[row][s_idx[c]] * xs[c] for c in range(3)) + sum(H[row][e_idx[c]] * xe[c] for c in range(3))
                    rhs[r0][a - 1] -= g
                    for c in (1, 2):
                        D[r0][a - 1][c - 1] += H[row][idx[c]]
                    other, oidx = (k + 1, e_idx) if side == 0 else (k, s_idx)
                    if side == 1 and 1 <= other <= S - 1:
                        for c in (1, 2):
                            Lo[r0][a - 1][c - 1] += H[row][oidx[c]]
        # block LDL^T forward elimination (upper block of row i is Lo[i+1]^T)
        def inv2(m):
            det = m[0][0] * m[1][1] - m[0][1] * m[1][0]
            return [[m[1][1] / det, -m[0][1] / det], [-m[1][0] / det, m[0][0] / det]]

        def mul(a, b):
            return [[a[i][0] * b[0][j] + a[i][1] * b[1][j] for j in range(2)] for i in range(2)]

        def mv(a, v):
            return [a[0][0] * v[0] + a[0][1] * v[1], a[1][0] * v[0] + a[1][1] * v[1]]

        def tr(a):
            return [[a[0][0], a[1][0]], [a[0][1], a[1][1]]]

        Dp, rp = [None] * n, [None] * n
        for i in range(n):
            if i == 0:
                Dp[i], rp[i] = D[i], rhs[i]
            else:
                W = mul(Lo[i], inv2(Dp[i - 1]))
                U = tr(Lo[i])
                WU = mul(W, U)
                Dp[i] = [[D[i][a][c] - WU[a][c] for c in range(2)] for a in range(2)]
                Wr = mv(W, rp[i - 1])
                rp[i] = [rhs[i][a] - Wr[a] for a in range(2)]
        u = [None] * n
        for i in range(n - 1, -1, -1):
            r = rp[i]
            if i + 1 < n:
                t = mv(tr(Lo[i + 1]), u[i + 1])
                r = [r[0] - t[0], r[1] - t[1]]
            u[i] = mv(inv2(Dp[i]), r)
        states = [state(i) for i in range(S + 1)]
        for i in range(1, S):
            states[i][1], states[i][2] = u[i - 1]
        for k in range(S):
            d = [states[k][0], states[k + 1][0], states[k][1], states[k + 1][1], states[k][2], states[k + 1][2]]
            Ai = forms[k][0]
            coeffs[k, ax] = [float(sum(Ai[j][m] * d[m] for m in range(6))) for j in range(6)]
    return coeffs


def random_tour(rng, S, t_lo=GRID_T[0], t_hi=GRID_T[1], scale=None):
    """S + 1 waypoints, start velocity / acceleration and segment times log-uniform in [t_lo, t_hi]; the waypoints
    are about 2 * t apart, as planExploreTraj's times |dp| / (max_vel * 0.5) with max_vel = 2 would make them"""
    times = np.exp(rng.uniform(np.log(t_lo), np.log(t_hi), S))
    steps = rng.normal(size=(S, 3))
    steps *= (times * (1.0 if scale is None else scale) / np.linalg.norm(steps, axis=1))[:, None]
    waypts = np.concatenate([rng.uniform(-3, 3, (1, 3)), rng.uniform(-3, 3, (1, 3)) + np.cumsum(steps, axis=0)])
    return waypts, rng.uniform(-1.2, 1.2, 3), rng.uniform(-1.2, 1.2, 3), times


def grid_cases(seed=7, per_S=3):
    """the exact-solve grid: per S in GRID_S, `per_S` tours whose times span GRID_T, one of them with every time at
    either end of the range"""
    rng = np.random.default_rng(seed)
    out = []
    for S in GRID_S:
        for c in range(per_S):
            w, v, a, t = random_tour(rng, S)
            if c == 0:
                t = np.where(np.arange(S) % 2 == 0, GRID_T[0], GRID_T[1])
                t = t.astype(np.float64)
            out.append((w, v, a, t))
    return out


def poly_eval(c, t, k):
    """d^k/dt^k of sum_j c[..., j] t^j in numpy (tests only)"""
    out = 0.0
    for j in range(k, 6):
        out = out + c[..., j] * (_fact(j) // _fact(j - k)) * t ** (j - k)
    return out
