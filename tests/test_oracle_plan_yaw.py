"""Pins the oracle's planYaw (oracle.plan_yaw, the kinodynamic replan's yaw) against the REFERENCE's own lines run
over its compiled NonUniformBspline (ref_plan_yaw in oracle/_ref/libfuel_ref_plan_yaw.so) bit for bit: seg_num, dt_yaw, the
waypoints and their indices, the end velocity and yaw, the initial guess and pt_dist_.  Pins the reference's
combineCost with dim_ == 1, seg_num + 3 control points and three end states (ref_plan_yaw_cost) against the oracle's
3-D combineCost on zero-padded control points.  Checks the oracle's dense solve against the exact rational minimizer.
Where the reference library is not built, the digests in tests/golden/refpin_plan_yaw.json stand in for it.

  FUEL_REFPIN_RECORD=1 python -m pytest tests/test_oracle_plan_yaw.py

rewrites the digests from a run against the built reference."""
import math

import numpy as np

import oracle.plan_yaw as OPY
from fuel_b200 import workloads as W
from tests.plan_yaw_cases import DURATIONS, LD_KINO, duration_batch, exact_minimizer, hover_tail, solve_bar
from tests.refgold import ref_map, refgold_fixture

OPY.build()

MAP = dict(resolution=0.1, map_size_x=8.0, map_size_y=6.0, map_size_z=3.0, ground_height=-0.5, obstacles_inflation=0.199,
           local_bound_inflate=0.5, local_map_margin=50, default_dist=0.0, optimistic=0, signed_dist=0, p_hit=0.65,
           p_miss=0.35, p_min=0.12, p_max=0.90, p_occ=0.80, max_ray_length=4.5, virtual_ceil_height=-10.0)
KEYS = ("seg_num", "dt_yaw", "duration", "waypts", "waypt_idx", "end_v", "end_in", "end_yaw", "guess", "pt_dist")

G = refgold_fixture("refpin_plan_yaw.json", OPY.ref_plan_yaw_lib)


def pinned(r):
    """what the reference's driver records, from a row of oracle.plan_yaw.plan_yaw (a ZERO_PT_DIST row is complete there:
    its undefined costs come later, in the optimizer)"""
    if r["status"] not in (OPY.OK, OPY.ZERO_PT_DIST):
        return dict(status=r["status"])
    out = {k: r[k] for k in KEYS}
    out["waypt_idx"] = [float(i) for i in r["waypt_idx"]]
    out["status"] = OPY.OK
    return out


def ref_pinned(x, n, sy):
    out = []
    for b in range(len(x)):
        o = OPY.ref_plan_yaw(x[b, :3 * n].reshape(n, 3), x[b, 3 * n], sy[b])
        if o["status"] == OPY.OK:
            o["waypt_idx"] = [float(i) for i in o["waypt_idx"]]
        out.append(o)
    return out


def line_batch(durations, n_pts=20, heading=0.0):
    """straight trajectories along `heading` (atan2 of every look-ahead difference is the same value)"""
    x = np.zeros((len(durations), 3 * n_pts + 1))
    s = np.linspace(0.0, 2.0, n_pts)
    for b, d in enumerate(durations):
        x[b, :3 * n_pts] = np.stack([s * math.cos(heading), s * math.sin(heading), np.ones(n_pts)], 1).reshape(-1)
        x[b, 3 * n_pts] = d / (n_pts - 3)
    return x


# ---- against the reference's own code ------------------------------------------------------------------------------
def test_plan_yaw_matches_reference(G):
    """seg_num 1, 2, 3, 4, 20, 127, 128 and one past the cap, a duration below 0.1 s, 20 and 64 control points, start
    yaws up to +-1000 with random rates"""
    for n, seed in ((20, 21), (64, 22)):
        x = duration_batch(DURATIONS, n_pts=n, seed=seed)
        B = len(x)
        rng = np.random.default_rng(seed)
        sy = np.stack([rng.uniform(-4.0, 4.0, B), rng.uniform(-1.0, 1.0, B), rng.uniform(-2.0, 2.0, B)], 1)
        sy[0, 0], sy[1, 0] = 1000.0, -1000.0
        rows = OPY.plan_yaw(x, n, sy)
        segs = [r["seg_num"] for r in rows]
        assert {1, 2, 3, 4, 20, 127, 128} <= set(segs), segs
        assert rows[-1]["status"] == OPY.TOO_LONG and rows[0]["duration"] < 0.1
        assert all(r["status"] == OPY.OK for r in rows[:-1])
        G.eq([pinned(r) for r in rows], lambda: ref_pinned(x, n, sy))


def test_stationary_stretches_and_pi(G):
    """a stationary tail (end velocity exactly 0), a stationary start (NO_LOOKAHEAD), a later stationary stretch
    (waypts.back() repeated), calcNextYaw with diff exactly +-pi, start yaw, rate and acceleration 0 along +x
    (ZERO_PT_DIST)"""
    n = 40
    x = duration_batch([8.0] * 3, n_pts=n, seed=23)
    x = np.vstack([hover_tail(x[:1], n, k=8), x[1:]])
    c = x[:, :3 * n].reshape(3, n, 3)
    c[1, :20] = c[1, 20]  # stationary for the first half: |pd| = 0 at i = 0
    c[2, 12:30] = c[2, 12]  # stationary for about 3 s in the middle
    x[:, :3 * n] = c.reshape(3, -1)
    sy = np.array([[0.4, 0.2, 0.0], [0.1, 0.0, 0.0], [-0.3, 0.0, 0.1]])
    rows = OPY.plan_yaw(x, n, sy)
    assert [r["status"] for r in rows] == [OPY.OK, OPY.NO_LOOKAHEAD, OPY.OK]
    assert rows[0]["end_v"] == [0.0, 0.0, 0.0] and rows[0]["end_in"] == 0.0
    w = rows[2]["waypts"]
    assert any(w[i] == w[i - 1] for i in range(1, len(w)))
    G.eq([pinned(r) for r in rows], lambda: ref_pinned(x, n, sy))

    xl = line_batch([1.0, 1.0, 1.0, 1.0, 1.0, 0.05])
    syl = np.array([[math.pi, 0.0, 0.0], [-math.pi, 0.0, 0.0], [3 * math.pi, 0.1, 0.0], [0.0, 0.0, 0.0],
                    [-1000.0, 0.0, 0.0], [0.0, 0.0, 0.0]])
    rows = OPY.plan_yaw(xl, 20, syl)
    assert [OPY.next_yaw_diff(syl[b, 0], 0.0) for b in (0, 1)] == [-math.pi, math.pi]
    assert [r["status"] for r in rows] == [OPY.OK] * 3 + [OPY.ZERO_PT_DIST, OPY.OK, OPY.ZERO_PT_DIST]
    G.eq([pinned(r) for r in rows], lambda: ref_pinned(xl, 20, syl))


def test_plan_yaw_cost_equals_reference(G):
    """the reference's combineCost with dim_ == 1, seg_num + 3 control points and three end states equals the oracle's
    3-D combineCost on the same points padded with zero y and z, cost and gradient bit for bit, at the initial guess
    and at probe points (seg_num up to 61: the oracle's 64-point limit)"""
    x = duration_batch([0.05, 0.29, 0.85, 1.2, 5.95, 18.2], seed=24)
    rng = np.random.default_rng(25)
    sy = np.stack([rng.uniform(-4.0, 4.0, len(x)), rng.uniform(-1.0, 1.0, len(x)), rng.uniform(-2.0, 2.0, len(x))], 1)
    rows = OPY.plan_yaw(x, 20, sy)
    assert [r["seg_num"] for r in rows] == [1, 1, 3, 4, 20, 61]
    m = ref_map(**MAP) if OPY.ref_plan_yaw_lib() is not None else None
    try:
        for r in rows:
            probes = np.array(r["guess"])[None] + rng.normal(0.0, 0.5, (3, r["n_pts"]))
            pts = np.vstack([np.array(r["guess"])[None], probes])
            f, g = OPY.objective([r] * len(pts), pts, **LD_KINO)
            G.eq(dict(f=f, grad=np.array(g)), lambda: dict(zip(("f", "grad"), OPY.ref_plan_yaw_cost(m, r, probes))))
    finally:
        if m is not None:
            m.close()


# ---- the oracle's solve --------------------------------------------------------------------------------------------
def test_dense_solve_vs_exact_minimizer():
    """the dense fp64 solve within solve_bar * max(1, max|q|) of the exact minimizer (banded elimination in Fraction)
    at seg_num 1 .. 128; its gradient vanishes to 1e-9 of the initial guess's"""
    x = duration_batch(DURATIONS[:-1], seed=26)
    ys = W.make_yaws(len(x), seed=27)
    rows = OPY.plan_yaw(x, 20, ys["start"])
    assert all(r["status"] == OPY.OK for r in rows)
    q = [OPY.solve(r, **LD_KINO) for r in rows]
    for r, qb in zip(rows, q):
        ex = np.array([float(v) for v in exact_minimizer(r, **LD_KINO)])
        assert np.abs(qb - ex).max() <= solve_bar(r, **LD_KINO) * max(1.0, np.abs(ex).max()), r["seg_num"]
    _, g = OPY.objective(rows, q, **LD_KINO)
    _, g0 = OPY.objective(rows, [r["guess"] for r in rows], **LD_KINO)
    for a, a0 in zip(g, g0):
        assert np.abs(a).max() <= 1e-9 * np.abs(a0).max()
