"""Pins the oracle's planYawExplore (oracle/yaw.py) against the REFERENCE's own lines run over its compiled
NonUniformBspline (oracle/ref_yaw_wrap.cpp in oracle/_ref/libfuel_ref_yaw.so, built by oracle/yaw.mk) bit for bit:
dt_yaw, relax_num, the waypoints and waypt_idx, calcNextYaw of the end yaw, the wrapped start, the initial guess and
pt_dist_.  Pins the reference's combineCost with dim_ == 1 (its BsplineOptimizer driven with a 15 x 1 matrix,
oracle/ref_yaw_cost_wrap.cpp) against the oracle's 3-D combineCost on zero-padded control points, cost and gradient.
Checks the oracle's dense solve against the exact rational minimizer (tests/yaw_cases.py).  Where the reference library
is not built, the digests in tests/golden/refpin_yaw.json stand in for it.

  FUEL_REFPIN_RECORD=1 python -m pytest tests/test_oracle_yaw.py

rewrites the digests from a run against the built reference."""
import math

import numpy as np
import pytest

import oracle.yaw as OY
from fuel_b200 import workloads as W
from tests.refgold import ref_map, refgold_fixture
from tests.yaw_cases import DT_YAW_GRID, LD, arc_batch, exact_minimizer, solve_bar

OY.build()

MAP = dict(resolution=0.1, map_size_x=8.0, map_size_y=6.0, map_size_z=3.0, ground_height=-0.5, obstacles_inflation=0.199,
           local_bound_inflate=0.5, local_map_margin=50, default_dist=0.0, optimistic=0, signed_dist=0, p_hit=0.65,
           p_miss=0.35, p_min=0.12, p_max=0.90, p_occ=0.80, max_ray_length=4.5, virtual_ceil_height=-10.0)


G = refgold_fixture("refpin_yaw.json", OY.ref_yaw)


def pinned(r):
    """what the reference's driver records, from a row of oracle.yaw.plan"""
    return dict(dt_yaw=r["dt_yaw"], relax_num=-1 if r["relax_num"] is None else r["relax_num"], waypts=list(r["waypts"]),
                waypt_idx=[float(i) for i in r["waypt_idx"]], end_yaw=r["end_yaw"], start=r["start"][0],
                guess=list(r["guess"]), pt_dist=r["pt_dist"])


def ref_pinned(x, b, n, dt, sy, ey, relax, lookfwd):
    o = OY.ref_plan(x[b, :3 * n].reshape(n, 3), dt, sy, ey, relax_time=relax, lookfwd=lookfwd)
    o["waypt_idx"] = [float(i) for i in o["waypt_idx"]]
    o["relax_num"] = -1 if o["relax_num"] is None else o["relax_num"]
    o["start"] = o["start"][0]
    return o


# ---- against the reference's own code ------------------------------------------------------------------------------
@pytest.mark.parametrize("relax", (0.0, 0.3, 1.0, 2.5, 20.0))
def test_plan_matches_reference(G, relax):
    """a grid of durations (dt_yaw 0.02 .. 1 s), start yaws up to five turns outside [-pi, pi], end yaws near +-pi of
    the heading, with and without lookfwd"""
    x = arc_batch([d for d in DT_YAW_GRID for _ in range(3)], seed=11)
    B = len(x)
    c = x[:, :60].reshape(B, 20, 3)
    ys = W.make_yaws(B, seed=12, heading=np.arctan2(c[:, -1, 1] - c[:, -4, 1], c[:, -1, 0] - c[:, -4, 0]))
    for lookfwd in (True, False):
        rows = OY.plan(x, 20, ys["start"], ys["end"], relax_time=relax, lookfwd=lookfwd)
        assert all(r["status"] == OY.OK for r in rows)
        got = [pinned(r) for r in rows]
        G.eq(got, lambda: [ref_pinned(x, b, 20, x[b, 60], ys["start"][b], ys["end"][b], relax, lookfwd)
                           for b in range(B)])


def test_calc_next_yaw_at_exactly_pi(G):
    """calcNextYaw with diff exactly +pi and -pi (the reference's first branch takes both), and wrapped starts at
    exactly +-pi"""
    x = arc_batch([0.2] * 6, seed=13)
    starts = [(0.0, math.pi), (0.0, -math.pi), (math.pi, 0.0), (-math.pi, 0.0), (3 * math.pi, 0.0), (-7 * math.pi, 1.0)]
    sy = np.array([[s, 0.1, -0.2] for s, _ in starts])
    ey = np.array([e for _, e in starts])
    rows = OY.plan(x, 20, sy, ey, lookfwd=False)
    diffs = [OY.next_yaw_diff(r["start"][0], e) for r, e in zip(rows, ey)]
    assert diffs[0] == math.pi and diffs[1] == -math.pi and diffs[2] == -math.pi and diffs[3] == math.pi
    got = [pinned(r) for r in rows]
    G.eq(got, lambda: [ref_pinned(x, b, 20, x[b, 60], sy[b], ey[b], 1.0, False) for b in range(len(x))])


def test_dim1_combine_cost_equals_padded_oracle(G):
    """the reference's combineCost with dim_ == 1 (15 x 1 control points) equals the oracle's 3-D combineCost on the
    same points padded with zero y and z, cost and gradient bit for bit, at the initial guess and at probe points"""
    x = arc_batch([0.05, 0.14, 0.43, 1.0] * 2, seed=14)
    ys = W.make_yaws(len(x), seed=15)
    rows = OY.plan(x, 20, ys["start"], ys["end"])
    assert any(r["waypts"] for r in rows) and any(not r["waypts"] for r in rows)
    rng = np.random.default_rng(16)
    m = ref_map(**MAP) if OY.ref_yaw() is not None else None
    try:
        for r in rows:
            probes = np.array(r["guess"])[None] + rng.normal(0.0, 0.5, (3, OY.PTS))
            pts = np.vstack([np.array(r["guess"])[None], probes])
            f, g = OY.objective([r] * len(pts), pts, **LD)
            G.eq(dict(f=f, grad=g), lambda: dict(zip(("f", "grad"), OY.ref_cost(m, r, probes, **LD))))
    finally:
        if m is not None:
            m.close()


# ---- the oracle's solve --------------------------------------------------------------------------------------------
def test_dense_solve_vs_exact_minimizer():
    """the dense fp64 solve within solve_bar * max(1, max|q|) of the exact minimizer;
    its gradient under the pinned combineCost vanishes to 1e-9 of the initial guess's"""
    x = arc_batch([d for d in DT_YAW_GRID for _ in range(4)], seed=17)
    ys = W.make_yaws(len(x), seed=18)
    rows = OY.plan(x, 20, ys["start"], ys["end"], relax_time=0.0)
    q = np.array([OY.solve(r, **LD) for r in rows])
    for r, qb in zip(rows, q):
        ex = np.array([float(v) for v in exact_minimizer(r, **LD)])
        bar = solve_bar(r, **LD)
        assert np.abs(qb - ex).max() <= bar * max(1.0, np.abs(ex).max()), r["dt_yaw"]
    _, g = OY.objective(rows, q, **LD)
    _, g0 = OY.objective(rows, np.array([r["guess"] for r in rows]), **LD)
    assert np.all(np.abs(g).max(1) <= 1e-9 * np.abs(g0).max(1))


def test_undefined_cases_get_statuses():
    """all-zero yaws -> ZERO_PT_DIST, a hovering trajectory -> NO_LOOKAHEAD, relax_time / dt_yaw >= 2^31 ->
    RELAX_OVERFLOW, refused inputs -> BAD_INPUT; the neighbours are planned as alone"""
    x = arc_batch([0.1] * 6, seed=19)
    x[1, :60] = np.stack([0.05 * np.arange(20), np.zeros(20), np.ones(20)], 1).reshape(-1)
    x[2, :60] = np.tile([0.3, -0.2, 1.0], 20)
    x[4, 60] = -1.0
    sy = np.tile([0.4, 0.1, 0.0], (6, 1))
    sy[1] = 0.0
    sy[5, 0] = 1000.5
    ey = np.array([0.2, 0.0, 0.1, 0.3, 0.0, 0.0])
    rows = OY.plan(x, 20, sy, ey)
    assert [r["status"] for r in rows] == [OY.OK, OY.ZERO_PT_DIST, OY.NO_LOOKAHEAD, OY.OK, OY.BAD_INPUT, OY.BAD_INPUT]
    assert pinned(rows[3]) == pinned(OY.plan(x[3:4], 20, sy[3:4], ey[3:4])[0])
    assert [r["status"] for r in OY.plan(x[:1], 20, sy[:1], ey[:1], relax_time=1e9)] == [OY.RELAX_OVERFLOW]
