"""The kinodynamic-search oracle in the device's arithmetic (ORC_KINO_DEVICE: correctly rounded powers outside the
search, correctly rounded acos / cos in cubic()'s three-root branch) against the reference's glibc arithmetic
(ORC_KINO_GLIBC): every discrete outcome equal on the MID rows of the office and office3 path queries and on the
hand-built cases; the doubles that differ are counted and bounded in ulps (DESIGN.md 4.14)."""
import numpy as np
import pytest

import oracle.astar as OA
import oracle.kino as OK
from fuel_b200 import workloads as W
from fuel_b200.kino_astar import NO_PATH, POOL, make_params
from tests.kino_cases import hand_cases, mid_queries

DISCRETE = ("status", "reason", "retried", "traj_status", "iter_num", "use_node_num", "n_nodes", "shot", "seg_num",
            "n_pts")


def ulps(a, b):
    a, b = np.asarray(a, np.float64).ravel(), np.asarray(b, np.float64).ravel()
    both = np.isnan(a) & np.isnan(b)
    ia, ib = a.view(np.int64), b.view(np.int64)
    ia = np.where(ia < 0, np.int64(-2 ** 63) - ia, ia)
    ib = np.where(ib < 0, np.int64(-2 ** 63) - ib, ib)
    d = np.abs(ia - ib)
    d[both] = 0
    return d


def compare_modes(om, size, q, **kw):
    p = make_params(**kw)
    a = OK.replan_batch(om, size, p, q["start"], q["vel"], q["acc"], q["goal"], math=OK.GLIBC, node_max=128)
    b = OK.replan_batch(om, size, p, q["start"], q["vel"], q["acc"], q["goal"], math=OK.DEVICE, node_max=128)
    for f in DISCRETE:
        assert np.array_equal(a["info"][f], b["info"][f]), f
    report = {}
    for k in ("points", "derivs", "dt", "nodes", "shot"):
        d = ulps(a[k], b[k]).reshape(len(q["start"]), -1)
        report[k] = (int(np.count_nonzero(d.any(axis=1))), int(d.max()) if d.size else 0)
    report["t_shot"] = (int(np.count_nonzero(ulps(a["info"]["t_shot"], b["info"]["t_shot"]))),
                        int(ulps(a["info"]["t_shot"], b["info"]["t_shot"]).max()))
    print("searches %d; rows that differ, max ulps: %s" % (len(q["start"]), report))
    # the search itself (node chain, shot time) is the reference's wherever no D < 0 branch runs, and the samples
    # differ only by the rounding of t^2 and t^3
    assert report["points"][1] <= 64 and report["derivs"][1] <= 64
    return a


@pytest.fixture(scope="module", params=["office", "office3"])
def world(request):
    g, inflate = W.office_map() if request.param == "office" else W.office3_map()
    tri = W.office_known(g, inflate)
    return g, inflate, tri, OA.Map(g, inflate, tri), g.map_max - g.origin


def test_device_math_matches_glibc_on_mid_rows(world):
    g, inflate, tri, om, size = world
    q = mid_queries(g, inflate, tri, B=1024, seed=20261019)
    assert len(q["start"]) >= 100
    r = compare_modes(om, size, q)
    assert np.count_nonzero(r["info"]["traj_status"] == 0) > len(q["start"]) // 2


@pytest.mark.parametrize("kw", [dict(), dict(optimistic=True), dict(allocate_num=40), dict(lambda_heu=0.0, allocate_num=3000),
                                dict(horizon=1.0)])
def test_device_math_matches_glibc_on_hand_cases(world, kw):
    g, inflate, tri, om, size = world
    r = compare_modes(om, size, hand_cases(g, inflate, tri), **kw)
    if kw.get("allocate_num") == 40:
        assert np.any(r["info"]["reason"] == POOL) and np.any(r["info"]["retried"] == 1)
    assert np.any(r["info"]["status"] == NO_PATH)


def test_three_root_branch_is_exercised():
    """states whose heuristic takes cubic()'s D < 0 branch: the two modes may differ there only in rounding"""
    g, inflate = W.office_map()
    tri = W.office_known(g, inflate)
    om = OA.Map(g, inflate, tri)
    q = mid_queries(g, inflate, tri, B=256, seed=99)
    # the resolvent cubic has three real roots when the goal is close and the velocity large and pointing at it: a
    # goal 0.2 to 0.45 m ahead of a start moving at 2 to 2.2 m/s towards it (the start lies within the goal tolerance,
    # so the heuristic of the start and of the shot take the branch)
    rng = np.random.default_rng(11)
    d = q["goal"] - q["start"]
    d[:, 2] = 0.0
    u = d / np.linalg.norm(d, axis=1, keepdims=True)
    q["vel"] = u * rng.uniform(2.0, 2.2, (len(u), 1))
    q["goal"] = q["start"] + u * rng.uniform(0.2, 0.45, (len(u), 1))
    OK.three_root_count(reset=True)
    compare_modes(om, g.map_max - g.origin, q)
    n = OK.three_root_count(reset=True)
    print("heuristic evaluations in the D < 0 branch: %d" % n)
    assert n > 0
