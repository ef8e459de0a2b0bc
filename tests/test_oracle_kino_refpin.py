"""Pins the kinodynamic-search oracle (oracle/fuel_oracle_kino.c) in its GLIBC mode on the REFERENCE's own
path_searching/src/kinodynamic_astar.cpp, compiled unmodified into oracle/_ref/libfuel_ref_kino.so (oracle/kino.mk)
over the reference's SDFMap, with kinodynamicReplan's lines 131-164 restated around it (oracle/ref_kino_wrap.cpp).
Bit for bit: status, retry, iter_num, use_node_num, the node chain (state, input, duration, g, f), the shot, ts, the
samples and the derivatives, on the MID rows of the office and office3 path queries and on the hand-built cases.  Where
the reference library is not built, the digests in tests/golden/refpin_kino.json stand in for it.

  FUEL_REFPIN_RECORD=1 python -m pytest tests/test_oracle_kino_refpin.py

rewrites the digests from a run against the built reference."""
import numpy as np
import pytest

import oracle as O
import oracle.kino as OK
from fuel_b200 import workloads as W
from fuel_b200.kino_astar import make_params
from tests.kino_cases import hand_cases, mid_queries
from tests.refgold import refgold_fixture

OK.build()

NODE_MAX = 128
# kinodynamic_astar.cpp's reasons are not outputs of the reference: the wrapper infers them, so they are left out
FIELDS = ("status", "retried", "traj_status", "iter_num", "use_node_num", "n_nodes", "shot", "seg_num", "n_pts",
          "t_shot", "T_sum")


def logit(p):
    return np.log(p / (1 - p))


G = refgold_fixture("refpin_kino.json", OK.ref_kino)


def flat(r):
    return [[r["info"][f].astype(np.float64) for f in FIELDS], r["points"], r["derivs"], r["dt"], r["nodes"], r["shot"]]


class Scene:
    """one map for both sides: the oracle's occupancy byte and, where it is built, the reference's SDFMap holding the
    same inflate bits and tri-state (as log-odds) with the same exploration box"""

    def __init__(self, g, inflate, tri):
        import oracle.astar as OA
        self.g, self.om = g, OA.Map(g, inflate, tri)
        self.ref = None
        if OK.ref_kino() is not None:
            p = dict(resolution=g.res, map_size_x=g.n[0] * g.res, map_size_y=g.n[1] * g.res, map_size_z=g.n[2] * g.res,
                     ground_height=g.origin[2], obstacles_inflation=0.199, local_bound_inflate=0.5, local_map_margin=50,
                     default_dist=0.0, optimistic=0, signed_dist=0, p_hit=0.65, p_miss=0.35, p_min=0.12, p_max=0.90,
                     p_occ=0.80, max_ray_length=4.5, virtual_ceil_height=-10.0)
            for k, a in enumerate("xyz"):
                p["box_min_" + a], p["box_max_" + a] = g.box_min[k], g.box_max[k]
            r = O.RefSDFMap(**p)
            assert r.n == g.n and np.array_equal(r.origin, g.origin)
            r.inflate[:] = np.asarray(inflate).reshape(-1)
            r.occupancy[:] = np.where(tri == W.UNKNOWN, logit(0.12) - 0.01,
                                      np.where(tri == W.OCCUPIED, logit(0.90), logit(0.12))).reshape(-1)
            self.ref = r

    def check(self, G, q, **kw):
        prm = make_params(**kw)
        got = OK.replan_batch(self.om, self.g.map_max - self.g.origin, prm, q["start"], q["vel"], q["acc"], q["goal"],
                              math=OK.GLIBC, node_max=NODE_MAX)

        def reference():
            rk = OK.RefKino(self.ref, prm)
            try:
                return flat(rk.replan_batch(q["start"], q["vel"], q["acc"], q["goal"], node_max=NODE_MAX))
            finally:
                rk.close()

        G.eq(flat(got), reference)
        return got

    def close(self):
        if self.ref is not None:
            self.ref.close()


@pytest.fixture(scope="module", params=["office", "office3"])
def scene(request):
    g, inflate = W.office_map() if request.param == "office" else W.office3_map()
    tri = W.office_known(g, inflate)
    s = Scene(g, inflate, tri)
    yield g, inflate, tri, s
    s.close()


def test_mid_rows_match_reference(G, scene):
    g, inflate, tri, s = scene
    q = mid_queries(g, inflate, tri, B=1024, seed=20261019)
    r = s.check(G, q)
    assert len(q["start"]) >= 100 and np.count_nonzero(r["info"]["traj_status"] == 0) > len(q["start"]) // 2


@pytest.mark.parametrize("kw", [dict(), dict(optimistic=True), dict(allocate_num=40), dict(lambda_heu=0.0, allocate_num=3000),
                                dict(horizon=1.0)])
def test_hand_cases_match_reference(G, scene, kw):
    g, inflate, tri, s = scene
    s.check(G, hand_cases(g, inflate, tri), **kw)
