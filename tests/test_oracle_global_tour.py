"""The global-tour oracle (oracle.gtour: Held-Karp over the integer ATSP FastExplorationManager::findGlobalTour hands
to LKH) against brute force over every permutation, and the C layout of FuelGlobalTourInfo and the new entries'
binding.  CPU only."""
import ctypes as C
import itertools
import os
import subprocess

import numpy as np
import pytest

import oracle.gtour as OG

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def brute(mat):
    """every tour of the integer matrix -> (cost, n_optimal, lexicographically smallest optimal tour), or None where
    an off-diagonal int(cost * 100) is undefined"""
    d = mat.shape[0]
    p = np.asarray(mat, np.float64) * 100.0
    off = ~np.eye(d, dtype=bool)
    with np.errstate(invalid="ignore"):
        if not np.all((p[off] > -2147483649.0) & (p[off] < 2147483648.0)):
            return None
    c = OG.int_matrix(np.where(off, mat, 0.0))
    best, count, first = None, 0, None
    for perm in itertools.permutations(range(d - 1)):  # lexicographic order
        v = OG.tour_cost(c, perm)
        if best is None or v < best:
            best, count, first = v, 1, list(perm)
        elif v == best:
            count += 1
    return best, count, first


def _cases():
    rng = np.random.default_rng(7)
    out = []
    for n in range(1, 9):
        d = n + 1
        out.append(("random%d" % n, rng.uniform(0, 20, (d, d))))
        out.append(("ints%d" % n, rng.integers(0, 4, (d, d)).astype(np.float64)))  # many ties
        out.append(("equal%d" % n, np.full((d, d), 3.5)))
        neg = rng.uniform(-10, 10, (d, d))
        out.append(("negative%d" % n, neg))
        z = rng.uniform(0, 20, (d, d))
        z[:, 0] = 0.0  # FUEL's open tour
        out.append(("col0zero%d" % n, z))
        # products that truncate across an integer, both signs: 0.29 * 100 = 28.999999999999996
        t = rng.choice([0.29, 0.57, -0.29, -0.57, 1.15, 0.3, 0.58], size=(d, d))
        out.append(("truncate%d" % n, t))
        nd = rng.uniform(0, 20, (d, d))
        np.fill_diagonal(nd, np.nan)
        out.append(("nandiag%d" % n, nd))
    return out


@pytest.mark.parametrize("name,mat", _cases(), ids=[c[0] for c in _cases()])
def test_oracle_matches_brute_force(name, mat):
    st, cost, nopt, idx = OG.global_tour(mat)
    want = brute(mat)
    assert st == OG.GTOUR_OK and want is not None
    assert (cost, nopt, idx.tolist()) == want


def test_truncation_is_the_references():
    # int(0.29 * 100) == 28 in C++, not 29
    assert OG.int_matrix([[0.29, -0.29]]).tolist() == [[28, -28]]
    mat = np.array([[0.0, 0.29, 0.3], [0.0, 0.0, 0.0], [0.0, 0.0, 0.0]])
    st, cost, nopt, idx = OG.global_tour(mat)
    assert (st, cost, nopt, idx.tolist()) == (OG.GTOUR_OK, 28, 1, [0, 1])


@pytest.mark.parametrize("bad", [np.nan, np.inf, -np.inf, 3e7, -3e7, 21474836.48])
def test_bad_input(bad):
    mat = np.ones((4, 4))
    mat[2, 1] = bad
    assert OG.global_tour(mat)[0] == OG.GTOUR_BAD_INPUT
    assert brute(mat) is None


def test_int32_edges_are_kept():
    mat = np.ones((3, 3))
    mat[0, 1] = 21474836.47  # 2147483647 after truncation
    mat[0, 2] = -21474836.48  # -2147483648
    st, cost, nopt, idx = OG.global_tour(mat)
    assert st == OG.GTOUR_OK and (cost, nopt, idx.tolist()) == brute(mat)


def test_saturating_count_and_size_limit():
    st, cost, nopt, idx = OG.global_tour(np.zeros((14, 14)))  # 13! = 6 227 020 800 optimal tours
    assert (st, cost, nopt, idx.tolist()) == (OG.GTOUR_OK, 0, 2 ** 31 - 1, list(range(13)))
    st, cost, nopt, idx = OG.global_tour(np.zeros((12, 12)))  # 11! = 39 916 800
    assert nopt == 39916800
    info, ind = OG.global_tour_batch([3, 22, 2], np.concatenate([np.ones(9), np.ones(22 * 22), np.ones(4)]))
    assert info["status"].tolist() == [OG.GTOUR_OK, OG.GTOUR_TOO_LARGE, OG.GTOUR_OK]
    assert info["n"].tolist() == [2, 21, 1]
    assert ind[2:23].tolist() == [-1] * 21 and ind[23] == 0


def test_layout_and_binding(tmp_path):
    from fuel_b200 import _lib
    from fuel_b200 import exploration_manager as EM
    prog = tmp_path / "layout.c"
    prog.write_text('''
#include <stdio.h>
#include <stddef.h>
#include "fuelgpu.h"
int main(void) {
  printf("%zu %zu %zu %zu %zu %zu %d\\n", sizeof(FuelGlobalTourInfo), offsetof(FuelGlobalTourInfo, status),
         offsetof(FuelGlobalTourInfo, n), offsetof(FuelGlobalTourInfo, n_optimal),
         offsetof(FuelGlobalTourInfo, reserved), offsetof(FuelGlobalTourInfo, cost), FUELGPU_GTOUR_MAX_CLUSTERS);
  printf("%d %d %d\\n", FUELGPU_GTOUR_OK, FUELGPU_GTOUR_BAD_INPUT, FUELGPU_GTOUR_TOO_LARGE);
  return 0;
}''')
    exe = tmp_path / "layout"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(prog), "-o", str(exe)])
    got = [int(v) for v in subprocess.check_output([str(exe)]).decode().split()]
    for dt in (EM.GTOUR_INFO_DTYPE, OG.GTOUR_DTYPE):
        assert got[:7] == [dt.itemsize] + [dt.fields[f][1] for f in dt.names] + [EM.GTOUR_MAX_CLUSTERS]
    assert got[7:] == [EM.GTOUR_OK, EM.GTOUR_BAD_INPUT, EM.GTOUR_TOO_LARGE]
    assert OG.GTOUR_MAX_CLUSTERS == EM.GTOUR_MAX_CLUSTERS
    for name in ("fuelgpu_global_tour_batch", "fuelgpu_global_tour_batch_dev"):
        res, args = _lib.SIGNATURES[name]
        assert res is C.c_int and len(args) == 6


# ---- pinned on the reference's own findGlobalTour with its real LKH ------------------------------------------------
import json  # noqa: E402

import oracle.view as OV  # noqa: E402
from fuel_b200 import workloads as W  # noqa: E402
from tests.refgold import RECORD, digest  # noqa: E402
from tests.test_oracle_astar import Scene  # noqa: E402

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "refpin_gtour.json")
VM, YD, W_DIR = 2.0, 60 * 3.1415926 / 180.0, 1.5  # algorithm.xml:95-99
PRM = (VM, YD, W_DIR, 0.4, 10000.0, 100000, 400)  # vm, yd, w_dir, resolution, lambda_heu, allocate_num, max_iter


def _instances(g, inflate, tri):
    """(name, n, kind, seed): the frontier lists findGlobalTour is given.  Viewpoints are free positions of the office
    map; the clusters' costs_ rows are workloads.make_global_tours' matrices ("geometric": distance / vm and yaw
    change / yd with the 1000 of a failed search; "random": integer-valued costs with far outliers); row 0 is
    getFullCostMatrix's own computeCost from the current state."""
    out = [("geometric%d_%d" % (n, s), n, "geometric", s) for n in (2, 4, 6, 8, 10, 12, 14, 16, 18, 20) for s in (1, 2)]
    out += [("random%d" % n, n, "random", 50 + n) for n in range(2, 21)]
    return out


def _problem(g, inflate, tri, n, kind, seed):
    q = W.make_path_queries(g, inflate, tri, B=n + 1, seed=seed)
    vp = q["start"][1:]
    pos = q["start"][0]
    rng = np.random.default_rng(seed)
    vy = rng.uniform(-np.pi, np.pi, n)
    costs = W.make_global_tours(n, seed=seed, kind=kind)[0][1:, 1:]
    paths = [[np.zeros((0, 3)) if i == j else np.stack([vp[i], vp[j]]) for j in range(n)] for i in range(n)]
    vel = np.array([0.4, -0.2, 0.0]) if seed % 2 else np.zeros(3)
    return vp, vy, costs, paths, pos, vel, np.array([rng.uniform(-np.pi, np.pi), 0.0, 0.0])


def _oracle_side(om, vp, vy, costs, paths, pos, vel, yaw):
    """getFullCostMatrix over the view-cost oracle (pinned to the reference's computeCost by test_oracle_view_cost),
    and getPathForTour of a tour from the oracle's searchPath and the stored paths"""
    n = len(vy)
    info, path = OV.view_cost_batch(om, np.repeat(pos[None], n, 0), vp, np.full(n, yaw[0]), vy,
                                    np.repeat(vel[None], n, 0), *PRM, path_max=4096)
    mat = np.zeros((n + 1, n + 1))
    mat[1:, 1:] = costs
    mat[0, 1:] = info["cost"]

    def tour_of(ids):
        first = path[ids[0], :info["n_path"][ids[0]]]
        return np.concatenate([first] + [paths[a][b] for a, b in zip(ids[:-1], ids[1:])]).reshape(-1, 3)
    return mat, tour_of


@pytest.fixture(scope="module")
def office_ref():
    g, inflate = W.office_map()
    tri = W.office_known(g, inflate)
    s = Scene(g, inflate, tri)
    yield g, inflate, tri, s
    s.close()


def test_oracle_against_reference_lkh(office_ref):
    """The reference's findGlobalTour (TSPLIB file, LKH with its parameter file, the tour parse, getPathForTour) on
    each instance: its matrix equals the oracle side's bit for bit; the oracle's cost is never above LKH's on the same
    integer matrix; where the optimum is unique and LKH reached it, the tours are identical; and where the tours are
    identical, so are the global tours.  Where the reference is not built, tests/golden/refpin_gtour.json holds LKH's
    tours and the digests of the reference's matrices and global tours."""
    g, inflate, tri, s = office_ref
    live = OG.ref_gtour() is not None and s.ref is not None
    stored = json.load(open(GOLD)) if os.path.exists(GOLD) else {}
    recorded = {}
    rg = OG.RefGTour(s.ref, *PRM[:3], *PRM[4:]) if live else None
    at_opt = unique = same = 0
    insts = _instances(g, inflate, tri)
    try:
        for name, n, kind, seed in insts:
            vp, vy, costs, paths, pos, vel, yaw = _problem(g, inflate, tri, n, kind, seed)
            mat, tour_of = _oracle_side(s.om, vp, vy, costs, paths, pos, vel, yaw)
            if live:
                lkh, ref_tour, ref_mat = rg.find(vp, vy, costs, paths, pos, vel, yaw)
                assert np.array_equal(ref_mat, mat), name
                recorded[name] = dict(lkh=lkh, mat=digest(ref_mat), tour=digest(ref_tour))
                if not RECORD:
                    assert stored.get(name) == recorded[name], "%s: %s is out of date (FUEL_REFPIN_RECORD=1)" % (
                        name, GOLD)
            else:
                assert name in stored, "%s: no stored reference result in %s" % (name, GOLD)
                assert digest(mat) == stored[name]["mat"], name
                lkh, ref_tour = stored[name]["lkh"], None
            assert sorted(lkh) == list(range(n)), name
            st, cost, nopt, idx = OG.global_tour(mat)
            assert st == OG.GTOUR_OK
            c = OG.int_matrix(mat)
            lkh_cost = OG.tour_cost(c, lkh)
            assert cost == OG.tour_cost(c, idx) <= lkh_cost, name
            at_opt += lkh_cost == cost
            if nopt == 1:
                unique += 1
                if lkh_cost == cost:
                    assert idx.tolist() == lkh, name
            if idx.tolist() == lkh:
                same += 1
                got = tour_of(idx.tolist())
                if live:
                    assert np.array_equal(got, ref_tour), name
                    assert np.array_equal(rg.path(pos, idx), ref_tour), name
                else:
                    assert digest(got) == stored[name]["tour"], name
    finally:
        if rg is not None:
            rg.close()
    print("\nLKH at the optimum on %d of %d instances (%d with a unique optimum; tours identical on %d)"
          % (at_opt, len(insts), unique, same))
    if live and RECORD:
        with open(GOLD, "w") as f:
            json.dump(dict(sorted(recorded.items())), f, indent=0)
            f.write("\n")
