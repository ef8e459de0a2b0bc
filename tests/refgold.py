"""What the reference's own code computes, for the tests that pin the oracle to it.

Where the reference's library is built (oracle/_ref, from the reference's sources), the tests run the reference and
compare the oracle with it directly; every reference result is also checked against its SHA-256 digest in the module's
golden file under tests/golden/ (refpin.json unless the module names another), so the stored digests cannot drift from
the code they stand for.  Everywhere else the digests stand in for the reference: the oracle's result must hash to the
digest of the reference's.  Values are hashed as float64 arrays (shape included, -0.0 as 0.0, every NaN alike), so a
digest match is np.array_equal with NaN == NaN.

  FUEL_REFPIN_RECORD=1 python -m pytest tests/test_oracle_refpin.py tests/test_host_frontier_bookkeeping.py

rewrites the digests from a run against the built reference.
"""
import hashlib
import json
import math
import os

import numpy as np
import pytest

import oracle as O

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
RECORD = os.environ.get("FUEL_REFPIN_RECORD") == "1"


def _pieces(x):
    if isinstance(x, dict):
        for k in sorted(x):
            yield b"k" + str(k).encode()
            yield from _pieces(x[k])
    elif isinstance(x, (list, tuple)):
        yield b"l%d" % len(x)
        for v in x:
            yield from _pieces(v)
    else:
        a = np.asarray(x, dtype=np.float64) + 0.0
        a = np.where(np.isnan(a), np.nan, a)
        yield repr(a.shape).encode() + np.ascontiguousarray(a).tobytes()


def digest(x):
    h = hashlib.sha256()
    for p in _pieces(x):
        h.update(p)
    return h.hexdigest()


def first_difference(a, b, path=""):
    """where two results differ (for the message of a failed live comparison)"""
    if isinstance(a, dict) and isinstance(b, dict):
        if sorted(a) != sorted(b):
            return path + ": keys %s vs %s" % (sorted(a), sorted(b))
        for k in sorted(a):
            d = first_difference(a[k], b[k], "%s[%r]" % (path, k))
            if d:
                return d
        return None
    if isinstance(a, (list, tuple)) and isinstance(b, (list, tuple)):
        if len(a) != len(b):
            return path + ": length %d vs %d" % (len(a), len(b))
        for i, (u, v) in enumerate(zip(a, b)):
            d = first_difference(u, v, "%s[%d]" % (path, i))
            if d:
                return d
        return None
    if digest(a) == digest(b):
        return None
    u, v = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    if u.shape != v.shape:
        return path + ": shape %s vs %s" % (u.shape, v.shape)
    bad = ~((u == v) | (np.isnan(u) & np.isnan(v)))
    return path + ": %d of %d values differ, first at %s" % (int(bad.sum()), u.size, np.argwhere(bad)[0].tolist())


class RefGold:
    """One per test: eq(got, lambda: <the reference's value>) in the order the test makes its comparisons.  The digests
    are in tests/golden/<gold>; the reference runs where live() is not None."""

    def __init__(self, test_id, gold="refpin.json", live=O.ref_raycast):
        self.live = live() is not None
        self.test_id = test_id
        self.gold = os.path.join(GOLDEN, gold)
        self.count = 0
        self.stored = json.load(open(self.gold)) if os.path.exists(self.gold) else {}
        self.recorded = {}

    def eq(self, got, reference):
        key = "%s#%d" % (self.test_id, self.count)
        self.count += 1
        if self.live:
            want = reference()
            diff = first_difference(got, want)
            assert diff is None, "%s: oracle vs reference%s" % (key, diff)
            d = digest(want)
            self.recorded[key] = d
            if not RECORD:
                assert self.stored.get(key) == d, "%s: %s is out of date (FUEL_REFPIN_RECORD=1 rewrites it)" % (
                    key, self.gold)
        else:
            assert key in self.stored, "%s: no stored reference result in %s" % (key, self.gold)
            assert digest(got) == self.stored[key], "%s: the oracle no longer computes what the reference computed" % key

    def finish(self):
        if self.live and RECORD:
            d = json.load(open(self.gold)) if os.path.exists(self.gold) else {}
            d = {k: v for k, v in d.items() if not k.startswith(self.test_id + "#")}
            d.update(self.recorded)
            with open(self.gold, "w") as f:
                json.dump(dict(sorted(d.items())), f, indent=0)
                f.write("\n")


def refgold_fixture(gold="refpin.json", live=O.ref_raycast):
    """The per-test fixture G of a module whose digests are in tests/golden/<gold>, live where live() is not None:
    G = refgold_fixture(...) at the module's top level."""

    @pytest.fixture
    def G(request):
        g = RefGold("%s::%s" % (request.module.__name__.split(".")[-1], request.node.name), gold, live)
        yield g
        g.finish()

    return G


class MapGeometry:
    """SDFMap::initMap's geometry (sdf_map.cpp:33-39) and its three buffers, standing in for O.RefSDFMap where the
    reference is not built: what the tests read from the map object besides the reference's results."""

    def __init__(self, **params):
        self.res = float(params["resolution"])
        self.map_size = np.array([float(params["map_size_" + a]) for a in "xyz"])
        self.origin = np.array([-self.map_size[0] / 2.0, -self.map_size[1] / 2.0, float(params["ground_height"])])
        self.n = tuple(int(math.ceil(s / self.res)) for s in self.map_size)
        nv = int(np.prod(self.n))
        self.occupancy, self.inflate, self.distance = np.zeros(nv), np.zeros(nv, np.int8), np.zeros(nv)

    grid = O.RefSDFMap.grid

    def close(self):
        pass


def ref_map(**params):
    """The reference's SDFMap where it is built, else its geometry; either way the geometry is the reference's."""
    geo = MapGeometry(**params)
    if O.ref_raycast() is None:
        return geo
    ref = O.RefSDFMap(**params)
    assert ref.n == geo.n and np.array_equal(ref.origin, geo.origin) and ref.res == geo.res
    return ref
