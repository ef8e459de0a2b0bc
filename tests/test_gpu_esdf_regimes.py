"""Every launch regime of the ESDF tile kernels (esdf_tile.cu) against the oracle at the exact bar of
tests/esdf_exact.py.

The transform runs K0 `zpack_kernel` (z records), K1 the zy tile (a line = the box's y extent) and K2 the x tile (a
line = the box's x extent), per z chunk.  How each is launched depends on the box; the rules are restated below
(`tile_regime`, `chunk_plan`, `zpack_plan`) and the CPU test at the end asserts that the case list reaches every
regime they can produce, so that a change of a threshold in the kernel file shows up as a hole in coverage.
"""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from fuel_b200 import workloads as W
from tests.esdf_exact import check_esdf
from tests.helpers import make_sdf_map, orc_grid, random_scene

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TILE_SRC = os.path.join(ROOT, "fuel_b200", "csrc", "esdf_tile.cu")
RES = 0.1

# ---- the selection rules, restated (each snippet must still be in esdf_tile.cu) ---------------------------------
RULE_SNIPPETS = [
    # launch_tile (esdf_tile.cu:692-755): band width, band count, cluster split, thread count
    "const int logm = (p.n > 128 && g_band_log2 == 6 && (FROMBITS || p.piece_rows % 64 == 0)) ? 6 : 5;",
    "const int nb = (p.n + m - 1) / m;",
    "const bool cl = logm == 5 && nb > 16 && g_use_cluster && (FROMBITS || p.piece_rows % 32 == 0);",
    "p.nb = cl ? (nb + 1) / 2 : nb;",
    "FUEL_TILE_LAUNCH(5, 512, 3, true);",
    "if (nb <= 8)\n      FUEL_TILE_LAUNCH(5, 256, 6, false);\n    else if (nb <= 16)\n      FUEL_TILE_LAUNCH(5, 512, 3, false);\n"
    "    else\n      FUEL_TILE_LAUNCH(5, 1024, 1, false);",
    "if (nb <= 8)\n      FUEL_TILE_LAUNCH(6, 256, 3, false);\n    else\n      FUEL_TILE_LAUNCH(6, 512, 1, false);",
    # the chunk planner (esdf_tile.cu:40-43, 760-771, 796-805)
    "constexpr size_t P_ONE_CHUNK = (size_t)24 << 20;",
    "constexpr size_t P_CHUNK = (size_t)16 << 20;",
    "const size_t per_word = (size_t)nxb * nyb * 128;",
    "if (per_word * NW > P_ONE_CHUNK) {\n    Wc = (int)(P_CHUNK / per_word);\n    if (Wc < 1) Wc = 1;\n  }",
    "if (per_word * Wc > m->esdf_p_bytes) Wc = (int)(m->esdf_p_bytes / per_word);",
    "const int nchunks = (NW + Wc - 1) / Wc;",
    # the zpack path (esdf_tile.cu:198-213)
    "const bool vec = (nzb % 32 == 0) && (nz % 16 == 0) && (base0 % 16 == 0) && (chunk_stride % 16 == 0);",
    "while ((1 << l2) < NW) ++l2;",
]


def tile_regime(n, band64=False, cluster=True):
    """launch_tile for a line of n samples (K1 FROMBITS; K2 reads P in one piece, piece_rows = 2^20, so the
    piece conditions hold for both): (band log2, threads per CTA, 2-CTA cluster, shape of the band list)."""
    logm = 6 if (n > 128 and band64) else 5
    m = 1 << logm
    nb = (n + m - 1) // m
    cl = logm == 5 and nb > 16 and cluster
    nbc = (nb + 1) // 2 if cl else nb
    if cl:
        maxt = 512
    elif logm == 5:
        maxt = 256 if nb <= 8 else 512 if nb <= 16 else 1024
    else:
        maxt = 256 if nb <= 8 else 512
    tail = n - (nb - 1) * m  # samples in the last band
    return dict(logm=logm, maxt=maxt, cl=cl, nb=nb, threads=nbc * 32, tail=tail, phantom=cl and 2 * nbc > nb)


def tile_features(n, band64=False, cluster=True):
    """The regimes a line of n samples runs into: the launch config, whether its band count is the least or the
    largest of that config, the last band (one sample / partial / full), a phantom band in CTA 1."""
    r = tile_regime(n, band64, cluster)
    cfg = (r["logm"], r["maxt"], r["cl"])
    lo, hi = _cfg_range(band64, cluster)[cfg]
    f = {("cfg",) + cfg, ("tail", cfg, "one" if r["tail"] == 1 else "full" if r["tail"] == 1 << r["logm"] else "partial")}
    if r["nb"] == lo:
        f.add(("least bands", cfg))
    if r["nb"] == hi:
        f.add(("most bands", cfg))
    if r["cl"]:
        f.add(("phantom band", r["phantom"]))
    return f


_CFG_CACHE = {}


def _cfg_range(band64, cluster):
    key = (band64, cluster)
    if key not in _CFG_CACHE:
        rng = {}
        for n in range(1, 1025):
            r = tile_regime(n, band64, cluster)
            cfg = (r["logm"], r["maxt"], r["cl"])
            lo, hi = rng.get(cfg, (r["nb"], r["nb"]))
            rng[cfg] = (min(lo, r["nb"]), max(hi, r["nb"]))
        _CFG_CACHE[key] = rng
    return _CFG_CACHE[key]


def chunk_plan(shape, lo, hi):
    """esdf_tile_scratch_sizes (map) + esdf_tile_transform (box): words per chunk, chunk count, clamp."""
    def wc_of(nx, ny, nw):
        per_word = nx * ny * 128
        w = nw
        if per_word * nw > 24 << 20:
            w = max(1, (16 << 20) // per_word)
        return per_word, w
    pw_map, w_map = wc_of(shape[0], shape[1], (shape[2] + 31) // 32)
    p_bytes = pw_map * w_map
    nxb, nyb, nzb = (hi[i] - lo[i] + 1 for i in range(3))
    NW = (nzb + 31) // 32
    per_word, Wc = wc_of(nxb, nyb, NW)
    clamp = per_word * Wc > p_bytes
    if clamp:
        Wc = p_bytes // per_word
    nchunks = (NW + Wc - 1) // Wc
    return dict(Wc=Wc, nchunks=nchunks, clamp=clamp, last=NW - (nchunks - 1) * Wc, NW=NW)


def chunk_features(shape, lo, hi):
    c = chunk_plan(shape, lo, hi)
    f = {("chunks", "one" if c["nchunks"] == 1 else "Wc=1" if c["Wc"] == 1 else "Wc>1")}
    if c["nchunks"] > 1 and c["last"] < c["Wc"]:
        f.add(("chunks", "short last chunk"))
    if c["clamp"]:
        f.add(("chunks", "clamped to the map's scratch"))
    return f


def zpack_plan(shape, lo, hi):
    nzb = hi[2] - lo[2] + 1
    base0 = (lo[0] * shape[1] + lo[1]) * shape[2] + lo[2]
    vec = nzb % 32 == 0 and shape[2] % 16 == 0 and base0 % 16 == 0
    NW = (nzb + 31) // 32
    l2 = 0
    while (1 << l2) < NW:
        l2 += 1
    return ("zpack vec", l2) if vec else ("zpack ballot", "partial word" if nzb % 32 else "whole words")


REQUIRED_ZPACK = {("zpack vec", l2) for l2 in range(6)} | {("zpack ballot", "partial word"),
                                                           ("zpack ballot", "whole words")}
REQUIRED_CHUNKS = {("chunks", "one"), ("chunks", "Wc=1"), ("chunks", "Wc>1"), ("chunks", "short last chunk"),
                   ("chunks", "clamped to the map's scratch")}
LINE_N = [1, 31, 33, 256, 257, 512, 513, 544, 545, 1023, 1024]


# ---- the cases --------------------------------------------------------------------------------------------------
def offset_box(shape):
    """A box off the map origin in all three axes whose z-hi ends inside a word (and whose z-lo is unaligned)."""
    lo = [min(7, s // 5) for s in shape]
    hi = [s - 1 - min(5, s // 7) for s in shape]
    if (hi[2] - lo[2] + 1) % 32 == 0:
        hi[2] -= 1
    return lo, hi


def C(cid, shape, pattern, seed, modes=("opt",), boxes=("full", "offset"), line=True):
    return dict(id=cid, shape=tuple(shape), pattern=pattern, seed=seed, modes=modes, boxes=boxes, line=line)


CASES = [
    # lines of 1..1024 samples as K2 (x extent) and K1 (y extent); z layouts 32..1024
    C("x1-y1024", (1, 1024, 416), "far_boundary", 1),
    C("x1024-y1", (1024, 1, 413), "far_cta1", 2),
    C("x31-y1023", (31, 1023, 96), "sparse", 3),
    C("x1023-y31", (1023, 31, 160), "floor", 4),
    C("x33-y545", (33, 545, 33), "planes", 5),
    C("x545-y33", (545, 33, 96), "sparse", 6),
    C("x256-y544", (256, 544, 33), "far_cta1", 7),
    C("x544-y256", (544, 256, 32), "floor", 8),
    C("x257-y513", (257, 513, 64), "blocks", 9, modes=("opt", "nonopt", "signed")),
    C("x513-y257", (513, 257, 33), "far_boundary", 10),
    C("x512-y512", (512, 512, 40), "sparse", 11),
    C("x33-y31-z544", (33, 31, 544), "all", 12),
    C("x31-y33-z1024", (31, 33, 1024), "planes", 13),
    C("x129-y192", (129, 192, 33), "sparse", 18),  # the fewest 64-sample bands (FUELGPU_ESDF_BAND=64)
    # z chunks: 8 + 5 words; a partial last word inside the partial chunk; exactly 24 MiB; two chunks of 2 words
    C("chunk8+5", (128, 128, 416), "blocks", 14, modes=("opt", "nonopt", "signed"),
      boxes=("full", "offset", "clamp", "clamp_unaligned", "vec_offset"), line=False),
    C("chunk8+5-z413", (128, 128, 413), "sparse", 15, line=False),
    C("one-chunk-24MiB", (256, 256, 96), "floor", 16, line=False),
    C("chunks2x2", (256, 256, 97), "sparse", 17, line=False),
]


def case_box(case, name):
    s = case["shape"]
    if name == "full":
        return [0, 0, 0], [v - 1 for v in s]
    if name == "offset":
        return offset_box(s)
    if name == "clamp":  # z 0..383 of a 416 map: the box's P fits 24 MiB, the map's scratch does not
        return [0, 0, 0], [s[0] - 1, s[1] - 1, 383]
    if name == "clamp_unaligned":  # the same with an unaligned z-lo: whole words, but zpack takes the ballot path
        return [0, 0, 8], [s[0] - 1, s[1] - 1, 391]
    if name == "vec_offset":  # offset in x and y, z on a 16-byte boundary: the 16-byte path with a box
        return [5, 7, 32], [s[0] - 3, s[1] - 2, 32 + 352 - 1]
    raise KeyError(name)


def far_sites(shape, pattern):
    """Two or three sites far apart: opposite corners plus sites on the cluster split rows of the lines, or sites
    only in the half of the lines that CTA 1 of a 2-CTA cluster holds."""
    sites = []
    nx, ny, nz = shape
    def split(n):  # first row of CTA 1 when a line of n samples is a cluster tile, else the middle
        r = tile_regime(n)
        return (r["threads"] // 32) * 32 if r["cl"] else n // 2
    if pattern == "far_boundary":
        sites = [(0, 0, 0), (nx - 1, ny - 1, nz - 1),
                 (max(0, split(nx) - 1), max(0, split(ny) - 1), nz // 3), (min(nx - 1, split(nx)), min(ny - 1, split(ny)), nz // 2)]
    else:  # far_cta1, inside the offset box too
        sx, sy = split(nx), split(ny)
        (_, _, z0), (x1, y1, z1) = offset_box(shape)
        sites = [(x1, y1, z1), (min(x1, sx), min(y1, sy), z0), (min(x1, sx + 7), y1, nz // 2)]
    return sites


def make_scene(case):
    n, seed, pat = case["shape"], case["seed"], case["pattern"]
    rng = np.random.default_rng(seed)
    tri = np.full(n, W.FREE, dtype=np.uint8)
    inflate = np.zeros(n, dtype=np.int8)
    if pat == "sparse":
        inflate, tri = random_scene(n, seed, p_site=0.002, p_unknown=0.2, blobs=4)
    elif pat == "floor":
        inflate[:, :, n[2] // 3] = 1
        tri[:, :, : n[2] // 5] = W.UNKNOWN
    elif pat == "planes":  # lines with no site next to lines with sites
        for x in range(0, n[0], 3):
            inflate[x] = rng.random(n[1:]) < 0.01
        tri[:, :, -4:] = W.UNKNOWN
    elif pat == "all":
        inflate[...] = 1
    elif pat in ("far_boundary", "far_cta1"):
        for s in far_sites(n, pat):
            inflate[s] = 1
    elif pat == "blocks":  # obstacles with an inside (signed mode), unknown blobs (non-optimistic mode)
        inflate, tri = random_scene(n, seed, p_site=0.0005, p_unknown=0.3, blobs=3)
        for _ in range(6):
            c = [rng.integers(0, max(1, s - 6)) for s in n]
            e = [rng.integers(1, min(s, 40) + 1) for s in n]
            inflate[c[0]:c[0] + e[0], c[1]:c[1] + e[1], c[2]:c[2] + e[2]] = 1
    else:
        raise KeyError(pat)
    tri[(inflate == 1) & (tri == W.FREE)] = W.OCCUPIED
    return inflate, tri


def case_regimes(case, box):
    lo, hi = case_box(case, box)
    return dict(K1=tile_regime(hi[1] - lo[1] + 1), K2=tile_regime(hi[0] - lo[0] + 1),
                chunks=chunk_plan(case["shape"], lo, hi), zpack=zpack_plan(case["shape"], lo, hi))


def run_case(fuel, orc, case, mode, threads=16, boxes=None):
    """Full box first (the field the box update starts from), then every box of the case: each against the
    oracle at the exact bar, voxels outside the box bit for bit unchanged.  -> statistics per box."""
    n = case["shape"]
    g = W.Grid(n, (0.3, -1.0, 0.0), RES)
    inflate, tri = make_scene(case)
    opt, sgn = mode != "nonopt", mode == "signed"
    m = make_sdf_map(fuel, g, inflate, tri, optimistic=opt, signed=sgn)
    og = orc_grid(orc, g)
    out = []
    try:
        full_lo, full_hi = case_box(case, "full")
        m.updateESDF3d()
        full = m.download().copy()
        ref_full = orc.update_esdf3d(og, inflate, tri, full_lo, full_hi, opt, sgn, threads=threads)
        for b in boxes or case["boxes"]:
            lo, hi = case_box(case, b)
            label = "%s/%s/%s" % (case["id"], mode, b)
            if b == "full":
                got, ref = full, ref_full
            else:
                m.local_bound_min_, m.local_bound_max_ = np.array(lo), np.array(hi)
                m.updateESDF3d()
                got = m.download().copy()
                ref = orc.update_esdf3d(og, inflate, tri, lo, hi, opt, sgn, dist=ref_full.copy(), threads=threads)
                outside = np.ones(n, dtype=bool)
                outside[lo[0]:hi[0] + 1, lo[1]:hi[1] + 1, lo[2]:hi[2] + 1] = False
                assert np.array_equal(got[outside].view(np.uint32), full[outside].view(np.uint32)), label
                m.local_bound_min_, m.local_bound_max_ = np.array(full_lo), np.array(full_hi)
                m.updateESDF3d()  # back to the full field the next box starts from
                assert np.array_equal(m.download().view(np.uint32), full.view(np.uint32)), label + ": not repeatable"
            st = check_esdf(got, ref, RES, box=(lo, hi), signed=sgn, label=label)
            rg = case_regimes(case, b)
            st.update(K1=rg["K1"], K2=rg["K2"], chunks=rg["chunks"], zpack=rg["zpack"])
            out.append(st)
    finally:
        m.close()
    return out


CASE_PARAMS = [pytest.param(c, md, id="%s-%s" % (c["id"], md)) for c in CASES for md in c["modes"]]


@pytest.mark.gpu
@pytest.mark.parametrize("case,mode", CASE_PARAMS)
def test_case(fuel, orc, case, mode):
    for st in run_case(fuel, orc, case, mode):
        print(json.dumps(dict(st, zpack=list(st["zpack"])), default=str))


# ---- the 1024 x 1024 x 32 map against a closed form ---------------------------------------------------------------
def closed_form_check(got, sites, label):
    """k = min over the sites of the squared voxel distance (int64), in slabs of x planes."""
    n = got.shape
    ys, zs = np.meshgrid(np.arange(n[1], dtype=np.int64), np.arange(n[2], dtype=np.int64), indexing="ij")
    stats = []
    for x0 in range(0, n[0], 64):
        xs = np.arange(x0, min(n[0], x0 + 64), dtype=np.int64)[:, None, None]
        k = None
        for s in sites:
            kk = (xs - s[0]) ** 2 + (ys[None] - s[1]) ** 2 + (zs[None] - s[2]) ** 2
            k = kk if k is None else np.minimum(k, kk)
        ref = RES * np.sqrt(k.astype(np.float64))
        stats.append(check_esdf(got[x0:x0 + 64], ref, RES, label=label, verbose=False))
    st = dict(label=label, n=sum(s["n"] for s in stats), max_ulp=max(s["max_ulp"] for s in stats),
              inseparable=sum(s["inseparable"] for s in stats))
    print(json.dumps(st))
    return st


@pytest.mark.gpu
def test_1024x1024_far_sites_closed_form(fuel):
    n = (1024, 1024, 32)
    g = W.Grid(n, (0, 0, 0), RES)
    for name, sites in [("corners+split rows", [(0, 0, 0), (1023, 1023, 31), (511, 511, 5), (512, 512, 20)]),
                        ("CTA 1 half only", [(1023, 1023, 31), (512, 700, 0), (900, 512, 16)])]:
        inflate = np.zeros(n, dtype=np.int8)
        for s in sites:
            inflate[s] = 1
        tri = np.full(n, W.FREE, dtype=np.uint8)
        m = make_sdf_map(fuel, g, inflate, tri, optimistic=True)
        m.updateESDF3d()
        got = m.download().copy()
        m.close()
        closed_form_check(got, sites, "1024x1024x32 " + name)


# ---- state and ordering on one map ----------------------------------------------------------------------------------
@pytest.mark.gpu
def test_state_and_ordering(fuel, orc):
    case = CASES[[c["id"] for c in CASES].index("chunk8+5")]
    n = case["shape"]
    g = W.Grid(n, (0.3, -1.0, 0.0), RES)
    inflate, tri = make_scene(case)
    og = orc_grid(orc, g)
    m = make_sdf_map(fuel, g, inflate, tri, optimistic=True)
    try:
        full_lo, full_hi = case_box(case, "full")
        ref_full = orc.update_esdf3d(og, inflate, tri, full_lo, full_hi, True, False, threads=16)
        # chunked update, then the queued download: equal to the blocking one bit for bit
        m.updateESDF3d()
        m.download(wait=False)
        m.synchronize()
        queued = m.distance_buffer_.copy()
        blocking = m.download().copy()
        assert np.array_equal(queued.view(np.uint32), blocking.view(np.uint32))
        check_esdf(blocking, ref_full, RES, label="state/full")
        d64 = m.download(dtype=np.float64).copy()
        want = np.where(np.isinf(blocking), RES * np.sqrt(np.finfo(np.float64).max), blocking.astype(np.float64))
        assert np.array_equal(d64.view(np.uint64), want.view(np.uint64))
        # the same update twice: identical bits
        m.updateESDF3d()
        assert np.array_equal(m.download().view(np.uint32), blocking.view(np.uint32))
        # box sequence large -> small -> large: the scratch of the small box is reused by the large one
        small = ([40, 30, 70], [90, 100, 140])
        large = case_box(case, "clamp")
        prev, ref_prev = blocking, ref_full
        for lo, hi in (large, small, large):
            m.local_bound_min_, m.local_bound_max_ = np.array(lo), np.array(hi)
            m.updateESDF3d()
            got = m.download().copy()
            ref = orc.update_esdf3d(og, inflate, tri, lo, hi, True, False, dist=ref_prev.copy(), threads=16)
            check_esdf(got, ref, RES, box=(lo, hi), label="state/box %s..%s" % (lo, hi))
            outside = np.ones(n, dtype=bool)
            outside[lo[0]:hi[0] + 1, lo[1]:hi[1] + 1, lo[2]:hi[2] + 1] = False
            assert np.array_equal(got[outside].view(np.uint32), prev[outside].view(np.uint32))
            prev, ref_prev = got, ref
        # a signed update after the unsigned ones: the negative field is allocated on first use
        m.local_bound_min_, m.local_bound_max_ = np.array(full_lo), np.array(full_hi)
        m.signed_dist_ = True
        m.updateESDF3d()
        got = m.download().copy()
        ref = orc.update_esdf3d(og, inflate, tri, full_lo, full_hi, True, True, threads=16)
        check_esdf(got, ref, RES, signed=True, label="state/signed after unsigned")
    finally:
        m.close()


# ---- the non-default forms: 64-sample bands, long lines without clusters --------------------------------------------
def long_cases():
    """The line cases with a K1 or K2 line of 129..1024 samples (the lines the two forms change)."""
    return [c for c in CASES if c["line"] and any(129 <= v <= 1024 for v in c["shape"][:2])]


@pytest.mark.gpu
@pytest.mark.parametrize("env", [{"FUELGPU_ESDF_BAND": "64"}, {"FUELGPU_ESDF_CLUSTER": "0"}],
                         ids=["band64", "no-cluster"])
def test_non_default_forms(fuel, orc, env):
    """The form variables are read once per process: each form runs the long-line cases in a process of its own."""
    e = dict(os.environ, **env)
    e["PYTHONPATH"] = ROOT + os.pathsep + e.get("PYTHONPATH", "")
    r = subprocess.run([sys.executable, "-s", "-m", "tests.test_gpu_esdf_regimes"], cwd=ROOT, env=e,
                       capture_output=True, text=True, timeout=900)
    print(r.stdout[-20000:])
    assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-4000:]
    assert r.stdout.count('"label"') >= sum(len(c["boxes"]) for c in long_cases())


# ---- CPU: the case list reaches every regime ------------------------------------------------------------------------
def test_rules_restated_from_the_kernel_file():
    with open(TILE_SRC) as f:
        src = f.read()
    for s in RULE_SNIPPETS:
        assert s in src, "selection rule changed in esdf_tile.cu; restate it here: %r" % s


def _line_features(cases, band64=False, cluster=True):
    got = {"K1": set(), "K2": set()}
    for c in cases:
        for b in c["boxes"]:
            lo, hi = case_box(c, b)
            got["K1"] |= tile_features(hi[1] - lo[1] + 1, band64, cluster)
            got["K2"] |= tile_features(hi[0] - lo[0] + 1, band64, cluster)
    return got


@pytest.mark.parametrize("band64,cluster,nmin", [(False, True, 1), (True, True, 129), (False, False, 129)],
                         ids=["default", "band64", "no-cluster"])
def test_cases_reach_every_tile_regime(band64, cluster, nmin):
    cases = CASES if nmin == 1 else long_cases()
    required = set()
    for n in range(nmin, 1025):
        required |= tile_features(n, band64, cluster)
    got = _line_features(cases, band64, cluster)
    for k in ("K1", "K2"):
        assert required <= got[k], "%s misses %s" % (k, sorted(required - got[k], key=str))


def test_cases_reach_every_line_length():
    for k, ax in (("K1", 1), ("K2", 0)):
        lens = {c["shape"][ax] for c in CASES}
        assert set(LINE_N) <= lens, (k, sorted(set(LINE_N) - lens))
    assert {33, 96, 160, 413, 416} <= {c["shape"][2] for c in CASES}


def test_cases_reach_every_chunk_and_zpack_regime():
    got = set()
    for c in CASES:
        for b in c["boxes"]:
            lo, hi = case_box(c, b)
            got |= chunk_features(c["shape"], lo, hi)
            got.add(zpack_plan(c["shape"], lo, hi))
    assert REQUIRED_CHUNKS | REQUIRED_ZPACK <= got, sorted((REQUIRED_CHUNKS | REQUIRED_ZPACK) - got, key=str)
    p = chunk_plan((128, 128, 416), [0, 0, 0], [127, 127, 415])
    assert (p["Wc"], p["nchunks"], p["last"]) == (8, 2, 5)
    p = chunk_plan((128, 128, 416), [0, 0, 0], [127, 127, 383])
    assert p["clamp"] and (p["Wc"], p["nchunks"]) == (8, 2)
    assert chunk_plan((256, 256, 96), [0, 0, 0], [255, 255, 95])["nchunks"] == 1
    p = chunk_plan((256, 256, 97), [0, 0, 0], [255, 255, 96])
    assert (p["Wc"], p["nchunks"]) == (2, 2)


def test_modes_on_cluster_chunked_and_offset_shapes():
    for c in CASES:
        if "signed" in c["modes"]:
            assert "nonopt" in c["modes"] and "offset" in c["boxes"]
    sig = [c for c in CASES if "signed" in c["modes"]]
    assert any(tile_regime(c["shape"][1])["cl"] or tile_regime(c["shape"][0])["cl"] for c in sig)
    assert any(chunk_plan(c["shape"], *case_box(c, "full"))["nchunks"] > 1 for c in sig)


if __name__ == "__main__":
    # one process per non-default form (test_non_default_forms): the long-line cases, optimistic
    import fuel_b200
    import oracle
    fuel_b200.lib()
    oracle.lib()
    for c in long_cases():
        for st in run_case(fuel_b200, oracle, c, "opt"):
            print(json.dumps(dict(st, zpack=list(st["zpack"])), default=str), flush=True)
