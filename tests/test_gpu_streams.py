"""The map's streams.  A FuelMap runs the ESDF, fusion, inflation and the solver on its main stream, the frontier
search on a stream of its own, the async ESDF mirror on a copy stream and the solver's H2D on an input stream; the
order between them is kept with events.  The parity suites run each kernel alone and synchronize before they compare,
so these tests run the calls the way a planner overlaps them and check what comes out:

1. the step bench.py times (GpuPlanner, both issue orders): every output against the oracle, against the same planner
   run back to back, and the end-to-end arm against the resident one;
2. the MapROS replan cycle on a map that changes: fuse, inflate, search beside the ESDF and the solver, the next frame
   fused before the search is collected; overlapped and serial handles must agree byte for byte after every step;
3. every write that may follow a pending read on another stream: writers of the occupancy behind a pending frontier
   search, writers of the distance field behind a pending mirror download."""
import ctypes as C

import numpy as np
import pytest

from fuel_b200 import workloads as W
from fuel_b200._lib import check, lib, ptr
from tests.esdf_exact import check_esdf
from tests.helpers import make_sdf_map, orc_grid
from tests.test_gpu_frontier_device_csr import assert_bitwise, assert_oracle

pytestmark = pytest.mark.gpu

ORDERS = ["frontier_first", "solver_first"]
B_BENCH, EVALS = 1024, 64


def orc_consts(orc, tr, B):
    tcs = orc.traj_consts(B)
    for b in range(B):
        orc.fill_traj_const(tcs[b], tr["pt_dist"][b], tr["dt"][b], tr["start"][b], tr["end_pos"][b][None, :])
    return tcs


def occupancy(m):
    """(tri-state, inflate) bytes of the device's resident occupancy"""
    tri = np.empty(m.shape, np.uint8)
    inf = np.empty(m.shape, np.int8)
    check(lib().fuelgpu_map_download_occupancy(m.handle, ptr(inf), ptr(tri)), m.handle)
    return tri, inf


def assert_same_bytes(a, b, what):
    a, b = np.asarray(a), np.asarray(b)
    assert a.dtype == b.dtype and a.shape == b.shape, what
    if a.tobytes() != b.tobytes():
        raise AssertionError("%s differs in %d of %d elements" % (what, int(np.count_nonzero(a != b)), a.size))


def frontier_arrays(ftr):
    """the cluster list as flat arrays, in the layout of bench.dump_outputs"""
    return dict(cells=np.concatenate([f.cells_addr_ for f in ftr] + [np.zeros(0, np.int32)]),
                offsets=np.cumsum([0] + [len(f.cells_addr_) for f in ftr]))


# ---- 1. the step bench.py times --------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def bench_ref(orc):
    """The oracle's view of the benchmark's workload: the ESDF over the whole box (optimistic), one frontier search from
    clear flags over the whole map, and the solver's start cost."""
    import bench
    from fuel_b200.bspline_optimizer import BsplineOptimizer
    g, inflate, tri, tr = bench.build_workload(B_BENCH)
    og = orc_grid(orc, g)
    esdf = orc.update_esdf3d(og, inflate, tri, [0, 0, 0], np.array(g.n) - 1, True, False, threads=8)
    fl = np.zeros(g.n, dtype=np.int8)
    ftr = orc.frontier_search(og, tri, fl, g.origin, g.map_max, orc.frontier_params(cell_order=1))
    mask = BsplineOptimizer.NORMAL_PHASE | BsplineOptimizer.MINTIME
    to = orc_consts(orc, tr, B_BENCH)
    f0, _ = orc.combine_cost_batch(og, esdf, orc.opt_params(), to, 20, mask, W.pack_x(tr["ctrl"], tr["dt"]), threads=8)
    return dict(bench=bench, g=g, og=og, esdf=esdf, flags=fl, frontiers=ftr, mask=mask, to=to, f0=f0)


@pytest.fixture
def planners():
    """GpuPlanner's made by the test; the default stream is made current again and the maps are closed afterwards
    (the planner makes its own stream current)."""
    import torch
    made = []
    yield made
    torch.cuda.synchronize()
    torch.cuda.set_stream(torch.cuda.default_stream(0))
    for P in made:
        P.m.close()


def run_resident(bench, planners, overlap, out_dir, steps=3):
    import torch
    P = bench.GpuPlanner(0, B_BENCH, EVALS, overlap=overlap)
    planners.append(P)
    for _ in range(2 + steps):  # warmup, then the timed steps
        P.l2_flush()
        P.replan_resident()
    torch.cuda.set_stream(P.stream)  # dump_outputs reads the solver's tensors on the current stream
    bench.dump_outputs(P, str(out_dir))
    out = {k: np.load(str(out_dir / (k + ".npy"))) for k in
           ("esdf", "frontier_cells", "frontier_offsets", "frontier_average", "frontier_box_min", "frontier_box_max",
            "solver_x", "solver_cost", "solver_evals")}
    return P, out


@pytest.mark.parametrize("order", ORDERS)
def test_bench_step_matches_oracle_and_serial_step(orc, bench_ref, planners, tmp_path, monkeypatch, order):
    monkeypatch.setenv("FUELGPU_BENCH_ORDER", order)
    bench, g, R = bench_ref["bench"], bench_ref["g"], bench_ref
    P, out = run_resident(bench, planners, True, tmp_path / "overlap")
    assert P.solver_first == (order == "solver_first")

    # the ESDF, voxel for voxel
    check_esdf(out["esdf"], R["esdf"], g.res, label="bench step")
    # the frontier clusters: cells and offsets bit for bit, averages within 1e-12, boxes as the device-CSR suite
    ref = R["frontiers"]
    assert len(ref) > 0 and len(out["frontier_offsets"]) == len(ref) + 1
    assert np.array_equal(out["frontier_cells"], np.concatenate([r["addr"] for r in ref]).astype(np.float64))
    assert np.array_equal(out["frontier_offsets"], np.cumsum([0] + [len(r["addr"]) for r in ref]).astype(np.float64))
    assert_oracle(P.frontiers, ref)
    assert np.allclose(out["frontier_average"], np.array([r["average"] for r in ref]), rtol=1e-12, atol=1e-12)
    assert np.allclose(out["frontier_box_min"], np.array([r["box_min"] for r in ref]), rtol=0, atol=1e-12)
    assert np.allclose(out["frontier_box_max"], np.array([r["box_max"] for r in ref]), rtol=0, atol=1e-12)
    assert np.array_equal(P.ff.download_flags(), R["flags"])
    # the solver: the whole budget, inside the bounds, at a cost the oracle agrees with and no worse than the start
    x, f = out["solver_x"], out["solver_cost"]
    assert np.all(out["solver_evals"] == EVALS)
    pts = x[:, :60].reshape(B_BENCH, 20, 3)
    assert np.all(pts >= g.box_min + 0.1 - 1e-12) and np.all(pts <= g.box_max - 0.1 + 1e-12)
    assert np.all(x[:, -1] >= 0.0) and np.all(x[:, -1] <= 5.0)
    fchk, _ = orc.combine_cost_batch(R["og"], R["esdf"], orc.opt_params(), R["to"], 20, R["mask"], x, threads=8)
    assert np.all(np.abs(fchk - f) <= 1e-4 * np.abs(f) + 1e-9), np.max(np.abs(fchk - f) / np.abs(f))
    assert np.all(f <= R["f0"] * (1 + 1e-9))  # (the start cost on the device's fp32 field: last bits)

    # the same planner with its stages back to back: the overlap must not change a bit
    _, serial = run_resident(bench, planners, False, tmp_path / "serial")
    for k in out:
        assert_same_bytes(out[k], serial[k], "%s (overlapped vs back to back)" % k)

    # the end-to-end arm: host buffers in and out, the solver's input stream and the async mirror download
    import torch
    resident_frontiers = P.frontiers
    torch.cuda.set_stream(P.stream)
    for _ in range(2):
        ftr, f_e2e = P.replan_e2e()
        f_e2e = f_e2e.copy()
        assert_bitwise(ftr, resident_frontiers)
        assert_same_bytes(f_e2e, out["solver_cost"], "e2e solver cost vs the resident step")
        assert np.all(P.last_neval == EVALS)
        mirror = P.m.distance_buffer_.copy()
        assert_same_bytes(mirror, P.m.download(), "host mirror vs the device field")
        assert_same_bytes(mirror, out["esdf"], "host mirror vs the resident step's field")


# ---- 2. the replan cycle on a map that changes -------------------------------------------------------------------------
POSES = [((0.0, 0.0, 1.0), 0.0), ((0.3, 0.1, 1.0), 0.8), ((0.8, 0.4, 1.1), 1.7), ((1.0, 1.0, 1.2), 3.0),
         ((0.5, -0.6, 1.0), 4.4), ((-0.4, -0.2, 1.1), 5.6)]
B_CYCLE = 256


class Replanner:
    """One handle of the MapROS cycle: the map, its frontier finder and optimizer.  serial: synchronize() after every
    call, so nothing on one stream overlaps another."""

    def __init__(self, fuel, g, serial):
        self.m = fuel.SDFMap(g.n, g.res, g.origin, g.box_min, g.box_max)
        self.m.setFusionParams()
        env = fuel.EDTEnvironment()
        env.setMap(self.m)
        self.ff = fuel.FrontierFinder(env)
        self.opt = fuel.BsplineOptimizer()
        self.opt.setEnvironment(env)
        self.serial = serial
        self.frontiers = None
        self.solved = None

    def call(self, fn, *a, **kw):
        r = fn(*a, **kw)
        if self.serial:
            self.m.synchronize()
        return r

    def step(self, box, x, tcs, mask, next_frame, solver_first):
        m, ff, opt = self.m, self.ff, self.opt
        if not solver_first:
            self.call(ff.search_box_begin, *box)
        self.call(m.updateESDF3d)
        self.call(opt.optimizeBatchBegin, x, tcs, 20, mask, EVALS, xtol_rel=0.0, exact_evals=True)
        if solver_first:
            self.call(ff.search_box_begin, *box)
        self.call(m.download, wait=False)
        self.call(m.inputPointCloud, next_frame[0], next_frame[0].shape[0], next_frame[1])  # behind the pending search
        self.frontiers = self.call(ff.search_box_end)
        self.solved = tuple(a.copy() for a in self.call(opt.optimizeBatchEnd))
        m.synchronize()
        self.mirror = m.distance_buffer_.copy()

    def close(self):
        self.m.close()


@pytest.mark.parametrize("order", ORDERS)
def test_replan_cycle_overlapped_equals_serial(fuel, orc, order):
    g, truth = W.office_map()
    og = orc_grid(orc, g)
    fus = orc.Fusion(og, orc.fusion_params())
    inf_o = np.zeros(g.n, np.int8)
    fl_o = np.zeros(g.n, np.int8)
    fp = orc.frontier_params(cell_order=1)
    tr = W.make_trajectories(g, truth, B=B_CYCLE, n_pts=20, seed=31)
    mask = fuel.BsplineOptimizer.NORMAL_PHASE | fuel.BsplineOptimizer.MINTIME
    x0 = W.pack_x(tr["ctrl"], tr["dt"])
    tcs = fuel.BsplineOptimizer.traj_consts_from_arrays(tr["pt_dist"], tr["dt"], tr["start"], tr["end_pos"])
    frames = [(W.depth_frame(g, truth, np.array(c), yaw), np.array(c)) for c, yaw in POSES]
    A, S = Replanner(fuel, g, serial=False), Replanner(fuel, g, serial=True)
    try:
        for h in (A, S):
            h.m.inputPointCloud(frames[0][0], frames[0][0].shape[0], frames[0][1])
        fus.input_point_cloud(*frames[0])
        for k in range(len(POSES) - 1):
            lo, hi = S.m.local_bound_min_.copy(), S.m.local_bound_max_.copy()
            assert np.array_equal(A.m.local_bound_min_, lo) and np.array_equal(A.m.local_bound_max_, hi)
            boxes = []
            for h in (A, S):
                h.call(h.m.clearAndInflateLocalMap, obstacles_inflation=0.199)
                boxes.append(h.m.getUpdatedBox(reset=True))
            assert np.array_equal(np.concatenate(boxes[0]), np.concatenate(boxes[1]))
            for h in (A, S):
                h.step(boxes[0], x0, tcs, mask, frames[k + 1], order == "solver_first")

            # the overlapped handle is the serial one, byte for byte
            label = "step %d: " % k
            assert_same_bytes(A.m.getLogOdds(), S.m.getLogOdds(), label + "log-odds")
            for what, a, s in zip(("tri-state", "inflate"), occupancy(A.m), occupancy(S.m)):
                assert_same_bytes(a, s, label + what)
            assert_same_bytes(A.mirror, S.mirror, label + "ESDF host mirror")
            assert_same_bytes(A.m.download(), S.m.download(), label + "ESDF")
            assert_same_bytes(A.mirror, S.m.distance_buffer_, label + "host mirror vs the field")
            assert_bitwise(A.frontiers, S.frontiers)
            assert_same_bytes(A.ff.download_flags(), S.ff.download_flags(), label + "frontier_flag_")
            for what, a, s in zip(("x", "f", "n"), A.solved, S.solved):
                assert_same_bytes(a, s, label + "solver " + what)

            # the serial handle against the oracle chain (the frontier search ran before frame k + 1 was fused)
            tri_o = fus.tristate().reshape(g.n).copy()
            orc.clear_and_inflate(og, tri_o, inf_o, lo, hi, 2, -1)
            ref = orc.update_esdf3d(og, inf_o, tri_o, lo, hi, False, False)
            check_esdf(S.mirror, ref, g.res, box=(lo, hi), label=label)
            want = orc.frontier_search(og, tri_o, fl_o, boxes[0][0], boxes[0][1], fp)
            assert_oracle(S.frontiers, want)
            assert np.array_equal(S.ff.download_flags(), fl_o)
            fus.input_point_cloud(*frames[k + 1])
            assert np.array_equal(S.m.getLogOdds().reshape(-1), fus.logodds)
        assert sum(len(h.frontiers) for h in (A, S)) > 0
    finally:
        A.close()
        S.close()


# ---- 3. writes that follow a pending read on another stream ------------------------------------------------------------
OFFICE_CEIL_Z = 20  # z index of 1.0 m on the office map: inside the known region
HOLD_CYCLES = 200_000_000  # ~0.1 s of GPU clock: longer than any writer's host side


def office_logodds(tri, p_min=0.12, p_max=0.90):
    """log-odds whose tri-state is `tri` (unknown below clamp_min - 1e-3, occupied above min_occupancy_log)"""
    lg = lambda p: np.log(p / (1 - p))  # noqa: E731
    lo = np.full(tri.shape, lg(p_min), np.float64)
    lo[tri == W.UNKNOWN] = lg(p_min) - 0.01
    lo[tri == W.OCCUPIED] = lg(p_max)
    return lo


def occ_writers(g, truth, tri):
    """name -> (prepare, write, has_logodds).  prepare(m) runs on both maps before the search, so that the write itself
    grows no scratch (a growing block waits for the whole device); write(m) changes the occupancy of the searched box."""
    tri2 = W.known_region(g, truth, seed=8, n_poses=12, radius=2.5)
    cams = [np.array([0.0, 0.0, 1.0]), np.array([2.5, -1.0, 1.1])]
    frames = [W.depth_frame(g, truth, c, yaw) for c, yaw in zip(cams, (0.5, 2.4))]
    images = [W.depth_image(g, truth, c, yaw) for c, yaw in zip(cams, (0.5, 2.4))]

    def upload(wait):
        def write(m):
            m.occupancy_tri_[...] = tri2
            m.upload(wait=wait)
        return (lambda m: None), write, False

    import torch
    unknown_plane = torch.zeros(g.n[0] * g.n[1], dtype=torch.uint8, device="cuda")  # UNKNOWN, not inflated
    torch.cuda.synchronize()  # (here: a device-wide wait behind the pending search would hide a missing order)

    def plane(m):
        check(lib().fuelgpu_map_occupancy_plane_dev(m.handle, OFFICE_CEIL_Z, C.c_void_p(unknown_plane.data_ptr()), 1),
              m.handle)

    ceil_h = g.origin[2] + (OFFICE_CEIL_Z + 0.5) * g.res
    return {
        "upload": upload(True),
        "upload_async": upload(False),
        "inflate": ((lambda m: occupancy(m)),
                    (lambda m: m.clearAndInflateLocalMap(obstacles_inflation=0.199, virtual_ceil_height=ceil_h)), False),
        "input_point_cloud": ((lambda m: m.inputPointCloud(frames[0], frames[0].shape[0], cams[0])),
                              (lambda m: m.inputPointCloud(frames[1], frames[1].shape[0], cams[1])), True),
        "input_depth_image": ((lambda m: m.inputDepthImage(images[0][0], images[0][1], cams[0])),
                              (lambda m: m.inputDepthImage(images[1][0], images[1][1], cams[1])), True),
        "set_logodds": ((lambda m: m.setLogOdds(office_logodds(tri))), (lambda m: m.setLogOdds(office_logodds(tri2))),
                        True),
        "occupancy_plane_set": ((lambda m: None), plane, False),
    }


@pytest.mark.parametrize("writer", ["upload", "upload_async", "inflate", "input_point_cloud", "input_depth_image",
                                    "set_logodds", "occupancy_plane_set"])
def test_occupancy_write_behind_pending_search(fuel, writer):
    """search_begin (the small path's asynchronous cluster kernel), then a writer of `occ`, then search_end: the search
    sees the occupancy of the time it was issued, and the write lands as it does alone.  The search is issued behind
    ~0.1 s of other work on the caller's stream and the write from a second caller stream (fuelgpu_map_set_stream), so
    a write that did not wait for the search would land before the search reads the map, every time."""
    import torch
    g, truth = W.office_map()
    tri = W.office_known(g, truth)
    prepare, write, has_logodds = occ_writers(g, truth, tri)[writer]
    maps = [make_sdf_map(fuel, g, truth, tri) for _ in range(2)]
    hold, other = torch.cuda.Stream(), torch.cuda.Stream()
    try:
        finders = []
        for m in maps:
            m.setFusionParams()
            m.setCameraParams()
            prepare(m)
            m.synchronize()
            env = fuel.EDTEnvironment()
            env.setMap(m)
            ff = fuel.FrontierFinder(env)
            for _ in range(2):  # the first searches allocate the search's scratch (both result blocks)
                ff.search_box(g.origin, g.map_max)
                ff.reset_flags()
            finders.append(ff)
        (m1, ff1), (m2, ff2) = zip(maps, finders)
        before = occupancy(m1)

        m1.set_stream(hold.cuda_stream)
        with torch.cuda.stream(hold):
            torch.cuda._sleep(HOLD_CYCLES)
        ff1.search_box_begin(g.origin, g.map_max)  # the frontier stream waits for `hold`
        m1.set_stream(other.cuda_stream)
        write(m1)
        got = ff1.search_box_end()
        m1.synchronize()
        m1.set_stream(None)

        want = ff2.search_box(g.origin, g.map_max)  # on the occupancy before the write
        write(m2)
        m2.synchronize()

        assert len(want) > 0
        assert_bitwise(got, want)
        assert_same_bytes(ff1.download_flags(), ff2.download_flags(), "frontier_flag_")
        after = occupancy(m1)
        for what, a, b, b0 in zip(("tri-state", "inflate"), after, occupancy(m2), before):
            assert_same_bytes(a, b, what + " after the write")
        assert not np.array_equal(after[0], before[0]), "the write must change the searched tri-state"
        if has_logodds:
            assert_same_bytes(m1.getLogOdds(), m2.getLogOdds(), "log-odds after the write")
    finally:
        for m in maps:
            m.close()


MIRROR_N = (256, 256, 256)  # 64 MiB of float32: the D2H copy outlasts an update of the field by far


def mirror_scenes():
    """Two occupancies that differ only in x >= 128, the half of the field the mirror's copy reaches last."""
    rng = np.random.default_rng(17)
    inflate = (rng.random(MIRROR_N) < 0.02).astype(np.int8)
    inflate2 = inflate.copy()
    inflate2[128:] = (rng.random((128,) + MIRROR_N[1:]) < 0.005).astype(np.int8)
    tri = [np.where(i == 1, W.OCCUPIED, W.FREE).astype(np.uint8) for i in (inflate, inflate2)]
    return (inflate, tri[0]), (inflate2, tri[1])


@pytest.mark.parametrize("writer", ["update_esdf", "set_from_slabs_1", "set_from_slabs_2"])
def test_dist_write_behind_pending_mirror(fuel, writer):
    """A different occupancy uploaded, download(wait=False), then a writer of the distance field on the main stream
    (the ESDF update, or fuelgpu_esdf_set_from_slabs_dev from one slab or from the two-slab all-gather layout): after
    synchronize() the host mirror holds the first field, whole, and the device holds the second."""
    import torch
    g = W.Grid(MIRROR_N, (-12.8, -12.8, -1.0), 0.1)
    (inf1, tri1), (inf2, tri2) = mirror_scenes()
    hi_box = (np.array([128, 0, 0], np.int32), np.array(MIRROR_N, np.int32) - 1)

    # the fields, one call at a time on a handle of their own
    ref = make_sdf_map(fuel, g, inf1, tri1)
    try:
        ref.updateESDF3d()
        field1 = ref.download().copy()
        ref.occupancy_buffer_inflate_[...] = inf2
        ref.occupancy_tri_[...] = tri2
        ref.upload(*hi_box)
        ref.updateESDF3d()
        field2 = ref.download().copy()
    finally:
        ref.close()
    late = np.count_nonzero(field1[128:] != field2[128:])
    assert late > field1[128:].size // 4, late  # the copy's late half changes

    m = make_sdf_map(fuel, g, inf1, tri1)
    try:
        m.updateESDF3d()
        m.download()  # (sizes and page-locks the mirror)
        slabs = None
        if writer.startswith("set_from_slabs"):
            G = int(writer[-1])  # [G][nx][ny][nz/G]
            slabs = torch.from_numpy(np.ascontiguousarray(np.stack(np.split(field2, G, axis=2)))).to("cuda")
            torch.cuda.synchronize()
        # the next occupancy goes in first (it does not touch the field), so the write follows the copy at once
        m.occupancy_buffer_inflate_[...] = inf2
        m.occupancy_tri_[...] = tri2
        m.upload(*hi_box)
        m.download(wait=False)  # the field of the last update
        if writer == "update_esdf":
            m.updateESDF3d()
        else:
            check(lib().fuelgpu_esdf_set_from_slabs_dev(m.handle, C.c_void_p(slabs.data_ptr()), G), m.handle)
        m.synchronize()
        mirror = m.distance_buffer_.copy()
        assert_same_bytes(mirror, field1, "host mirror (the field when the download was issued)")
        assert_same_bytes(m.download(), field2, "device field after the write")
    finally:
        m.close()
