#!/usr/bin/env python
"""Where one office replan (bench.py's metric step: office.pcd 200x120x40, B = 1024, K = 64) spends its time.

Prints, for one `replan_resident` each:
  * the device timeline of the overlapped step (`overlap=True`, as the metric runs it): every kernel, copy and memset
    on every stream, start and end in microseconds after the first device activity of the step (torch.profiler);
  * the same kernels with the stages back to back (`overlap=False`);
  * the host time of `fuelgpu_frontier_search_end` (the wait for the frontier stream plus the result hand-off) and
    of `FrontierFinder._fetch`, and of the whole `search_box_end`; in a FUEL_PROF build, `search_end` with the device
    idle split into the stream wait, the rest of `_end` (the host marshalling when the host orders the result) and
    the closing timing event;
  * in a FUEL_PROF build, the %globaltimer stamps of `cluster_small_kernel` (one per cluster.sync()), by phase.

FUELGPU_FRONTIER_HOST_CSR=1 times the host-ordered result instead of the device-ordered one.

  python tools/office_step.py [--reps 20] [--trace DIR]
"""
import argparse
import ctypes as C
import json
import os
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

import bench  # noqa: E402


def device_timeline(P, trace_dir=None, tag="overlap"):
    """Kernels / copies / memsets of one replan_resident (the last of three profiled ones), sorted by start."""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA, ProfilerActivity.CPU]) as prof:
        for _ in range(3):
            P.l2_flush()
            torch.cuda.synchronize()
            P.replan_resident()
            torch.cuda.synchronize()
    d = trace_dir or tempfile.mkdtemp()
    path = os.path.join(d, "office_step_%s.pt.trace.json" % tag)
    prof.export_chrome_trace(path)
    ev = json.load(open(path))["traceEvents"]
    if not trace_dir:
        os.remove(path)
    dev = [e for e in ev if e.get("ph") == "X" and e.get("cat") in ("kernel", "gpu_memcpy", "gpu_memset")]
    dev.sort(key=lambda e: e["ts"])
    # the step = the device work after the last flush (the flush is a memset / fill kernel of 256 MB)
    flush = [i for i, e in enumerate(dev) if e.get("dur", 0) > 20 and ("fill" in e["name"].lower() or
                                                                      e.get("cat") == "gpu_memset")]
    start = flush[-1] + 1 if flush else 0
    rows = dev[start:]
    t0 = rows[0]["ts"] if rows else 0.0
    out = []
    for e in rows:
        out.append((e.get("args", {}).get("stream", e.get("tid")), e["name"][:70], e["ts"] - t0, e["ts"] - t0 + e["dur"]))
    return out


def print_timeline(title, rows):
    print("== %s ==" % title)
    print("%6s %9s %9s %8s  %s" % ("stream", "start_us", "end_us", "dur_us", "name"))
    for s, n, a, b in rows:
        print("%6s %9.1f %9.1f %8.1f  %s" % (s, a, b, b - a, n))
    if rows:
        by = {}
        for s, n, a, b in rows:
            lo, hi = by.get(s, (a, b))
            by[s] = (min(lo, a), max(hi, b))
        print("per stream (first start, last end):", {k: (round(v[0], 1), round(v[1], 1)) for k, v in by.items()})
        print("device span %.1f us" % (max(r[3] for r in rows) - min(r[2] for r in rows)))


def host_times(P, reps):
    """Host time of search_box_end and its two halves, in the overlapped step (median of reps)."""
    L = P.fuel.lib()
    h = P.m.handle
    ff = P.ff
    t_end, t_fetch, t_all, t_step = [], [], [], []
    for _ in range(reps):
        P.l2_flush()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(P.stream)
        P._frontier_begin()
        P.m.updateESDF3d()
        P.d_xw.copy_(P.d_x, non_blocking=True)
        rc = L.fuelgpu_bspline_optimize_batch_dev(h, P.B, 20, P.mask, C.byref(P.opt.params_), C.c_void_p(P.d_tc.data_ptr()),
                                                  C.byref(P.sp), C.c_void_p(P.d_xw.data_ptr()),
                                                  C.c_void_p(P.d_f.data_ptr()), C.c_void_p(P.d_n.data_ptr()))
        assert rc == 0
        nc, ncell, nf = C.c_int32(), C.c_int32(), C.c_int32()
        a = time.perf_counter()
        L.fuelgpu_frontier_search_end(h, C.byref(nc), C.byref(ncell), C.byref(nf))
        b = time.perf_counter()
        ff._fetch(nc.value, ncell.value, nf.value)
        c = time.perf_counter()
        e1.record(P.stream)
        torch.cuda.synchronize()
        t_end.append(b - a)
        t_fetch.append(c - b)
        t_all.append(c - a)
        t_step.append(e0.elapsed_time(e1))
    med = lambda v: 1e6 * float(np.median(v))  # noqa: E731
    print("== host, overlapped step (median of %d) ==" % reps)
    print("fuelgpu_frontier_search_end %.1f us (wait for the frontier stream + marshalling), FrontierFinder._fetch %.1f us, "
          "together %.1f us; step %.1f us" % (med(t_end), med(t_fetch), med(t_all), 1e3 * float(np.median(t_step))))
    # the marshalling alone: the same calls once the frontier stream is known to be idle
    so = C.CDLL(P.fuel._lib.SO)
    split = hasattr(so, "fuelgpu_debug_frontier_end_prof")
    if split:
        so.fuelgpu_debug_frontier_end_prof.argtypes = [C.c_void_p, C.POINTER(C.c_double)]
    t_m, t_f, parts = [], [], []
    for _ in range(reps):
        P.l2_flush()
        P._frontier_begin()
        torch.cuda.synchronize()
        a = time.perf_counter()
        L.fuelgpu_frontier_search_end(h, C.byref(nc), C.byref(ncell), C.byref(nf))
        b = time.perf_counter()
        ff._fetch(nc.value, ncell.value, nf.value)
        c = time.perf_counter()
        t_m.append(b - a)
        t_f.append(c - b)
        if split:
            buf = (C.c_double * 3)()
            so.fuelgpu_debug_frontier_end_prof(h, buf)
            parts.append(list(buf))
    print("with the device idle: fuelgpu_frontier_search_end %.1f us, _fetch %.1f us (%d clusters, %d cells, %d filtered)"
          % (med(t_m), med(t_f), nc.value, ncell.value, nf.value))
    if split:
        p = np.median(np.array(parts), axis=0)
        print("  search_end split (FUEL_PROF steady clock, median): cudaStreamSynchronize %.1f us, result assembly %.1f us, "
              "tend %.1f us, rest (ABI entry, ctypes) %.1f us" % (p[0], p[1], p[2], med(t_m) - p.sum()))
    else:
        print("  (search_end split into stream wait / result assembly / tend: FUEL_PROF builds only)")


def prof_stamps(P):
    so = C.CDLL(P.fuel._lib.SO)
    if not hasattr(so, "fuelgpu_debug_frontier_prof"):
        print("== cluster_small_kernel stamps: not a FUEL_PROF build ==")
        return
    P.l2_flush()
    P._frontier_begin()
    P.ff.search_box_end()
    torch.cuda.synchronize()
    buf = (C.c_longlong * 256)()
    so.fuelgpu_debug_frontier_prof.argtypes = [C.c_void_p, C.POINTER(C.c_longlong), C.c_int]
    so.fuelgpu_debug_frontier_prof(P.m.handle, buf, 256)
    t = np.array(buf[:], dtype=np.int64)
    t = t[t > 0]
    head = ["init_parent", "union", "flatten", "claim", "assign", "mark", "chunk_scan", "gather+init_meta"]
    level = ["stat_accum", "mean+downsample", "cov", "pca", "side_count", "split_alloc", "relabel", "next_level"]
    names = list(head)
    # the last level stops after its relabel (no next_level stamp); a search whose result the kernel ordered ends with
    # the four phases of its tail
    tail = ["tail count+rank", "tail places", "tail scatter", "tail filtered"] if (len(t) - 1 - len(head)) % len(level) == 3 else []
    while len(names) < len(t) - 1 - len(tail):
        lv = (len(names) - len(head)) // len(level)
        names += ["L%d %s" % (lv, n) for n in level]
    names += tail
    d = np.diff(t) / 1e3
    print("== cluster_small_kernel: %d stamps, %.1f us from the first to the last ==" % (len(t), (t[-1] - t[0]) / 1e3))
    for n, v in zip(names, d):
        print("  %-26s %7.2f us" % (n, v))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--trace", default=None, help="keep the chrome traces in this directory")
    a = ap.parse_args()
    torch.cuda.set_device(0)
    pr = torch.cuda.get_device_properties(0)
    print("device:", pr.name)
    for overlap in (True, False):
        P = bench.GpuPlanner(0, 1024, 64, overlap=overlap)
        for _ in range(5):
            P.l2_flush()
            P.replan_resident()
        torch.cuda.synchronize()
        print_timeline("one replan_resident, overlap=%s" % overlap, device_timeline(P, a.trace, "overlap" if overlap else "serial"))
        if overlap:
            host_times(P, a.reps)
            prof_stamps(P)
        P.m.close()


if __name__ == "__main__":
    main()
