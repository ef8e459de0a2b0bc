#!/usr/bin/env python
"""Device time of the mid-range branch's search (fuelgpu_kino_search_batch_dev: kinodynamicReplan's search, retry and
getSamples) at FUEL's parameters (fuel_b200.kino_astar.DEFAULTS, allocate_num 100 000) against the same searches on one
host thread through the reference's own kinodynamic_astar.cpp (oracle/_ref/libfuel_ref_kino.so, where build() made it;
else the oracle's GLIBC mode, which tests/test_oracle_kino_refpin.py pins on it bit for bit).  Queries: the MID rows of
office path queries (tests/kino_cases.mid_queries), tiled to B = 1024 with fresh start velocities and accelerations, and
B = 1 (the row of the batch that allocates the most nodes: one search's latency).  Device time: CUDA events around the
launch on the map's stream, inputs on the device, median over the repetitions after one call that grows the scratch.
Also the node counts the searches use.  One JSON line per batch, then a summary line with the card's name and power
limit."""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

import fuel_b200  # noqa: E402
import oracle as O  # noqa: E402
import oracle.kino as OK  # noqa: E402
from fuel_b200 import workloads as W  # noqa: E402
from fuel_b200._lib import MAX_PTS, lib  # noqa: E402
from fuel_b200.kino_astar import INFO_DTYPE, make_params  # noqa: E402
from tests.helpers import make_sdf_map  # noqa: E402
from tests.kino_cases import mid_queries  # noqa: E402
from tests.test_oracle_kino_refpin import Scene  # noqa: E402
from tools.solver_long import card  # noqa: E402


def device_ms(m, q, prm, reps):
    B = len(q["start"])
    t = {k: torch.tensor(q[k], device="cuda") for k in ("start", "vel", "acc", "goal")}
    info = torch.zeros(B * INFO_DTYPE.itemsize, dtype=torch.uint8, device="cuda")
    pts = torch.zeros((B, MAX_PTS - 2, 3), dtype=torch.float64, device="cuda")
    der = torch.zeros((B, 4, 3), dtype=torch.float64, device="cuda")
    dt = torch.zeros(B, dtype=torch.float64, device="cuda")
    stream = torch.cuda.Stream()
    m.set_stream(stream.cuda_stream)
    torch.cuda.synchronize()
    ms = []
    for r in range(reps + 1):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        rc = lib().fuelgpu_kino_search_batch_dev(m.handle, B, t["start"].data_ptr(), t["vel"].data_ptr(),
                                                 t["acc"].data_ptr(), t["goal"].data_ptr(), None, C.byref(prm),
                                                 info.data_ptr(), pts.data_ptr(), der.data_ptr(), dt.data_ptr(), 0,
                                                 None, None)
        e1.record(stream)
        assert rc == 0
        torch.cuda.synchronize()
        if r:
            ms.append(e0.elapsed_time(e1))
    m.set_stream(0)
    return float(np.median(ms)), np.frombuffer(info.cpu().numpy().tobytes(), dtype=INFO_DTYPE)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--cpu-queries", type=int, default=256, help="queries timed on the host (scaled to B)")
    a = ap.parse_args()
    fuel_b200.lib()
    dev = card()
    prm = make_params()
    g, inflate = W.office_map()
    tri = W.office_known(g, inflate)
    m = make_sdf_map(fuel_b200, g, inflate, tri)
    base = mid_queries(g, inflate, tri, B=1024, seed=20261019)
    n0 = len(base["start"])
    rng = np.random.default_rng(5)
    reps = -(-1024 // n0)
    big = {k: np.concatenate([base[k]] * reps)[:1024] for k in ("start", "goal")}
    big["vel"] = np.concatenate([base["vel"]] + [rng.uniform(-1.2, 1.2, (n0, 3)) * [1, 1, 0.3] for _ in range(reps - 1)])[:1024]
    big["acc"] = np.concatenate([base["acc"]] + [rng.uniform(-1, 1, (n0, 3)) for _ in range(reps - 1)])[:1024]
    _, info = device_ms(m, big, prm, 1)
    i = int(np.argmax(info["use_node_num"]))
    one = {k: v[i:i + 1] for k, v in big.items()}
    scene = Scene(g, inflate, tri)
    ref = OK.RefKino(scene.ref, prm) if scene.ref is not None else None
    for B, q in ((1, one), (1024, big)):
        ms, info = device_ms(m, q, prm, a.reps)
        n = min(B, a.cpu_queries)
        t = time.perf_counter()
        if ref is not None:
            ref.replan_batch(q["start"][:n], q["vel"][:n], q["acc"][:n], q["goal"][:n])
        else:
            OK.replan_batch(scene.om, g.map_max - g.origin, prm, q["start"][:n], q["vel"][:n], q["acc"][:n],
                            q["goal"][:n], math=OK.GLIBC)
        cpu_ms = (time.perf_counter() - t) * 1e3 * B / n
        u = info["use_node_num"]
        print(json.dumps(dict(map="office", B=B, allocate_num=prm.allocate_num, device_ms=round(ms, 3),
                              cpu_one_thread_ms=round(cpu_ms, 2),
                              cpu_side="reference kinodynamic_astar.cpp" if ref is not None else "oracle GLIBC mode",
                              use_node_num=dict(median=int(np.median(u)), p90=int(np.percentile(u, 90)), max=int(u.max())),
                              iter_num_max=int(info["iter_num"].max()), retried=int(info["retried"].sum()),
                              with_samples=int(np.sum(info["traj_status"] == 0)))), flush=True)
    if ref is not None:
        ref.close()
    scene.close()
    m.close()
    print(json.dumps(dict(summary="kino_search", **dev)), flush=True)


if __name__ == "__main__":
    main()
