"""Kinodynamic-search queries shared by the oracle and GPU tests: the MID rows of the path search on the office maps
and hand-built cases at the search's edges."""
import numpy as np

import oracle.astar as OA
from fuel_b200 import workloads as W


def mid_queries(g, inflate, tri, B, seed):
    """the MID rows (1.5 m <= shortened path <= 5 m) of B path queries, searched by the A* oracle at FUEL's 0.4 m"""
    q = W.make_path_queries(g, inflate, tri, B=B, seed=seed)
    info = OA.search_batch(OA.Map(g, inflate, tri), q["start"], q["goal"], 0.4, 10000.0, 40000, 100000)[0]
    return W.make_kino_queries(g, inflate, tri, info, q["start"], q["goal"], seed=seed + 1)


def hand_cases(g, inflate, tri):
    """(start, vel, acc, goal) rows: a goal within 1e-2 of the start and one just outside, the velocity at the limit
    (max_vel + vel_margin) and beyond it, a goal beyond the horizon, goals inside occupied space, starts next to the
    exploration box's faces, close goals ahead of a fast start (the three-root branch)"""
    free = np.argwhere((np.asarray(tri) == W.FREE) & (np.asarray(inflate) == 0))
    pos = g.index_to_pos(free)
    inner = pos[np.all((pos > g.box_min + 0.3) & (pos < g.box_max - 0.3), axis=1)]
    rng = np.random.default_rng(7)
    s0 = inner[rng.integers(len(inner))] + 0.013
    occ = g.index_to_pos(np.argwhere(np.asarray(inflate) != 0))
    far = inner[np.argmax(np.linalg.norm(inner - s0, axis=1))]
    rows = [
        (s0, (0, 0, 0), (0, 0, 0), s0 + (0.005, 0.0, 0.0)),
        (s0, (0, 0, 0), (0, 0, 0), s0 + (0.011, 0.0, 0.0)),
        (s0, (0, 0, 0), (0, 0, 0), s0 + (0.3, 0.2, 0.0)),
        (s0, (2.25, 0, 0), (0, 0, 0), s0 + (2.0, 0.5, 0.0)),
        (s0, (-2.25, 2.25, 0), (1.0, -1.0, 0), s0 + (-2.0, 1.5, 0.2)),
        (s0, (2.3, 0, 0), (0, 0, 0), s0 + (2.0, 0.0, 0.0)),
        (s0, (0.5, 0.5, 0), (0, 0, 0), far),
        (s0, (0, 0, 0), (0, 0, 0), occ[np.argmin(np.linalg.norm(occ - s0, axis=1))]),
        (s0, (0, 0, 0), (0, 0, 0), occ[len(occ) // 2]),
    ]
    for ang in (0.3, 1.9, 3.5, 5.1):  # a close goal ahead of a fast start: cubic()'s three-real-root branch
        u = np.array([np.cos(ang), np.sin(ang), 0.0])
        rows.append((s0, 2.1 * u, (0, 0, 0), s0 + 0.3 * u))
    for k in range(3):  # next to the low and the high face of the box
        lo = inner[np.argmin(inner[:, k])].copy()
        hi = inner[np.argmax(inner[:, k])].copy()
        lo[k] = g.box_min[k] + 0.05
        hi[k] = g.box_max[k] - 0.05
        v = np.zeros(3)
        v[k] = -1.0
        rows.append((lo, v, (0, 0, 0), lo + np.eye(3)[k] * 2.0 + 0.1))
        rows.append((hi, -v, (0, 0, 0), hi - np.eye(3)[k] * 2.0 - 0.1))
    s, v, a, gl = (np.array([np.asarray(r[i], dtype=np.float64) for r in rows]) for i in range(4))
    return dict(start=s, vel=v, acc=a, goal=gl)
