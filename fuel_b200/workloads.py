"""Deterministic workloads (BASELINE.md section 3) shared by tests/ and bench.py.

Inputs only; everything is derived from the committed fixtures in tests/golden/ (voxelised
reference .pcd maps, see tools/make_fixtures.py) or from seeded numpy PCG64 generators.
Nothing here touches /root/reference or the oracle.
"""
import os

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")

UNKNOWN, FREE, OCCUPIED = 0, 1, 2


class Grid:
    def __init__(self, voxel_num, origin, resolution=0.1, box_min=None, box_max=None):
        self.n = tuple(int(v) for v in voxel_num)
        self.origin = np.asarray(origin, dtype=np.float64)
        self.res = float(resolution)
        self.map_max = self.origin + np.asarray(self.n) * self.res
        self.box_min = self.origin.copy() if box_min is None else np.asarray(box_min, dtype=np.float64)
        self.box_max = self.map_max.copy() if box_max is None else np.asarray(box_max, dtype=np.float64)

    @property
    def nvox(self):
        return self.n[0] * self.n[1] * self.n[2]

    def pos_to_index(self, pos):
        return np.floor((np.asarray(pos, dtype=np.float64) - self.origin) * (1 / self.res)).astype(np.int64)

    def index_to_pos(self, idx):
        return (np.asarray(idx) + 0.5) * self.res + self.origin


def load_occupancy(name):
    """-> (Grid on the fixture's natural extents, inflate int8 [nx,ny,nz])."""
    d = np.load(os.path.join(GOLDEN, name + ".npz"))
    n = tuple(int(v) for v in d["voxel_num"])
    inflate = np.zeros(n[0] * n[1] * n[2], dtype=np.int8)
    inflate[d["addr"]] = 1
    return Grid(n, d["origin"], float(d["resolution"])), inflate.reshape(n)


def office_map(interior_box=True):
    """Config 1/2: office.pcd on 200x120x40 @0.1 m, origin (-10,-6,-1).  The exploration box
    is kept strictly inside the map (SURVEY H9), as the reference's launch files do."""
    g, inflate = load_occupancy("office_200x120x40")
    if interior_box:
        g = Grid(g.n, g.origin, g.res, box_min=(-9.0, -5.0, -0.8), box_max=(9.0, 5.0, 2.0))
    return g, inflate


def office3_map():
    """Config 5: office3.pcd on 200x300x40."""
    g, inflate = load_occupancy("office3_200x300x40")
    return Grid(g.n, g.origin, g.res, box_min=(-9.0, -14.0, -0.8), box_max=(9.0, 14.0, 2.0)), inflate


def pillar_map(variant="V1"):
    """Config 3: pillar.pcd on 512^3 @0.1 m, origin (-25.6,-25.6,-1).
    V0 = file as is (mostly empty cube); V1 = the occupied voxels tiled with periods
    (150, 280, 40) voxels = (15, 28, 4) m so that the cube is filled."""
    g, inflate = load_occupancy("pillar_512")
    if variant == "V1":
        idx = np.argwhere(inflate == 1)
        lo = idx.min(axis=0)
        rel = idx - lo
        out = np.zeros_like(inflate)
        per = (150, 280, 40)
        for ox in range(-4, 5):
            for oy in range(-3, 4):
                for oz in range(-13, 14):
                    sh = rel + lo + np.array([ox * per[0], oy * per[1], oz * per[2]])
                    ok = np.all(sh >= 0, axis=1) & np.all(sh < np.array(g.n), axis=1)
                    s = sh[ok]
                    out[s[:, 0], s[:, 1], s[:, 2]] = 1
        inflate = out
    elif variant != "V0":
        raise ValueError(variant)
    g = Grid(g.n, g.origin, g.res, box_min=g.origin + 0.5, box_max=g.map_max - 0.5)
    return g, inflate


def random_boxes_map(n=(1024, 1024, 256), seed=11, n_boxes=4096, ground_idx=10, origin=None):
    """Config 4: synthetic map, axis-aligned boxes with side U[0.3,3] m + a ground plane."""
    rng = np.random.default_rng(seed)
    res = 0.1
    if origin is None:
        origin = (-n[0] * res / 2, -n[1] * res / 2, -1.0)
    g = Grid(n, origin, res)
    inflate = np.zeros(n, dtype=np.int8)
    side = rng.uniform(0.3, 3.0, size=(n_boxes, 3))
    ctr = rng.uniform(0, 1, size=(n_boxes, 3)) * (np.array(n) * res)
    lo = np.clip(np.floor((ctr - side / 2) / res).astype(np.int64), 0, np.array(n) - 1)
    hi = np.clip(np.floor((ctr + side / 2) / res).astype(np.int64), 0, np.array(n) - 1)
    for a, b in zip(lo, hi):
        inflate[a[0]:b[0] + 1, a[1]:b[1] + 1, a[2]:b[2] + 1] = 1
    if 0 <= ground_idx < n[2]:
        inflate[:, :, ground_idx] = 1
    return g, inflate


def known_region(g, inflate, seed=7, n_poses=64, radius=4.5, z_range=(0.5, 2.0)):
    """Tri-state occupancy for the frontier sweep: FREE = voxels within `radius` metres
    (max_ray_length, algorithm.xml:50) of seeded camera poses in free space and not
    occupied; OCCUPIED = occupied voxels inside the same balls; everything else UNKNOWN."""
    rng = np.random.default_rng(seed)
    n = np.array(g.n)
    tri = np.zeros(g.n, dtype=np.uint8)
    r = int(np.ceil(radius / g.res))
    ax = np.arange(-r, r + 1)
    ball = (ax[:, None, None] ** 2 + ax[None, :, None] ** 2 + ax[None, None, :] ** 2) * g.res ** 2 <= radius ** 2
    placed = 0
    tries = 0
    lo_b = g.pos_to_index(g.box_min + 0.3)
    hi_b = g.pos_to_index(g.box_max - 0.3)
    zlo = max(lo_b[2], int(g.pos_to_index([0, 0, z_range[0]])[2]))
    zhi = min(hi_b[2], int(g.pos_to_index([0, 0, z_range[1]])[2]))
    while placed < n_poses and tries < 100 * n_poses:
        tries += 1
        c = np.array([rng.integers(lo_b[0], hi_b[0] + 1), rng.integers(lo_b[1], hi_b[1] + 1),
                      rng.integers(zlo, max(zlo, zhi) + 1)])
        if inflate[c[0], c[1], c[2]]:
            continue
        placed += 1
        a0 = np.maximum(c - r, 0)
        a1 = np.minimum(c + r + 1, n)
        b0 = a0 - (c - r)
        b1 = b0 + (a1 - a0)
        sub = tri[a0[0]:a1[0], a0[1]:a1[1], a0[2]:a1[2]]
        sub[ball[b0[0]:b1[0], b0[1]:b1[1], b0[2]:b1[2]]] = FREE
    tri[(tri == FREE) & (inflate == 1)] = OCCUPIED
    return tri


def office_known(g, inflate):
    """The known region used with the office maps (configs 1, 2, 5): 8 camera balls of 2.5 m,
    which leaves ~2/3 of the map unknown and a dozen frontier clusters above cluster_min."""
    return known_region(g, inflate, seed=7, n_poses=8, radius=2.5)


def cubic_boundary_states(ctrl, dt):
    """Uniform cubic B-spline boundary maps (bspline_optimizer.cpp:367-389, 405-427)."""
    q = ctrl
    start = np.stack([(q[0] + 4 * q[1] + q[2]) / 6.0, (q[2] - q[0]) / (2 * dt), (q[0] - 2 * q[1] + q[2]) / (dt * dt)])
    end_pos = (q[-1] + 4 * q[-2] + q[-3]) / 6.0
    return start, end_pos


def make_trajectories(g, inflate, B=1024, n_pts=20, seed=20260922, sigma=0.3, spacing=0.35, max_vel=2.0):
    """Config 2 trajectory batch.  Straight lines between seeded start/goal voxels in the free
    space of the box interior, control points spaced ~ctrl_pt_dist 0.35 m (algorithm.xml:140),
    interior control points perturbed by N(0, sigma) so a realistic fraction lies inside
    dist0; boundary states from the unperturbed spline; time_lb = -1 (SURVEY 8d).
    Returns dict(ctrl [B,N,3], dt [B], start [B,3,3], end_pos [B,3], pt_dist [B])."""
    rng = np.random.default_rng(seed)
    lo = g.box_min + 0.15
    hi = g.box_max - 0.15
    length = spacing * (n_pts - 1)
    ctrl = np.zeros((B, n_pts, 3))
    dts = np.zeros(B)
    starts = np.zeros((B, 3, 3))
    ends = np.zeros((B, 3))
    ptd = np.zeros(B)
    b = 0
    while b < B:
        s = rng.uniform(lo, hi)
        si = g.pos_to_index(s)
        if inflate[si[0], si[1], si[2]]:
            continue
        d = rng.normal(size=3)
        d[2] *= 0.15
        d /= np.linalg.norm(d)
        L = length * rng.uniform(0.7, 1.15)
        e = s + d * L
        if np.any(e < lo) or np.any(e > hi):
            continue
        ei = g.pos_to_index(e)
        if inflate[ei[0], ei[1], ei[2]]:
            continue
        t = np.linspace(0.0, 1.0, n_pts)[:, None]
        line = s[None, :] * (1 - t) + e[None, :] * t
        dt = (L / (n_pts - 1)) / (max_vel * rng.uniform(0.55, 0.95))
        st, en = cubic_boundary_states(line, dt)
        pert = line.copy()
        pert[3:n_pts - 3] += rng.normal(scale=sigma, size=(n_pts - 6, 3))
        pert = np.minimum(np.maximum(pert, g.box_min + 0.1), g.box_max - 0.1)  # optimize() clamp :196-204
        ctrl[b] = pert
        dts[b] = dt
        starts[b] = st
        ends[b] = en
        # pt_dist_ is frozen from the initial control points (:136-140)
        seg = np.sqrt(np.sum((pert[1:] - pert[:-1]) ** 2, axis=1))
        acc = 0.0
        for v in seg:
            acc += float(v)
        ptd[b] = acc / float(n_pts)
        b += 1
    return dict(ctrl=ctrl, dt=dts, start=starts, end_pos=ends, pt_dist=ptd)


def pack_x(ctrl, dt, mintime=True):
    B = ctrl.shape[0]
    x = ctrl.reshape(B, -1)
    if mintime:
        x = np.concatenate([x, dt[:, None]], axis=1)
    return np.ascontiguousarray(x, dtype=np.float64)


def _camera_rotation(yaw, pitch=0.0):
    """camera -> world rotation: camera z = forward, x = right, y = down"""
    cyw, syw, cp, sp = np.cos(yaw), np.sin(yaw), np.cos(pitch), np.sin(pitch)
    fwd = np.array([cyw * cp, syw * cp, sp])
    right = np.array([syw, -cyw, 0.0])
    down = np.cross(fwd, right)
    return np.stack([right, down, fwd], axis=1)


def depth_image(g, inflate, cam_pos, yaw, pitch=0.0, width=640, height=480, fx=387.229248046875, fy=387.229248046875,
                cx=321.04638671875, cy=243.44969177246094, margin=2, skip=2, maxdist=5.0, mindist=0.2):
    """Synthetic sensor frame: a pinhole depth camera (intrinsics of exploration.launch:38-41) at cam_pos looking
    along `yaw`, ray-marched against the ground-truth occupancy `inflate`; uint16 millimetres, 0 = no return.  Rays
    are marched for the pixels MapROS samples (margin + k*skip) and replicated to their neighbours.
    -> (image uint16 [height,width], R [3,3] camera->world)"""
    cam_pos = np.asarray(cam_pos, dtype=np.float64)
    off = margin % skip
    us = np.arange(off, width, skip)
    vs = np.arange(off, height, skip)
    U, V = np.meshgrid(us, vs)
    dirs_c = np.stack([(U - cx) / fx, (V - cy) / fy, np.ones_like(U, dtype=np.float64)], axis=-1).reshape(-1, 3)
    R = _camera_rotation(yaw, pitch)
    dirs_w = dirs_c @ R.T
    n = np.asarray(g.n)
    depth = np.zeros(dirs_c.shape[0])  # 0 = no return
    alive = np.ones(dirs_c.shape[0], dtype=bool)
    flat = np.ascontiguousarray(inflate).reshape(-1)
    for t in np.arange(mindist, maxdist + 0.3, 0.04):
        idx_alive = np.nonzero(alive)[0]
        if idx_alive.size == 0:
            break
        p = cam_pos + dirs_w[idx_alive] * t
        vi = np.floor((p - np.asarray(g.origin)) / g.res).astype(np.int64)
        inside = np.all((vi >= 0) & (vi < n), axis=1)
        adr = (np.clip(vi[:, 0], 0, n[0] - 1) * n[1] + np.clip(vi[:, 1], 0, n[1] - 1)) * n[2] + np.clip(vi[:, 2], 0, n[2] - 1)
        hit = inside & (flat[adr] != 0)
        depth[idx_alive[hit]] = t
        alive[idx_alive[hit]] = False
    low = np.round(depth * 1000.0).astype(np.uint16).reshape(len(vs), len(us))
    vi = np.clip((np.arange(height) - off) // skip, 0, len(vs) - 1)
    ui = np.clip((np.arange(width) - off) // skip, 0, len(us) - 1)
    return np.ascontiguousarray(low[vi][:, ui]), R


def depth_frame(g, inflate, cam_pos, yaw, pitch=0.0, width=640, height=480, fx=387.229248046875, fy=387.229248046875,
                cx=321.04638671875, cy=243.44969177246094, margin=2, skip=2, maxdist=5.0, mindist=0.2):
    """depth_image() projected to world points the way MapROS::proessDepthImage (plan_env/src/map_ros.cpp:176-215) hands
    them to inputPointCloud (no-return pixels at depth_filter_maxdist).  Input generation only (numpy); the parity-checked
    projection is fuelgpu_map_input_depth_image vs the oracle.  -> float32 [n,3] world points."""
    img, R = depth_image(g, inflate, cam_pos, yaw, pitch, width, height, fx, fy, cx, cy, margin, skip, maxdist, mindist)
    us = np.arange(margin, width - margin, skip)
    vs = np.arange(margin, height - margin, skip)
    U, V = np.meshgrid(us, vs)
    d16 = img[V, U].reshape(-1)
    d = d16 * (1.0 / 1000.0)
    # the reference's "no return" test looks at the pixel `skip` further along the row buffer (map_ros.cpp:190-198)
    flat = img.reshape(-1)
    nxt_at = (V * width + U + skip).reshape(-1)
    nxt = np.where(nxt_at < flat.size, flat[np.minimum(nxt_at, flat.size - 1)], 0)
    far = (nxt == 0) | (d > maxdist)
    keep = far | (d >= mindist)
    d = np.where(far, maxdist, d)
    dirs_c = np.stack([(U - cx) / fx, (V - cy) / fy, np.ones_like(U, dtype=np.float64)], axis=-1).reshape(-1, 3)
    pts = (dirs_c * d[:, None]) @ R.T + np.asarray(cam_pos, dtype=np.float64)
    return np.ascontiguousarray(pts[keep], dtype=np.float32)


def make_tours(g, inflate, B=1024, seed=20261015, spacing=3.0, max_vel=2.0, max_acc=2.0):
    """Candidate tours for planExploreTraj, shaped like shortenPath's output (fast_exploration_manager.cpp:239-263,
    321-323): 3 to 12 waypoints about `spacing` apart in the free space of the exploration box, a short midpoint
    inserted into the first leg of some of them (always into a one-leg tour, as shortenPath does).  Most tours are 1.5 to
    8 m long, so their point counts span several groups from 11 up; about 4 % are 13 to 18 m (n_pts up to about 64), and the
    last tour is about 30 m (past FUELGPU_MAX_PTS).  Start velocity / acceleration are random within max_vel / max_acc.
    Returns dict(tours: list of [W, 3] arrays, start_vel [B, 3], start_acc [B, 3])."""
    rng = np.random.default_rng(seed)
    lo = g.box_min + 0.15
    hi = g.box_max - 0.15

    def free(p):
        if np.any(p < lo) or np.any(p > hi):
            return False
        i = g.pos_to_index(p)
        return not inflate[i[0], i[1], i[2]]

    tours = []
    while len(tours) < B:
        last = len(tours) == B - 1
        r = rng.uniform()
        L = 30.0 if last else (rng.uniform(13.0, 18.0) if r < 0.04 else rng.uniform(1.5, 8.0))
        n_leg = int(min(11, max(1, round(L / spacing))))
        p = rng.uniform(lo, hi)
        if not free(p):
            continue
        pts = [p]
        for _ in range(n_leg):
            for _try in range(20):
                d = rng.normal(size=3)
                d[2] *= 0.15
                q = pts[-1] + d / np.linalg.norm(d) * (L / n_leg) * rng.uniform(0.85, 1.15)
                if free(q):
                    pts.append(q)
                    break
            else:
                break
        if len(pts) != n_leg + 1:
            continue
        if n_leg == 1 or rng.uniform() < 0.2:
            pts.insert(1, 0.5 * (pts[0] + pts[1]))
        tours.append(np.array(pts))
    dirs = rng.normal(size=(B, 3))
    dirs /= np.linalg.norm(dirs, axis=1, keepdims=True)
    start_vel = dirs * rng.uniform(0.0, max_vel, (B, 1))
    dirs = rng.normal(size=(B, 3))
    dirs /= np.linalg.norm(dirs, axis=1, keepdims=True)
    start_acc = dirs * rng.uniform(0.0, max_acc, (B, 1))
    return dict(tours=tours, start_vel=start_vel, start_acc=start_acc)


def make_yaws(B, seed=20261016, heading=None):
    """Start and end yaws for planYawExplore (planner_manager.cpp:774-865) over a batch of B trajectories.
    start [B, 3] = (yaw, yawdot, yawddot): yaw uniform in [-pi, pi], a quarter of them 1 to 5 whole turns outside it
    (the wrapping loops run); rates uniform in [-1, 1] rad/s and [-1, 1] rad/s^2.  end [B]: uniform in [-pi, pi].
    heading [B] (optional, e.g. the direction of travel at each trajectory's end): then every fourth end yaw lies 1e-3 to
    0.1 rad inside heading +- pi, where calcNextYaw's |diff| is close to pi.
    Returns dict(start [B, 3], end [B])."""
    rng = np.random.default_rng(seed)
    start = np.empty((B, 3))
    start[:, 0] = rng.uniform(-np.pi, np.pi, B)
    turns = rng.integers(1, 6, B) * rng.choice([-1, 1], B)
    outside = rng.uniform(size=B) < 0.25
    start[outside, 0] += 2 * np.pi * turns[outside]
    start[:, 1] = rng.uniform(-1.0, 1.0, B)
    start[:, 2] = rng.uniform(-1.0, 1.0, B)
    end = rng.uniform(-np.pi, np.pi, B)
    if heading is not None:
        h = np.broadcast_to(np.asarray(heading, dtype=np.float64), (B,))
        near = np.arange(B) % 4 == 3
        side = rng.choice([-1.0, 1.0], B)
        end[near] = h[near] + side[near] * (np.pi - rng.uniform(1e-3, 0.1, B)[near])
    return dict(start=start, end=end)


def make_path_queries(g, inflate, tri, B=1024, seed=20261017):
    """Start / goal pairs for Astar::search as planExploreMotion issues them (fast_exploration_manager.cpp:238-241).
    Starts lie in known-free space inside the exploration box (tri = office_known's).  Goals, in turn: a candidate
    viewpoint of a frontier cluster (a point 1.5 to 2.5 m from a known-free voxel next to unknown space, in the
    sampleViewpoints ring, known-free itself); a known-free point 0.3 to 20 m away; a goal inside unknown, occupied
    (inflated) or enclosed space; and, rarely, start == goal or a goal one voxel away.
    Returns dict(start [B, 3], goal [B, 3], kind [B]: 0 viewpoint, 1 free, 2 unknown, 3 occupied, 4 same, 5 adjacent)."""
    rng = np.random.default_rng(seed)
    lo = g.box_min + 0.15
    hi = g.box_max - 0.15
    free = (np.asarray(tri) == FREE) & (np.asarray(inflate) == 0)
    fidx = np.argwhere(free)
    fpos = g.index_to_pos(fidx)
    inb = np.all((fpos > lo) & (fpos < hi), axis=1)
    fidx, fpos = fidx[inb], fpos[inb]
    unk = np.asarray(tri) == UNKNOWN
    # known-free voxels with an unknown 6-neighbour: where frontier clusters sit
    edge = np.zeros_like(free)
    for a in range(3):
        for s in (-1, 1):
            edge |= np.roll(unk, s, axis=a)
    fr = free & edge
    fr_idx = np.argwhere(fr)
    fr_pos = g.index_to_pos(fr_idx)
    fr_pos = fr_pos[np.all((fr_pos > lo) & (fr_pos < hi), axis=1)]
    occ_pos = g.index_to_pos(np.argwhere(np.asarray(inflate) == 1))
    occ_pos = occ_pos[np.all((occ_pos > lo) & (occ_pos < hi), axis=1)]
    unk_pos = g.index_to_pos(np.argwhere(unk))
    unk_pos = unk_pos[np.all((unk_pos > lo) & (unk_pos < hi), axis=1)]
    fset = set(map(tuple, fidx.tolist()))

    def is_free(p):
        if np.any(p <= lo) or np.any(p >= hi):
            return False
        return tuple(g.pos_to_index(p).tolist()) in fset

    start = np.empty((B, 3))
    goal = np.empty((B, 3))
    kind = np.empty(B, np.int32)
    b = 0
    while b < B:
        s = fpos[rng.integers(len(fpos))] + rng.uniform(-0.04, 0.04, 3)
        if not is_free(s):
            continue
        r = rng.uniform()
        if r < 0.45:
            k = 0
            c = fr_pos[rng.integers(len(fr_pos))]
            phi = rng.uniform(-np.pi, np.pi)
            q = c + rng.uniform(1.5, 2.5) * np.array([np.cos(phi), np.sin(phi), 0.0])
            if not is_free(q):
                continue
        elif r < 0.80:
            k = 1
            d = rng.normal(size=3)
            d[2] *= 0.2
            q = s + d / np.linalg.norm(d) * rng.uniform(0.3, 20.0)
            if not is_free(q):
                continue
        elif r < 0.88:
            k = 2
            q = unk_pos[rng.integers(len(unk_pos))] + rng.uniform(-0.04, 0.04, 3)
        elif r < 0.96:
            k = 3
            q = occ_pos[rng.integers(len(occ_pos))] + rng.uniform(-0.04, 0.04, 3)
        elif r < 0.98:
            k = 4
            q = s.copy()
        else:
            k = 5
            q = s + rng.choice([-1.0, 0.0, 1.0], 3) * g.res
        start[b], goal[b], kind[b] = s, q, k
        b += 1
    return dict(start=start, goal=goal, kind=kind)


def make_view_pairs(g, inflate, tri, P=4096, seed=20261018):
    """Viewpoint pairs for ViewNode::computeCost (graph_node.cpp:63-85) as the tour's cost asks for them: the pairs of
    make_path_queries (clear and blocked lines, goals in unknown or occupied space, start == goal), one in eight with
    its second point moved above the exploration box so that the line leaves it, yaws over the whole circle, and a
    velocity on half of the pairs -- some below the 1e-3 threshold and some along the pair's own direction, where
    acos meets a dot product at 1.  Returns dict(p1, p2, v1 [P, 3], y1, y2 [P])."""
    rng = np.random.default_rng(seed)
    q = make_path_queries(g, inflate, tri, B=P, seed=seed)
    p1, p2 = q["start"].copy(), q["goal"].copy()
    out = rng.uniform(size=P) < 0.125
    p2[out, 2] = g.box_max[2] + rng.uniform(0.05, 0.5, int(out.sum()))
    y1, y2 = rng.uniform(-np.pi, np.pi, P), rng.uniform(-np.pi, np.pi, P)
    v1 = np.zeros((P, 3))
    r = rng.uniform(size=P)
    moving = r < 0.4
    v1[moving] = rng.normal(size=(int(moving.sum()), 3)) * np.array([1.0, 1.0, 0.3])
    tiny = (r >= 0.4) & (r < 0.45)
    v1[tiny] = rng.normal(size=(int(tiny.sum()), 3)) * 3e-4
    along = (r >= 0.45) & (r < 0.5)
    v1[along] = (p2[along] - p1[along]) * rng.uniform(0.2, 2.0, (int(along.sum()), 1))
    return dict(p1=p1, p2=p2, y1=y1, y2=y2, v1=v1)


def make_local_tours(g, inflate, tri, B=256, seed=20261019):
    """refineLocalTour problems (fast_exploration_manager.cpp:429-503) as planExploreMotion builds them: a current
    state in known-free space and 2 to 7 groups of 1 to 15 viewpoints, each group spread 1.5 to 2.5 m around a point
    2 to 6 m on from the one before (some in unknown or occupied space, so lines are blocked and searches fail).
    Half the problems move; among them some fly exactly along the first edge (acos at a dot product of 1).  The
    special cases, one problem in twelve each: duplicated viewpoints (equal g values), a group of one repeated
    viewpoint (all its costs equal), an empty middle group (unreachable), a first group of one viewpoint at cur_pos
    (a zero-length tour segment), a single group.
    Returns dict(prob_off [B+1], group_off [G+1], cur_pos, cur_vel [B, 3], cur_yaw [B], vp_pos [N, 3], vp_yaw [N],
    kind [B]: 0 plain, 1 duplicates, 2 repeated group, 3 empty middle group, 4 refined point at cur_pos, 5 one group)."""
    rng = np.random.default_rng(seed)
    pool = make_path_queries(g, inflate, tri, B=4 * B + 64, seed=seed)["start"]
    prob_off, group_off = [0], [0]
    cur_pos, cur_vel, cur_yaw, vp_pos, vp_yaw, kinds = [], [], [], [], [], []
    for b in range(B):
        kind = int(rng.integers(12)) if rng.uniform() < 0.5 else 0
        kind = kind if kind <= 5 else 0
        p0 = pool[rng.integers(len(pool))]
        ng = 1 if kind == 5 else int(rng.integers(2, 8))
        c = p0.copy()
        groups = []
        for i in range(ng):
            d = np.linalg.norm(pool - c, axis=1)
            near = np.flatnonzero((d > 2.0) & (d < 6.0))
            c = pool[rng.choice(near)] if len(near) else c
            n = int(rng.integers(1, 16))
            phi = rng.uniform(-np.pi, np.pi, n)
            r = rng.uniform(1.5, 2.5, n)
            pts = c + np.stack([r * np.cos(phi), r * np.sin(phi), rng.uniform(-0.3, 0.3, n)], axis=1)
            ys = rng.uniform(-np.pi, np.pi, n)
            groups.append([pts, ys])
        if kind == 1:  # duplicates: repeat viewpoints inside groups
            for grp in groups[:-1]:
                k = rng.integers(len(grp[0]), size=max(1, len(grp[0]) // 2))
                grp[0], grp[1] = np.concatenate([grp[0], grp[0][k]]), np.concatenate([grp[1], grp[1][k]])
        elif kind == 2 and ng > 1:  # one group of a single repeated viewpoint
            i = int(rng.integers(ng - 1))
            n = len(groups[i][0])
            groups[i] = [np.repeat(groups[i][0][:1], n, axis=0), np.repeat(groups[i][1][:1], n)]
        elif kind == 3 and ng > 2:
            groups[int(rng.integers(1, ng - 1))] = [np.zeros((0, 3)), np.zeros(0)]
        elif kind == 4 and ng > 1:
            groups[0] = [p0.reshape(1, 3).copy(), groups[0][1][:1]]
        for pts, ys in groups:
            vp_pos.append(pts)
            vp_yaw.append(ys)
            group_off.append(group_off[-1] + len(pts))
        prob_off.append(prob_off[-1] + ng)
        v = np.zeros(3)
        u = rng.uniform()
        if u < 0.35:
            v = rng.normal(size=3) * np.array([1.0, 1.0, 0.3])
        elif u < 0.45 and len(groups[0][0]):  # along the edge to the first group's first viewpoint
            v = (groups[0][0][0] - p0) * rng.uniform(0.2, 2.0)
        elif u < 0.5:
            v = rng.normal(size=3) * 3e-4
        cur_pos.append(p0)
        cur_vel.append(v)
        cur_yaw.append(rng.uniform(-np.pi, np.pi))
        kinds.append(kind)
    return dict(prob_off=np.asarray(prob_off, np.int32), group_off=np.asarray(group_off, np.int32),
                cur_pos=np.asarray(cur_pos), cur_vel=np.asarray(cur_vel), cur_yaw=np.asarray(cur_yaw),
                vp_pos=np.concatenate(vp_pos), vp_yaw=np.concatenate(vp_yaw), kind=np.asarray(kinds, np.int32))


def make_global_tours(n, B=1, seed=20261020, kind="geometric", vm=2.0, yd=60 * 3.1415926 / 180.0):
    """B cost matrices of findGlobalTour's shape ([B, n + 1, n + 1], column 0 zero) for the global tour:
    "geometric": ViewNode::computeCost's form over random viewpoints of a 20 x 20 x 3 m box, max(distance / vm,
    yaw change / yd), one pair in ten at the 1000 of a failed search (in both directions, as updateFrontierCostMatrix
    stores it), row 0 from a current state with a velocity term; "random": integer-valued costs 0 .. 19.99 with one
    entry in five at 500 (an asymmetric matrix with far outliers)."""
    rng = np.random.default_rng(seed)
    d = n + 1
    out = np.zeros((B, d, d))
    for b in range(B):
        if kind == "random":
            m = rng.integers(0, 2000, (d, d)) / 100.0
            m[rng.random((d, d)) < 0.2] = 500.0
        else:
            p = rng.uniform([0, 0, 0], [20, 20, 3], (d, 3))
            y = rng.uniform(-3.1415926, 3.1415926, d)
            dist = np.linalg.norm(p[:, None] - p[None], axis=2)
            dy = np.abs(y[:, None] - y[None])
            dy = np.minimum(dy, 2 * 3.1415926 - dy)
            m = np.maximum(dist / vm, dy / yd)
            fail = np.triu(rng.random((d, d)) < 0.1, 1)
            m[fail | fail.T] = 1000.0
            m[0, 1:] += rng.uniform(0, 0.5, n)  # the velocity change from the current state
        m[:, 0] = 0.0
        np.fill_diagonal(m, 0.0)
        out[b] = m
    return out


def make_kino_queries(g, inflate, tri, info, start, goal, seed=20261019, max_vel=2.0, max_acc=2.0):
    """kinodynamicReplan queries from the MID rows of a path search (info: FuelPathInfo rows of fuelgpu_astar_batch for
    start / goal): start, goal and a start velocity and acceleration within the search's limits, as the exploration
    FSM hands over the current state.  Returns dict(rows, start, vel, acc, goal) with rows the MID indices."""
    rng = np.random.default_rng(seed)
    rows = np.flatnonzero((info["status"] == 1) & (info["branch"] == 2))
    n = len(rows)
    vel = rng.uniform(-1, 1, (n, 3)) * max_vel * 0.6
    vel[:, 2] *= 0.3
    acc = rng.uniform(-1, 1, (n, 3)) * max_acc * 0.5
    still = rng.random(n) < 0.2  # hovering before the replan
    vel[still] = 0.0
    acc[still] = 0.0
    return dict(rows=rows, start=np.asarray(start)[rows].copy(), vel=vel, acc=acc, goal=np.asarray(goal)[rows].copy())
