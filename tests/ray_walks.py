"""Ray families for the voxel walks of the device (RayCaster::input / nextId, plan_env/src/raycast.cpp:329-407) and the
verdicts they must give, taken from the reference's own RayCaster only (oracle.ref_raycast_ids over
oracle/_ref/libfuel_ref.so) and the occupancy of the map.

A walk goes wrong at ties between tMax values, on axes with a zero voxel delta (intbound = inf, tDelta = 0/0), at starts
on voxel faces, edges and corners, in nextId's cast<int> (truncation toward zero for the voxels just below the origin)
and on grids whose origin is not a multiple of the resolution.  Some rays never meet their end voxel: their last steps
tie at t = 1 and the walk steps past it for ever ("overshooting"); the device walks stop after GUARD steps, so on those
rays the expected verdict is the one over the reference's first GUARD ids."""
import os
import re

import numpy as np

import oracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WALK_SRC = [os.path.join(ROOT, "fuel_b200", "csrc", f) for f in ("raycast.cuh", "fusion.cu")]

FAMILIES = ("random", "axis", "lattice", "diagonal", "short", "below_origin", "overshoot")
FUSION_FAMILIES = FAMILIES[:-1]


def guard_constants():
    """the step guard of every device walk, read from the kernel files"""
    out = []
    for path in WALK_SRC:
        with open(path) as f:
            out += [int(v) for v in re.findall(r"for \(int guard = 0; guard < (\d+); \+\+guard\)", f.read())]
    return out


GUARD = 4096


def has_reference():
    return oracle.ref_raycast() is not None


class Geo:
    """the geometry a walk needs: resolution, origin, voxel counts, exploration box in voxel indices"""

    def __init__(self, n, res, origin, box_mind=None, box_maxd=None, map_size=None):
        self.n = np.asarray(n, np.int64)
        self.res = float(res)
        self.origin = np.asarray(origin, np.float64)
        # map_max_boundary_ = origin + map_size_ (sdf_map.cpp:39), n * res unless the map size says otherwise
        self.map_size = self.n * self.res if map_size is None else np.asarray(map_size, np.float64)
        self.map_max = self.origin + self.map_size
        self.box_mind = self.origin.copy() if box_mind is None else np.asarray(box_mind, np.float64)
        self.box_maxd = self.map_max.copy() if box_maxd is None else np.asarray(box_maxd, np.float64)
        # posToIndex(box_mind_ / box_maxd_), sdf_map.cpp:83-84
        self.box_min = np.floor((self.box_mind - self.origin) * (1 / self.res)).astype(np.int64)
        self.box_max = np.floor((self.box_maxd - self.origin) * (1 / self.res)).astype(np.int64)
        self.orc = oracle.make_grid(self.n, self.res, self.origin)

    @property
    def shape(self):
        return tuple(int(v) for v in self.n)

    def grid(self):
        """the same geometry as a workloads.Grid, for the device map and the A* oracle's map"""
        from fuel_b200 import workloads as W
        return W.Grid(self.shape, self.origin, self.res, box_min=self.box_mind, box_max=self.box_maxd)

    def lattice(self, k):
        """k * res + origin, per axis, as the code computes voxel faces"""
        return np.asarray(k, np.float64) * self.res + self.origin


def walk(geo, a, b):
    """the ids the reference's nextId reports for input(a, b), at most GUARD of them"""
    return oracle.ref_raycast_ids(geo.orc, a, b, max_ids=GUARD)


def overshoots(geo, a, b):
    """True when the reference's walk takes more steps than |dx| + |dy| + |dz|: it never meets its end voxel"""
    d = np.abs(np.floor(np.asarray(b) / geo.res) - np.floor(np.asarray(a) / geo.res)).sum()
    return len(oracle.ref_raycast_ids(geo.orc, a, b, max_ids=int(d) + 2)) > d


def ray_families(geo, rng, count=300, end=None, float32=False, span_lo=-0.1, span_hi=1.1, special=(), n_overshoot=None):
    """family -> (a [N, 3], b [N, 3]): rays a -> b.  With `end` every ray ends there and the family shapes its start.
    float32: starts rounded to float32, like the points of a pcl cloud.  special: extra voxel indices per axis (box
    faces, ...) the lattice families snap to as well as random ones.  n_overshoot: overshooting rays wanted (count)."""
    o, r, n = geo.origin, geo.res, geo.n
    span = n * r
    fixed = end is not None
    end = None if end is None else np.asarray(end, np.float64)

    def rand_pt(m):
        return o + rng.uniform(span_lo, span_hi, (m, 3)) * span

    def rand_k(m):
        k = np.stack([rng.integers(-2, n[i] + 3, m) for i in range(3)], axis=1)
        extra = np.asarray(special, np.int64).reshape(-1, 3)
        pick = [np.concatenate([[0, 1, n[i] - 1, n[i]], extra[:, i]]) for i in range(3)]
        sel = rng.random((m, 3)) < 0.25
        for i in range(3):
            k[sel[:, i], i] = rng.choice(pick[i], int(sel[:, i].sum()))
        return k

    def f32_exact(k):
        """k moved to the nearest lattice index whose position k * res + origin a float32 holds exactly: points on a
        voxel face that stay there after pcl's float32"""
        k = np.array(k)
        for i in range(3):
            for q in range(len(k)):
                for dk in range(0, 64):
                    v = geo.lattice(np.full(3, k[q, i] + dk))[i]
                    if np.float32(v) == v:
                        k[q, i] += dk
                        break
        return k

    def near_end(m, scale=3.0):
        # flatter in z: a viewpoint's FOV spans +-top_angle about the horizontal
        return end + rng.uniform(-scale, scale, (m, 3)) * np.array([1.0, 1.0, 0.35])

    fam = {}
    m = count
    # 1. random, inside the map and across its border
    a = near_end(m) if fixed else rand_pt(m)
    b = np.repeat(end[None], m, 0) if fixed else rand_pt(m)
    fam["random"] = (a, b)
    # 2. axis-aligned: one or two zero voxel deltas
    a = near_end(m) if fixed else rand_pt(m)
    b = np.repeat(end[None], m, 0) if fixed else rand_pt(m)
    for q in range(m):
        axes = rng.choice(3, 1 + q % 2, replace=False)
        a[q, axes] = b[q, axes]
    fam["axis"] = (a, b)
    # 3. on voxel faces (one coordinate k * res + origin), edges (two) and corners (three)
    a = near_end(m) if fixed else rand_pt(m)
    b = np.repeat(end[None], m, 0) if fixed else rand_pt(m)
    ka = np.round((a - o) / r).astype(np.int64) if fixed else rand_k(m)  # with an end: the faces next to the start
    snap_a = geo.lattice(f32_exact(ka) if float32 else ka)
    snap_b = geo.lattice(rand_k(m))
    for q in range(m):
        axes = rng.choice(3, 1 + q % 3, replace=False)
        if fixed:
            a[q, axes] = snap_a[q, axes]
            continue
        which = q // 3 % 3  # start, end or both on the lattice
        if which != 1:
            a[q, axes] = snap_a[q, axes]
        if which != 0:
            b[q, axes] = snap_b[q, axes]
    fam["lattice"] = (a, b)
    # 4. exact lattice diagonals: tMax ties on two or three axes
    s = rng.choice([-1, 0, 1], (m, 3))
    if fixed:
        s[rng.random(m) < 0.6, 2] = 0
    s[np.count_nonzero(s, axis=1) < 2, :2] = 1
    steps = rng.integers(1, 40, (m, 1))
    f = rng.choice([0.0, 0.25, 0.5, 0.75], (m, 1))
    if fixed:
        a = end + (steps * s) * r
        b = np.repeat(end[None], m, 0)
    else:
        k = rand_k(m)
        a = geo.lattice(k + f)
        b = geo.lattice(k + steps * s + f)
    fam["diagonal"] = (a, b)
    # 5. zero-length rays and rays within one voxel
    a = near_end(m) if fixed else rand_pt(m)
    b = np.repeat(end[None], m, 0) if fixed else a + rng.uniform(-0.6, 0.6, (m, 3)) * r
    if fixed:
        a = end + rng.uniform(-0.6, 0.6, (m, 3)) * r
    zero = np.arange(m) % 3 == 0
    a[zero] = b[zero]
    fam["short"] = (a, b)
    # 6. through the strip just below the origin, where (int)(x + 0.5 - origin / res) truncates to index 0
    a = near_end(m) if fixed else rand_pt(m)
    b = np.repeat(end[None], m, 0) if fixed else rand_pt(m)
    for q in range(m):
        ax = rng.integers(0, 3)
        a[q, ax] = o[ax] - rng.choice([rng.uniform(0.0, 1.0), 0.5, 1.0 - 1e-9]) * r
        if not fixed and q % 2 == 0:
            b[q, ax] = o[ax] - rng.uniform(0.0, 1.0) * r  # the whole ray runs in the strip
    fam["below_origin"] = (a, b)
    if float32:
        fam = {k: (v[0].astype(np.float32).astype(np.float64), v[1]) for k, v in fam.items()}
    # 8. overshooting rays, found by running the reference's walk with a cap: one or both ends on the lattice.  Their
    # first crossing falls a rounding error after t = 0, which a start rounded to float32 does not keep: none for pcl
    # points
    if has_reference() and not float32:
        got_a, got_b = [], []
        for _ in range(400):
            if len(got_a) >= (n_overshoot or count):
                break
            a = near_end(256) if fixed else rand_pt(256)
            b = np.repeat(end[None], 256, 0) if fixed else rand_pt(256)
            k = np.round((a - o) / r).astype(np.int64) if fixed else rand_k(256)
            for q in range(256):
                axes = rng.choice(3, 1 + q % 3, replace=False)
                a[q, axes] = geo.lattice(k[q])[axes]
                if not fixed and q % 2:
                    b[q, axes] = geo.lattice(k[q] + rng.integers(-30, 31, 3))[axes]
            for q in range(256):
                if overshoots(geo, a[q], b[q]):
                    got_a.append(a[q])
                    got_b.append(b[q])
        got = n_overshoot or count
        fam["overshoot"] = (np.array(got_a[:got]).reshape(-1, 3), np.array(got_b[:got]).reshape(-1, 3))
    return fam


def occ_flags(inflate, tri):
    """per voxel: blocks a walk (inflated or UNKNOWN)"""
    return (np.asarray(inflate) == 1) | (np.asarray(tri) == oracle.UNKNOWN)


def verdict(geo, blocks, a, b, box=False):
    """True when the ray a -> b is clear: countVisibleCells / shortenPath (frontier_finder.cpp:743-751,
    fast_exploration_manager.cpp:308-316) and, with box, searchPath's straight line (graph_node.cpp:36-43), from the
    reference's own ids"""
    ids = walk(geo, a, b)
    if len(ids) == 0:
        return True
    inmap = np.all((ids >= 0) & (ids < geo.n), axis=1)
    j = ids[inmap]
    if np.any(blocks[j[:, 0], j[:, 1], j[:, 2]]):
        return False
    if box and not np.all((ids >= geo.box_min) & (ids < geo.box_max)):
        return False
    return True


def verdicts(geo, blocks, a, b, box=False):
    return np.array([verdict(geo, blocks, a[q], b[q], box) for q in range(len(a))], bool)


def scattered_map(geo, seed, p=0.004, p_plane=0.08):
    """(inflate int8, tri uint8): scattered inflated and UNKNOWN voxels, denser on the index-0 planes that the strip
    below the origin reads"""
    from fuel_b200 import workloads as W
    rng = np.random.default_rng(seed)
    n = tuple(int(v) for v in geo.n)
    pr = np.full(n, p)
    pr[0, :, :] = pr[:, 0, :] = pr[:, :, 0] = p_plane
    inflate = (rng.random(n) < pr).astype(np.int8)
    tri = np.full(n, W.FREE, np.uint8)
    tri[(rng.random(n) < pr) & (inflate == 0)] = W.UNKNOWN
    tri[inflate == 1] = W.OCCUPIED
    return inflate, tri


# ------------------------------------------------------------------------------------------------------------------
# Fusion: SDFMap::inputPointCloud (sdf_map.cpp:259-345) with the reference's ray ids
# ------------------------------------------------------------------------------------------------------------------

def _norm(d):
    return np.sqrt((d[0] * d[0] + d[1] * d[1]) + d[2] * d[2])


def expected_fusion(geo, logodds, pts, cam, max_ray_length=4.5, p_hit=0.65, p_miss=0.35, p_min=0.12, p_max=0.90,
                    p_occ=0.80):
    """one frame on the log-odds volume `logodds` (flat, updated in place): clipping and hit / miss flags of
    :273-306, the end voxel's hit or miss, a miss on every id of the reference's walk after the first that lies in the
    map (:307-311), the update of :326-344.  -> (touched voxel count, every walk ended in the map)"""
    logit = lambda q: np.log(q / (1 - q))  # noqa: E731
    hit, miss, cmin, cmax, mocc = logit(p_hit), logit(p_miss), logit(p_min), logit(p_max), logit(p_occ)
    o, mx = geo.origin, geo.map_max
    n = geo.n
    cam = np.asarray(cam, np.float64)
    count_hit, count_miss, rayend = {}, {}, set()
    clean = True
    for pt in np.asarray(pts, np.float32).astype(np.float64):
        p = [float(v) for v in pt]
        c = [float(v) for v in cam]
        inmap = not any(p[k] < o[k] + 1e-4 or p[k] > mx[k] - 1e-4 for k in range(3))
        if not inmap:  # closetPointInMap, :347-362
            diff = [p[k] - c[k] for k in range(3)]
            min_t = 1000000.0
            for k in range(3):
                if abs(diff[k]) > 0:
                    t1 = (mx[k] - c[k]) / diff[k]
                    if 0 < t1 < min_t:
                        min_t = t1
                    t2 = (o[k] - c[k]) / diff[k]
                    if 0 < t2 < min_t:
                        min_t = t2
            p = [c[k] + (min_t - 1e-3) * diff[k] for k in range(3)]
        d = [p[k] - c[k] for k in range(3)]
        length = float(_norm(d))
        if length > max_ray_length:
            p = [d[k] / length * max_ray_length + c[k] for k in range(3)]
            if p[2] < 0.2:
                continue
            flag = 0
        elif not inmap:
            if p[2] < 0.2:
                continue
            flag = 0
        else:
            flag = 1
        idx = np.floor((np.array(p) - o) * (1 / geo.res)).astype(np.int64)
        if np.any(idx < 0) or np.any(idx >= n):
            clean = False  # the reference would address outside its buffers
            continue
        adr = tuple(idx)
        if flag:
            count_hit[adr] = count_hit.get(adr, 0) + 1
        else:
            count_miss[adr] = 1
        if adr in rayend:
            continue
        rayend.add(adr)
        ids = walk(geo, np.array(p), cam)
        if len(ids) >= GUARD or (len(ids) and not np.all((ids >= 0) & (ids < n))):
            clean = False
        for j in ids[1:]:
            if np.all(j >= 0) and np.all(j < n):
                count_miss[tuple(j)] = 1
    touched = set(count_hit) | set(count_miss)
    shape = tuple(int(v) for v in n)
    for adr in touched:
        a = np.ravel_multi_index(adr, shape)
        upd = hit if count_hit.get(adr, 0) >= count_miss.get(adr, 0) else miss
        v = logodds[a]
        if v < cmin - 1e-3:
            v = mocc
        logodds[a] = min(max(v + upd, cmin), cmax)
    return len(touched), clean


def fusion_frames(geo, rng, per_family=60):
    """[(family, points float32 [N, 3], camera [3])]: cameras on voxel faces, corners, centres and outside the map, points
    from every family ending at the camera, some far enough to be clipped by max_ray_length or closetPointInMap"""
    o, r = geo.origin, geo.res
    mid = o + 0.5 * geo.n * r
    k = np.floor((mid - o) / r).astype(np.int64)
    cams = {
        "face": np.array([geo.lattice(k)[0], mid[1] + 0.037, mid[2] + 0.011]),
        "corner": geo.lattice(k + np.array([3, -2, 1])),
        "centre": geo.lattice(k + 0.5),
        "outside": np.array([o[0] - 0.35, mid[1] + 0.2, mid[2] + 0.1]),
    }
    frames = []
    for name, cam in cams.items():
        fam = ray_families(geo, rng, count=per_family, end=cam, float32=True)
        for fname, (a, _) in fam.items():
            if fname == "random":  # far points: clipped by max_ray_length and by closetPointInMap
                a = (cam + (a - cam) * rng.uniform(1.0, 3.0, (len(a), 1))).astype(np.float32).astype(np.float64)
            frames.append(("%s/%s" % (name, fname), a.astype(np.float32), cam))
    return frames


def tristate(logodds, p_min=0.12, p_occ=0.80):
    """getOccupancy of each log-odds (sdf_map.h:194-200): UNKNOWN below clamp_min_log - 1e-3, OCCUPIED above
    min_occupancy_log, FREE between"""
    cmin, mocc = np.log(p_min / (1 - p_min)), np.log(p_occ / (1 - p_occ))
    return np.where(logodds < cmin - 1e-3, oracle.UNKNOWN, np.where(logodds > mocc, oracle.OCCUPIED, oracle.FREE))


def fresh_logodds(geo):
    """initMap's occupancy_buffer_: clamp_min_log - unknown_flag everywhere (sdf_map.cpp:56,64)"""
    return np.full(int(np.prod(geo.n)), np.log(0.12 / (1 - 0.12)) - 0.01)


FUSION_MAP = dict(resolution=0.1, map_size_x=8.0, map_size_y=6.0, map_size_z=3.0, ground_height=-0.5,
                  obstacles_inflation=0.199, local_bound_inflate=0.5, local_map_margin=50, default_dist=0.0, optimistic=0,
                  signed_dist=0, p_hit=0.65, p_miss=0.35, p_min=0.12, p_max=0.90, p_occ=0.80, max_ray_length=4.5,
                  virtual_ceil_height=-10.0)


FUSION_RES = (0.1, 0.15)


def fusion_geo(res):
    """the map of FUSION_MAP at resolution res: origin (-size_x / 2, -size_y / 2, ground_height) (sdf_map.cpp:33), a
    multiple of 0.1 but not of 0.15, where the RayCaster's first id is often not the voxel posToIndex gives the point"""
    size = np.array([FUSION_MAP["map_size_" + a] for a in "xyz"])
    n = np.ceil(size / res).astype(np.int64)  # sdf_map.cpp:36
    return Geo(n, res, (-size[0] / 2, -size[1] / 2, FUSION_MAP["ground_height"]), map_size=size)


def ref_fusion_map(res):
    return oracle.RefSDFMap(**dict(FUSION_MAP, resolution=res))


# ------------------------------------------------------------------------------------------------------------------
# The straight-line test and countVisibleCells
# ------------------------------------------------------------------------------------------------------------------

LINE_CASES = ("res0.1", "offgrid_origin", "ties", "ties_offgrid_origin")
VIEW_CASES = LINE_CASES[:2]


def line_case(case):
    """(geo, inflate, tri, family -> (a, b)) for the straight-line test: scattered inflated and UNKNOWN voxels and an
    exploration box smaller than the map (index 0 inside it on x and z, so the strip below the origin reads in-box
    voxels there).  offgrid_origin: origin (0.3, -2.7, 0.05) at res 0.15, not a multiple of it.  ties*: the same
    grids, free but for the voxels tie_blockers inflates beside the walks of the diagonal and lattice families."""
    base = case.replace("ties_", "").replace("ties", "res0.1")
    geo, inflate, tri = line_case_map(base)
    ties = case.startswith("ties")
    fam = ray_families(geo, np.random.default_rng(17), count=4000 if ties else 400, special=[geo.box_min, geo.box_max],
                       n_overshoot=400)
    if ties:
        from fuel_b200 import workloads as W
        inflate[...] = 0
        tri[...] = W.FREE

        def in_box(a, b):
            ids = walk(geo, a, b)
            return len(ids) > 0 and bool(np.all((ids >= geo.box_min) & (ids < geo.box_max)))

        for name, (a, b) in fam.items():  # diagonal and lattice walks that stay in the box, where only ties block
            keep = [q for q in range(len(a)) if in_box(a[q], b[q])] if name in ("diagonal", "lattice") else range(len(a))
            keep = np.array(list(keep)[:400], np.int64)
            fam[name] = (a[keep], b[keep])
        tie_blockers(geo, inflate, tri, [fam["diagonal"], fam["lattice"]], np.random.default_rng(19))
    return geo, inflate, tri, fam


def tie_blockers(geo, inflate, tri, rays, rng, frac=0.5):
    """inflate (in place) a fraction of the corner voxels beside the reference's walks, and none on them: where a walk
    steps along one axis and then another, the voxel it reaches by taking the two steps in the other order -- the one
    a walk that breaks the tie between their tMax values the other way enters instead.  Every walk of `rays` stays
    clear, so a walk that breaks a tie wrongly is seen as blocked half the time."""
    from fuel_b200 import workloads as W
    on_walk, alt = set(), set()
    for a, b in rays:
        for q in range(len(a)):
            ids = walk(geo, a[q], b[q])
            on_walk.update(map(tuple, ids))
            d = np.diff(ids, axis=0)
            for i in range(len(d) - 1):
                if np.any(d[i] != d[i + 1]):
                    alt.add(tuple(ids[i] + d[i + 1]))
    cand = [v for v in sorted(alt - on_walk) if all(0 <= v[k] < geo.n[k] for k in range(3))]
    for v in cand:
        if rng.random() < frac:
            inflate[v] = 1
            tri[v] = W.OCCUPIED


def longest_case():
    """a 1024 x 1024 x 64 map and its corner-to-corner ray, one inflated voxel on the walk's last id"""
    geo = Geo((1024, 1024, 64), 0.1, (-51.2, -51.2, -1.0))
    a = geo.lattice([0.5, 0.5, 0.5])
    b = geo.lattice([1023.5, 1023.5, 63.5])
    from fuel_b200 import workloads as W
    inflate = np.zeros(geo.shape, np.int8)
    tri = np.full(geo.shape, W.FREE, np.uint8)
    last = walk(geo, a, b)[-1]
    inflate[tuple(last)] = 1
    return geo, inflate, tri, a, b, last


VIEW_PARAMS = dict(candidate_rmin=1.0, candidate_rmax=2.0, candidate_rnum=2, candidate_dphi=0.5,
                   min_candidate_clearance=0.21, top_angle=0.56125, left_angle=0.69, right_angle=0.69, max_dist=4.5)


VIEW_AVERAGE = {"res0.1": (-4.4, 0.3, 0.2), "offgrid_origin": (2.0, 1.0, 1.2)}


def view_setup(case):
    """(geo, inflate, tri, average_, view params): the line map of `case`, a cluster average whose candidates reach the
    strip below the origin in x"""
    geo, inflate, tri = line_case_map(case)
    return geo, inflate, tri, np.array(VIEW_AVERAGE[case]), dict(VIEW_PARAMS)


def line_case_map(case):
    if case == "res0.1":
        geo = Geo((120, 100, 40), 0.1, (-6.0, -5.0, -1.0), box_mind=(-6.0, -4.5, -1.0), box_maxd=(5.5, 4.5, 2.7))
    else:
        geo = Geo((60, 50, 30), 0.15, (0.3, -2.7, 0.05), box_mind=(0.3, -2.4, 0.05), box_maxd=(8.7, 4.5, 4.0))
    inflate, tri = scattered_map(geo, 3)
    return geo, inflate, tri


def clear_near(geo, inflate, tri, pos, clearance):
    """copies of the map with every voxel within isNearUnknown's reach of a candidate FREE and not inflated"""
    from fuel_b200 import workloads as W
    inflate, tri = inflate.copy(), tri.copy()
    v = int(np.floor(clearance / geo.res)) + 1
    for p in pos:
        c = np.floor((p - geo.origin) / geo.res).astype(np.int64)
        lo = np.maximum(c - [v, v, 2], 0)
        hi = np.minimum(c + [v, v, 2] + 1, geo.n)
        if np.any(hi <= lo):
            continue
        sl = tuple(slice(lo[k], hi[k]) for k in range(3))
        tri[sl] = W.FREE
        inflate[sl] = 0
    return inflate, tri


def view_clusters(geo, pos, rng, targets=8, per=80, left_angle=VIEW_PARAMS["left_angle"]):
    """(clusters [k][c, 3], family of each, target candidate of each): single cells from every family ending at one of
    `targets` candidates, and for each target a two-cell cluster at +-left_angle about the direction to it (both cells
    on the FOV planes)"""
    clusters, fams, tgt = [], [], []
    for j in np.linspace(0, len(pos) - 1, targets).astype(int):
        for name, (a, _) in ray_families(geo, rng, count=per, end=pos[j]).items():
            clusters += [c[None] for c in a]
            fams += [name] * len(a)
            tgt += [j] * len(a)
        th = rng.uniform(-np.pi, np.pi)
        d = 1.5
        cells = np.array([pos[j] + d * np.array([np.cos(th + s * left_angle), np.sin(th + s * left_angle), 0.0])
                          for s in (1, -1)])
        clusters.append(cells)
        fams.append("border")
        tgt.append(j)
    return clusters, fams, np.array(tgt)


def in_fov(cell, p, vp, margin=0.05):
    """a single cell well inside the FOV of a candidate whose yaw points at it; a cell on the candidate itself has no
    direction, and is left out"""
    d = cell - p
    dist = float(_norm(d))
    return 0 < dist < vp["max_dist"] - margin and np.arctan2(abs(d[2]), np.hypot(d[0], d[1])) < vp["top_angle"] - margin


def check_visib(geo, blocks, pos, clusters, fams, tgt, vis, vp, rejected=None):
    """visib of every single-cell cluster at every candidate whose FOV holds the cell well inside: the reference walk's
    0 / 1 (countVisibleCells, frontier_finder.cpp:743-751); rejected candidates report -1 in every cluster.
    -> per family, the rays checked that join a cell to the candidate its family shaped it for"""
    rej = vis[0] < 0 if rejected is None else rejected
    assert np.all((vis < 0) == rej[None]), "rejected candidates differ between clusters"
    assert (~rej).sum() >= 5
    counts = {}
    for q, c in enumerate(clusters):
        if fams[q] == "border":
            continue
        for i in np.flatnonzero(~rej):
            if not in_fov(c[0], pos[i], vp):
                continue
            want = int(verdict(geo, blocks, c[0], pos[i]))
            assert vis[q, i] == want, "%s cell %s candidate %s: visib %d, reference walk %d" % (
                fams[q], c[0].tolist(), pos[i].tolist(), vis[q, i], want)
            if i == tgt[q]:
                counts[fams[q]] = counts.get(fams[q], 0) + 1
    return counts


# ------------------------------------------------------------------------------------------------------------------
# shortenPath (fast_exploration_manager.cpp:295-325) on A* paths whose nodes sit on the map's voxel faces
# ------------------------------------------------------------------------------------------------------------------

# the strip below the origin lies outside the map, where no search starts, and a zero-length or within-one-voxel query
# gives a path of two points, which shortenPath does not walk: those families cannot reach this probe
ASTAR_FAMILIES = ("random", "axis", "lattice", "diagonal", "overshoot")


def astar_case(count=120):
    """(geo, inflate, tri, family -> (start, goal)): test_lattice_ties's box with scattered inflated and UNKNOWN voxels;
    starts and goals on the voxel corners k * res + origin, with no offset, so A* node centres (idx + 0.5) * res_astar +
    origin at 0.2 and 0.4 m land on the faces of the 0.1 m map and every shortenPath ray starts and ends on them"""
    geo = Geo((60, 60, 30), 0.1, (-3.0, -3.0, -1.5), box_mind=(-2.95, -2.95, -1.45), box_maxd=(2.95, 2.95, 1.45))
    inflate, tri = scattered_map(geo, 7, p=0.006, p_plane=0.006)
    rng = np.random.default_rng(23)
    lo, hi = np.array([3, 3, 3]), geo.n - 3

    def corner(m):
        return np.stack([rng.integers(lo[i], hi[i], m) for i in range(3)], axis=1)

    q = {}
    k = np.arange(-5, 6) * 0.2  # test_lattice_ties's queries, on the corners
    s0 = np.stack([k, k, 0.5 * k], axis=1)
    g0 = np.stack([-k, k + 0.4, -0.5 * k], axis=1)
    q["lattice"] = (np.concatenate([s0, geo.lattice(corner(count))]), np.concatenate([g0, geo.lattice(corner(count))]))
    ks, kg = corner(count), corner(count)
    for i in range(count):
        axes = rng.choice(3, 1 + i % 2, replace=False)
        kg[i, axes] = ks[i, axes]
    q["axis"] = (geo.lattice(ks), geo.lattice(kg))
    ks = corner(count)
    s = rng.choice([-1, 1], (count, 3))
    s[rng.random(count) < 0.3, 2] = 0
    m = rng.integers(5, 25, (count, 1))
    kg = np.clip(ks + m * s, lo, hi - 1)
    q["diagonal"] = (geo.lattice(ks), geo.lattice(kg))
    span = geo.box_maxd - geo.box_mind
    q["random"] = tuple(geo.box_mind + 0.05 + rng.uniform(0, 1, (count, 3)) * (span - 0.1) for _ in range(2))
    return geo, inflate, tri, q


def _norm3(d):
    return float(np.sqrt((d[0] * d[0] + d[1] * d[1]) + d[2] * d[2]))


def expected_tour(geo, blocks, path):
    """shortenPath over the raw path with the reference's walk, then planExploreMotion's branch
    (fast_exploration_manager.cpp:243-263) -> (tour, rays shortenPath walked, every one of them ended)"""
    tour, rays = [path[0]], []
    for i in range(1, len(path) - 1):
        if _norm3(path[i] - tour[-1]) > 3.0:
            tour.append(path[i])
        else:
            rays.append((tour[-1], path[i + 1]))
            if not verdict(geo, blocks, tour[-1], path[i + 1]):
                tour.append(path[i])
    if _norm3(path[-1] - tour[-1]) > 1e-3:
        tour.append(path[-1])
    if len(tour) == 2:
        tour.insert(1, 0.5 * (tour[0] + tour[1]))
    length = sum(_norm3(tour[i + 1] - tour[i]) for i in range(len(tour) - 1))
    if length > 5.0:
        cut, len2 = [tour[0]], 0.0
        for p in tour[1:]:
            if len2 >= 5.0:
                break
            len2 += _norm3(p - cut[-1])
            cut.append(p)
        tour = cut
    ended = not any(overshoots(geo, a, b) for a, b in rays)
    return np.array(tour), rays, ended


def check_tours(geo, blocks, fam_of, info, path, n_wp, wp):
    """the waypoints of every search that reached its goal against expected_tour over its raw path.
    -> (rays walked per family, overshooting rays, mask of the searches whose walks all ended)"""
    counts, n_over = {}, 0
    ended = np.ones(len(info), bool)
    for b in np.flatnonzero(info["status"] == 1):
        tour, rays, ok = expected_tour(geo, blocks, path[b, :info["n_path"][b]])
        ended[b] = ok
        counts[fam_of[b]] = counts.get(fam_of[b], 0) + len(rays)
        n_over += sum(overshoots(geo, a, c) for a, c in rays)
        if info["tour_status"][b] == 0:
            assert n_wp[b] == len(tour) and np.array_equal(wp[b, :n_wp[b]], tour), (
                "%s search %d: waypoints differ from shortenPath over the reference's walk" % (fam_of[b], b))
    counts["overshoot"] = n_over
    return counts, ended


def astar_queries(q):
    """(start [B, 3], goal [B, 3], family of each) from astar_case's families"""
    start = np.concatenate([v[0] for v in q.values()])
    goal = np.concatenate([v[1] for v in q.values()])
    return start, goal, sum([[k] * len(v[0]) for k, v in q.items()], [])


def first_astar_difference(got, want):
    """None when two (info, path, n_wp, waypts) results agree bit for bit, else where they differ"""
    for f in want[0].dtype.names:
        bad = np.flatnonzero(np.any((got[0][f] != want[0][f]).reshape(len(want[0]), -1), axis=1))
        if bad.size:
            return "%s at %s" % (f, bad[:5])
    for i, name in ((1, "path"), (2, "n_wp"), (3, "waypts")):
        bad = np.flatnonzero(np.any((got[i] != want[i]).reshape(len(want[i]), -1), axis=1))
        if bad.size:
            return "%s at %s" % (name, bad[:5])
    return None
