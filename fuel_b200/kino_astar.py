"""KinodynamicAstar (path_searching/include/path_searching/kinodynamic_astar.h) and the search of
FastPlannerManager::kinodynamicReplan (plan_manage/src/planner_manager.cpp:131-164) on the device, over
fuelgpu_kino_search_batch.

kino_search_batch runs B replans' searches -- the close-goal refusal, search(init = true), the retry at init = false and
getSamples -- and returns the arrays fuelgpu_bspline_parameterize_batch takes.  kinodynamic_replan_batch carries them
on through parameterizeToBspline and getBoundaryStates, and kino_replan_traj_batch through the solver and planYaw, like
plan_explore_traj_batch.  KinodynamicAstar is
the reference's class over one search; only the non-dynamic search exists (FUEL's exploration never asks for another).
"""
import ctypes as C

import numpy as np

from ._lib import MAX_PTS, FuelKinoParams, check, lib, ptr
from .non_uniform_bspline import _handle

# KinodynamicAstar's codes, then the rows not searched (FuelKinoInfo.status)
REACH_HORIZON, REACH_END, NO_PATH, NEAR_END, SKIPPED, BAD_INPUT = 1, 2, 3, 4, 5, 6
# FuelKinoInfo.reason
FOUND, OPEN_EMPTY, POOL, START_NEAR_END, CLOSE_GOAL = 0, 1, 2, 3, 4
# FuelKinoInfo.traj_status
TRAJ_OK, TOO_LONG, NO_TRAJ = 0, 1, 2
NODE_FIELDS = 12  # state (6), input (3), duration, g, f

INFO_DTYPE = np.dtype([("status", np.int32), ("reason", np.int32), ("retried", np.int32), ("traj_status", np.int32),
                       ("iter_num", np.int32), ("use_node_num", np.int32), ("n_nodes", np.int32), ("shot", np.int32),
                       ("seg_num", np.int32), ("n_pts", np.int32), ("t_shot", np.float64), ("T_sum", np.float64)])

# exploration_manager/launch/algorithm.xml, with exploration.launch's max_vel = max_acc = 2.0
DEFAULTS = dict(max_tau=0.8, init_max_tau=1.0, max_vel=2.0, vel_margin=0.25, max_acc=2.0, w_time=10.0, horizon=5.0,
                lambda_heu=10.0, resolution=0.025, ctrl_pt_dist=0.35, manager_max_vel=2.0, allocate_num=100000,
                check_num=10, optimistic=False)


def make_params(**kw):
    """FuelKinoParams from DEFAULTS overridden by kw"""
    unknown = set(kw) - set(DEFAULTS)
    if unknown:
        raise TypeError("unknown kinodynamic search parameters: %s" % sorted(unknown))
    p = dict(DEFAULTS, **kw)
    return FuelKinoParams(*[float(p[k]) for k in ("max_tau", "init_max_tau", "max_vel", "vel_margin", "max_acc",
                                                  "w_time", "horizon", "lambda_heu", "resolution", "ctrl_pt_dist",
                                                  "manager_max_vel")],
                          int(p["allocate_num"]), int(p["check_num"]), int(bool(p["optimistic"])), 0)


def _rows(a, B=None):
    a = np.ascontiguousarray(np.asarray(a, dtype=np.float64).reshape(-1, 3))
    if B is not None and len(a) != B:
        raise ValueError("start, vel, acc and goal must all be [B, 3]")
    return a


def kino_search_batch(sdf_map, start, vel, acc, goal, *, node_max=0, **params):
    """fuelgpu_kino_search_batch over B queries -> dict(info [B] of INFO_DTYPE, points [B, MAX_PTS-2, 3],
    derivs [B, 4, 3], dt [B], nodes [B, node_max, 12] or None, shot [B, 3, 4])"""
    s = _rows(start)
    B = len(s)
    v, a, g = _rows(vel, B), _rows(acc, B), _rows(goal, B)
    prm = make_params(**params)
    info = np.empty(B, dtype=INFO_DTYPE)
    points = np.empty((B, MAX_PTS - 2, 3))
    derivs = np.empty((B, 4, 3))
    dt = np.empty(B)
    nodes = np.empty((B, node_max, NODE_FIELDS)) if node_max > 0 else None
    shot = np.empty((B, 3, 4))
    h = _handle(sdf_map)
    check(lib().fuelgpu_kino_search_batch(h, B, ptr(s), ptr(v), ptr(a), ptr(g), C.byref(prm), ptr(info), ptr(points),
                                          ptr(derivs), ptr(dt), int(max(node_max, 0)), ptr(nodes), ptr(shot)), h)
    return dict(info=info, points=points, derivs=derivs, dt=dt, nodes=nodes, shot=shot)


def kinodynamic_replan_batch(sdf_map, start, vel, acc, goal, time_lb=None, **params):
    """kinodynamicReplan(start, vel, acc, goal, 0, time_lb) up to the solver's input for every row that has samples:
    returns (res, groups) with res the kino_search_batch dict and groups a list of (rows, x, traj) per point count,
    x and traj from parameterizeToBspline and getBoundaryStates (non_uniform_bspline.parameterize_batch)."""
    from .non_uniform_bspline import parameterize_batch
    res = kino_search_batch(sdf_map, start, vel, acc, goal, **params)
    info = res["info"]
    groups = []
    ok = np.flatnonzero(info["traj_status"] == TRAJ_OK)
    for n in np.unique(info["n_pts"][ok]):
        rows = ok[info["n_pts"][ok] == n]
        K = int(n) - 2
        tlb = None if time_lb is None else np.asarray(time_lb, dtype=np.float64).reshape(-1)[rows]
        x, traj = parameterize_batch(sdf_map, res["points"][rows, :K], res["derivs"][rows], res["dt"][rows], tlb)
        groups.append((rows, x, traj))
    return res, groups


def kino_replan_traj_batch(sdf_map, start, vel, acc, goal, opt, solve, start_yaw, time_lb=None, **params):
    """KinoReplanFSM::callKinodynamicReplan's planner calls for B replans: kinodynamicReplan(start, vel, acc, goal, 0,
    time_lb) -- kinodynamic_replan_batch, then opt.optimizeBatch on each point count's group -- and planYaw(start_yaw)
    (polynomial_traj.plan_yaw_batch) on each group's solver output.
    opt: a BsplineOptimizer set up on `sdf_map`; solve: keyword arguments of optimizeBatch besides x / traj_consts /
    n_pts, with cost_function (NORMAL_PHASE, with MINTIME where manager/min_time sets it); start_yaw: [3] or [B, 3].
    Returns dict(res: the kino_search_batch dict, x: a list of [nvar] solver outputs or None per row, yaw [B, 131],
    yaw_info [B] of PLANYAW_INFO_DTYPE); rows without samples keep None, NaN yaw and status -1."""
    from .polynomial_traj import PLANYAW_INFO_DTYPE, PLANYAW_MAX_PTS, plan_yaw_batch
    res, groups = kinodynamic_replan_batch(sdf_map, start, vel, acc, goal, time_lb, **params)
    B = len(res["info"])
    sy = np.broadcast_to(np.asarray(start_yaw, dtype=np.float64), (B, 3))
    mask = int(solve["cost_function"])
    mintime = bool(mask & opt.MINTIME)
    kw = {k: v for k, v in solve.items() if k != "cost_function"}
    xs = [None] * B
    yaw = np.full((B, PLANYAW_MAX_PTS), np.nan)
    yaw_info = np.zeros(B, dtype=PLANYAW_INFO_DTYPE)
    yaw_info["dt_yaw"] = yaw_info["pt_dist"] = np.nan
    yaw_info["status"] = -1
    for rows, x0, tc in groups:
        n = (x0.shape[1] - 1) // 3
        dt = None if mintime else x0[:, 3 * n].copy()
        x, _, _ = opt.optimizeBatch(x0 if mintime else np.ascontiguousarray(x0[:, :3 * n]), tc, n, mask, **kw)
        yaw[rows], yaw_info[rows], _ = plan_yaw_batch(sdf_map, x, n, sy[rows], opt, dt=dt)
        for r, b in enumerate(rows):
            xs[b] = x[r].copy()
    return dict(res=res, x=xs, yaw=yaw, yaw_info=yaw_info)


class KinodynamicAstar:
    """kinodynamicReplan's use of the reference's KinodynamicAstar, over one query on the device of an EDTEnvironment's
    map (setParam + init -> the constructor, with the search/ parameters as keywords).  search() is not the reference's
    single search(init) call: it runs what kinodynamicReplan runs -- the close-goal refusal, search(init = true) and,
    after NO_PATH, reset and search(init = false) -- and returns the status of the attempt that counted (retried()
    tells whether the retry ran).  getSamples() returns the samples at kinodynamicReplan's ts = ctrl_pt_dist /
    manager_max_vel, fixed when the search ran."""

    REACH_HORIZON, REACH_END, NO_PATH, NEAR_END = REACH_HORIZON, REACH_END, NO_PATH, NEAR_END

    def __init__(self, env, node_max=4096, **params):
        self.env_ = env
        make_params(**params)
        self.params_ = dict(params)
        p = dict(DEFAULTS, **params)
        self.ts0_ = float(p["ctrl_pt_dist"]) / float(p["manager_max_vel"])
        self.node_max = int(node_max)
        self.reset()

    def reset(self):
        self.res_ = None
        self.use_node_num_ = 0
        self.iter_num_ = 0
        self.is_shot_succ_ = False

    def search(self, start_pt, start_v, start_a, end_pt, end_v=(0.0, 0.0, 0.0), init=True, dynamic=False,
               time_start=-1.0):
        """kinodynamicReplan's search sequence (see the class); init = False, a non-zero end_v and dynamic = True are
        refused, since kinodynamicReplan never starts there"""
        if dynamic:
            raise NotImplementedError("the dynamic (time-indexed) search is not implemented")
        if not init or np.any(np.asarray(end_v, dtype=np.float64) != 0.0):
            raise NotImplementedError("only kinodynamicReplan's sequence from search(init = true, end_v = 0) runs here")
        m = getattr(self.env_, "sdf_map_", self.env_)
        res = kino_search_batch(m, [start_pt], [start_v], [start_a], [end_pt], node_max=self.node_max,
                                **self.params_)
        i = res["info"][0]
        self.res_ = res
        self.use_node_num_ = int(i["use_node_num"])
        self.iter_num_ = int(i["iter_num"])
        self.is_shot_succ_ = bool(i["shot"])
        return int(i["status"])

    def retried(self):
        return bool(self.res_["info"][0]["retried"])

    def getSamples(self, ts=None):
        """-> (ts, point_set [K, 3], start_end_derivatives [4, 3]) at kinodynamicReplan's ts = ctrl_pt_dist /
        manager_max_vel; a different ts is refused"""
        if ts is not None and ts != self.ts0_:
            raise ValueError("getSamples runs at ctrl_pt_dist / manager_max_vel = %r" % self.ts0_)
        i = self.res_["info"][0]
        if i["traj_status"] != TRAJ_OK:
            raise RuntimeError("no samples: status %d, traj_status %d" % (i["status"], i["traj_status"]))
        K = int(i["n_pts"]) - 2
        return float(self.res_["dt"][0]), self.res_["points"][0, :K].copy(), self.res_["derivs"][0].copy()
