"""ctypes binding of libfuelgpu.so (the C ABI of include/fuelgpu.h).

There is no CPU fallback: if the shared library is missing this module raises, and if no
sm_90 device is present every call through it fails with FUELGPU_ENODEVICE.
"""
import ctypes as C
import os

HERE = os.path.dirname(os.path.abspath(__file__))
SO = os.path.join(HERE, "libfuelgpu.so")

MAX_PTS = 64
UNKNOWN, FREE, OCCUPIED = 0, 1, 2
ESDF_OPTIMISTIC, ESDF_SIGNED = 1, 2
EDT_INF = 0x3FFFFFFF
OK, EINVAL, ENODEVICE, ECUDA, ENOMEM, EUNSUPPORTED = 0, -1, -2, -3, -4, -5


class FuelGpuError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__("fuelgpu error %d: %s" % (code, msg))
        self.code = code


class FuelGridDesc(C.Structure):
    _fields_ = [("n", C.c_int32 * 3), ("resolution", C.c_double), ("origin", C.c_double * 3),
                ("box_mind", C.c_double * 3), ("box_maxd", C.c_double * 3), ("map_size", C.c_double * 3)]


class FuelFrontierParams(C.Structure):
    _fields_ = [("cluster_min", C.c_int32), ("cluster_size_xy", C.c_double),
                ("down_sample", C.c_int32), ("min_z", C.c_double)]


class FuelFusionParams(C.Structure):
    _fields_ = [(k, C.c_double) for k in
                ("p_hit", "p_miss", "p_min", "p_max", "p_occ", "max_ray_length", "local_bound_inflate")]


class FuelCameraParams(C.Structure):
    _fields_ = [(k, C.c_double) for k in ("fx", "fy", "cx", "cy", "k_depth_scaling_factor", "depth_filter_maxdist",
                                          "depth_filter_mindist")] + [("depth_filter_margin", C.c_int32),
                                                                      ("skip_pixel", C.c_int32)]


class FuelViewParams(C.Structure):
    _fields_ = [("candidate_rmin", C.c_double), ("candidate_rmax", C.c_double), ("candidate_rnum", C.c_int32),
                ("candidate_dphi", C.c_double), ("min_candidate_clearance", C.c_double), ("top_angle", C.c_double),
                ("left_angle", C.c_double), ("right_angle", C.c_double), ("max_dist", C.c_double)]


class FuelOptParams(C.Structure):
    _fields_ = [(k, C.c_double) for k in
                ("ld_smooth", "ld_dist", "ld_feasi", "ld_start", "ld_end", "ld_guide", "ld_waypt",
                 "ld_view", "ld_time", "dist0", "max_vel", "max_acc")] + [("order", C.c_int32), ("wnl", C.c_double)]


class FuelTrajConst(C.Structure):
    _fields_ = [("pt_dist", C.c_double), ("knot_span", C.c_double),
                ("start", (C.c_double * 3) * 3), ("end", (C.c_double * 3) * 3),
                ("n_end", C.c_int32), ("time_lb", C.c_double), ("n_guide", C.c_int32),
                ("guide", (C.c_double * 3) * MAX_PTS), ("n_waypt", C.c_int32),
                ("waypt", (C.c_double * 3) * MAX_PTS), ("waypt_idx", C.c_int32 * MAX_PTS),
                ("view_pt", C.c_double * 3), ("view_dir", C.c_double * 3), ("view_idx", C.c_int32)]


class FuelSolveParams(C.Structure):
    _fields_ = [("max_eval", C.c_int32), ("lbfgs_m", C.c_int32), ("xtol_rel", C.c_double), ("flags", C.c_int32),
                ("reserved", C.c_int32)]


SOLVE_EXACT_EVALS = 1


class FuelTrajCheckParams(C.Structure):
    _fields_ = [("max_vel", C.c_double), ("max_acc", C.c_double), ("t_now", C.c_double)]


class FuelPolyParams(C.Structure):
    _fields_ = [("max_vel", C.c_double), ("ctrl_pt_dist", C.c_double), ("min_seg_num", C.c_int32),
                ("reserved", C.c_int32)]


class FuelYawParams(C.Structure):
    _fields_ = [("relax_time", C.c_double), ("lookfwd", C.c_int32), ("reserved", C.c_int32)]


class FuelYawInfo(C.Structure):
    _fields_ = [("dt_yaw", C.c_double), ("pt_dist", C.c_double), ("n_waypt", C.c_int32), ("status", C.c_int32)]


class FuelPlanYawInfo(C.Structure):
    _fields_ = [("dt_yaw", C.c_double), ("pt_dist", C.c_double), ("seg_num", C.c_int32), ("n_waypt", C.c_int32),
                ("status", C.c_int32), ("reserved", C.c_int32)]


class FuelAstarParams(C.Structure):
    _fields_ = [("resolution", C.c_double), ("lambda_heu", C.c_double), ("allocate_num", C.c_int32),
                ("max_iter", C.c_int32)]


class FuelKinoParams(C.Structure):
    _fields_ = [(k, C.c_double) for k in ("max_tau", "init_max_tau", "max_vel", "vel_margin", "max_acc", "w_time",
                                          "horizon", "lambda_heu", "resolution", "ctrl_pt_dist", "manager_max_vel")] + \
               [(k, C.c_int32) for k in ("allocate_num", "check_num", "optimistic", "reserved")]


class FuelViewCostParams(C.Structure):
    _fields_ = [("vm", C.c_double), ("yd", C.c_double), ("w_dir", C.c_double), ("astar", FuelAstarParams)]


class FuelLocalTourParams(C.Structure):
    _fields_ = [("view", FuelViewCostParams), ("tour_lambda_heu", C.c_double)]


class FuelTrajReport(C.Structure):
    _fields_ = [("duration", C.c_double), ("jerk", C.c_double), ("ratio", C.c_double), ("distance", C.c_double),
                ("safe", C.c_int32), ("feasible", C.c_int32), ("n_checked", C.c_int32), ("reserved", C.c_int32)]


CHECK_MAX_SAMPLES = 1 << 20


# every symbol include/fuelgpu.h declares: name -> (restype, argtypes)
_vp, _i32, _i64, _dbl = C.c_void_p, C.c_int32, C.c_int64, C.c_double
SIGNATURES = {
    "fuelgpu_version": (C.c_char_p, []),
    "fuelgpu_last_error": (C.c_char_p, [_vp]),
    "fuelgpu_device_info": (C.c_int, [C.c_int, C.c_char_p, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int)]),
    "fuelgpu_map_create": (C.c_int, [C.POINTER(FuelGridDesc), C.c_int, C.POINTER(_vp)]),
    "fuelgpu_map_destroy": (C.c_int, [_vp]),
    "fuelgpu_map_set_stream": (C.c_int, [_vp, _vp]),
    "fuelgpu_map_synchronize": (C.c_int, [_vp]),
    "fuelgpu_map_device_ptrs": (C.c_int, [_vp, C.POINTER(_vp), C.POINTER(_vp), C.POINTER(_vp)]),
    "fuelgpu_map_last_timing": (C.c_int, [_vp, C.POINTER(C.c_float)]),
    "fuelgpu_map_last_timeline": (C.c_int, [_vp, C.POINTER(C.c_float), C.POINTER(C.c_float)]),
    "fuelgpu_host_register": (C.c_int, [_vp, C.c_uint64]),
    "fuelgpu_host_unregister": (C.c_int, [_vp]),
    "fuelgpu_map_upload_occupancy": (C.c_int, [_vp, _vp, _vp, _vp, _dbl, _dbl, _vp, _vp]),
    "fuelgpu_map_upload_occupancy_async": (C.c_int, [_vp, _vp, _vp, _vp, _dbl, _dbl, _vp, _vp]),
    "fuelgpu_map_inflate": (C.c_int, [_vp, _vp, _vp, _i32, _i32]),
    "fuelgpu_map_download_occupancy": (C.c_int, [_vp, _vp, _vp]),
    "fuelgpu_map_input_point_cloud": (C.c_int, [_vp, _vp, _i32, _i32, _vp, C.POINTER(FuelFusionParams), _vp, _vp]),
    "fuelgpu_map_input_depth_image": (C.c_int, [_vp, _vp, _i32, _i32, C.POINTER(FuelCameraParams), _vp, _vp,
                                                C.POINTER(FuelFusionParams), _vp, _vp, C.POINTER(_i32)]),
    "fuelgpu_map_get_updated_box": (C.c_int, [_vp, _vp, _vp, _i32]),
    "fuelgpu_map_set_logodds": (C.c_int, [_vp, _vp, _dbl, _dbl]),
    "fuelgpu_map_get_logodds": (C.c_int, [_vp, _vp]),
    "fuelgpu_esdf_update": (C.c_int, [_vp, _vp, _vp, C.c_int]),
    "fuelgpu_esdf_download": (C.c_int, [_vp, _vp, _vp, _vp, _vp]),
    "fuelgpu_esdf_download_async": (C.c_int, [_vp, _vp, _vp, _vp]),
    "fuelgpu_esdf_sample": (C.c_int, [_vp, _i64, _vp, _vp, _vp]),
    "fuelgpu_frontier_search": (C.c_int, [_vp, _vp, _vp, C.POINTER(FuelFrontierParams),
                                          C.POINTER(_i32), C.POINTER(_i32), C.POINTER(_i32)]),
    "fuelgpu_frontier_search_begin": (C.c_int, [_vp, _vp, _vp, C.POINTER(FuelFrontierParams)]),
    "fuelgpu_frontier_search_end": (C.c_int, [_vp, C.POINTER(_i32), C.POINTER(_i32), C.POINTER(_i32)]),
    "fuelgpu_frontier_fetch": (C.c_int, [_vp] + [_vp] * 7),
    "fuelgpu_frontier_clear_flags": (C.c_int, [_vp, _i32, _vp]),
    "fuelgpu_frontier_is_changed": (C.c_int, [_vp, _i32, _vp, _vp, _vp]),
    "fuelgpu_frontier_reset_flags": (C.c_int, [_vp]),
    "fuelgpu_frontier_changed_counts": (C.c_int, [_vp, _i32, _vp, _vp, _vp]),
    "fuelgpu_viewpoint_candidate_count": (_i32, [C.POINTER(FuelViewParams)]),
    "fuelgpu_frontier_sample_viewpoints": (C.c_int, [_vp, _i32, _vp, _vp, _vp, C.POINTER(FuelViewParams), _i32, _vp, _vp,
                                                     _vp]),
    "fuelgpu_map_launch_count": (C.c_int, [_vp, C.POINTER(C.c_int64)]),
    "fuelgpu_frontier_download_flags": (C.c_int, [_vp, _vp]),
    "fuelgpu_frontier_upload_flags": (C.c_int, [_vp, _vp]),
    "fuelgpu_bspline_cost_batch": (C.c_int, [_vp, _i32, _i32, _i32, C.POINTER(FuelOptParams), _vp, _vp,
                                             _vp, _vp]),
    "fuelgpu_bspline_cost_batch_dev": (C.c_int, [_vp, _i32, _i32, _i32, C.POINTER(FuelOptParams), _vp,
                                                 _vp, _vp, _vp]),
    "fuelgpu_bspline_optimize_batch": (C.c_int, [_vp, _i32, _i32, _i32, C.POINTER(FuelOptParams), _vp,
                                                 C.POINTER(FuelSolveParams), _vp, _vp, _vp]),
    "fuelgpu_bspline_optimize_batch_begin": (C.c_int, [_vp, _i32, _i32, _i32, C.POINTER(FuelOptParams), _vp,
                                                       C.POINTER(FuelSolveParams), _vp]),
    "fuelgpu_bspline_optimize_batch_end": (C.c_int, [_vp, _vp, _vp, _vp]),
    "fuelgpu_bspline_optimize_batch_dev": (C.c_int, [_vp, _i32, _i32, _i32, C.POINTER(FuelOptParams), _vp,
                                                     C.POINTER(FuelSolveParams), _vp, _vp, _vp]),
    "fuelgpu_frontier_set_cell_order": (C.c_int, [_vp, _i32]),
    "fuelgpu_frontier_candidates": (C.c_int, [_vp, _vp, _vp, C.POINTER(FuelFrontierParams), _i32, _i32, C.POINTER(_i32)]),
    "fuelgpu_frontier_candidates_fetch": (C.c_int, [_vp, _i32, _vp, _vp]),
    "fuelgpu_frontier_search_from_candidates": (C.c_int, [_vp, _vp, _vp, C.POINTER(FuelFrontierParams), _i32, _vp, _vp,
                                                          C.POINTER(_i32), C.POINTER(_i32), C.POINTER(_i32)]),
    "fuelgpu_map_occupancy_plane_dev": (C.c_int, [_vp, _i32, _vp, _i32]),
    "fuelgpu_comm_get_unique_id": (C.c_int, [_vp]),
    "fuelgpu_comm_init": (C.c_int, [_i32, _i32, _vp, _i32, C.POINTER(_vp)]),
    "fuelgpu_comm_info": (C.c_int, [_vp, C.POINTER(_i32), C.POINTER(_i32)]),
    "fuelgpu_comm_destroy": (C.c_int, [_vp]),
    "fuelgpu_sharded_esdf_create": (C.c_int, [_vp, C.POINTER(_i32), _dbl, C.POINTER(_vp)]),
    "fuelgpu_sharded_esdf_update": (C.c_int, [_vp, _vp, _vp, C.c_int, _vp]),
    "fuelgpu_sharded_esdf_last_timing": (C.c_int, [_vp, C.POINTER(C.c_float)]),
    "fuelgpu_sharded_esdf_bytes_exchanged": (_i64, [_vp]),
    "fuelgpu_sharded_esdf_uses_peer_memory": (C.c_int, [_vp]),
    "fuelgpu_sharded_esdf_allgather": (C.c_int, [_vp, _vp, _vp, _vp]),
    "fuelgpu_sharded_esdf_destroy": (C.c_int, [_vp]),
    "fuelgpu_esdf_set_from_slabs_dev": (C.c_int, [_vp, _vp, _i32]),
    "fuelgpu_bspline_check_batch": (C.c_int, [_vp, _i32, _i32, _i32, _vp, _vp, C.POINTER(FuelTrajCheckParams), _vp, _vp]),
    "fuelgpu_bspline_check_batch_dev": (C.c_int, [_vp, _i32, _i32, _i32, _vp, _vp, C.POINTER(FuelTrajCheckParams), _vp,
                                                  _vp]),
    "fuelgpu_bspline_evaluate_batch": (C.c_int, [_vp, _i32, _i32, _i32, _vp, _vp, _i32, _vp, _i32, _vp]),
    "fuelgpu_bspline_parameterize_batch": (C.c_int, [_vp, _i32, _i32, _i32, _vp, _vp, _vp, _vp, _vp, _vp]),
    "fuelgpu_bspline_parameterize_batch_dev": (C.c_int, [_vp, _i32, _i32, _i32, _vp, _vp, _vp, _vp, _vp, _vp]),
    "fuelgpu_poly_waypoints_batch": (C.c_int, [_vp, _i32, _i32, _vp, _vp, _vp, _vp, _vp, _vp, _vp,
                                               C.POINTER(FuelPolyParams), _vp, _vp, _vp, _vp]),
    "fuelgpu_poly_waypoints_batch_dev": (C.c_int, [_vp, _i32, _i32, _vp, _vp, _vp, _vp, _vp, _vp, _vp,
                                                   C.POINTER(FuelPolyParams), _vp, _vp, _vp, _vp]),
    "fuelgpu_yaw_explore_batch": (C.c_int, [_vp, _i32, _i32, _i32, _vp, _vp, _vp, _vp, C.POINTER(FuelOptParams),
                                            C.POINTER(FuelYawParams), _vp, _vp, _vp]),
    "fuelgpu_yaw_explore_batch_dev": (C.c_int, [_vp, _i32, _i32, _i32, _vp, _vp, _vp, _vp, C.POINTER(FuelOptParams),
                                                C.POINTER(FuelYawParams), _vp, _vp, _vp]),
    "fuelgpu_plan_yaw_batch": (C.c_int, [_vp, _i32, _i32, _i32, _vp, _vp, _vp, C.POINTER(FuelOptParams), _vp, _vp, _vp]),
    "fuelgpu_plan_yaw_batch_dev": (C.c_int, [_vp, _i32, _i32, _i32, _vp, _vp, _vp, C.POINTER(FuelOptParams), _vp, _vp,
                                             _vp]),
    "fuelgpu_astar_batch": (C.c_int, [_vp, _i32, _vp, _vp, C.POINTER(FuelAstarParams), _vp, _i32, _vp, _i32, _vp, _vp]),
    "fuelgpu_astar_batch_dev": (C.c_int, [_vp, _i32, _vp, _vp, C.POINTER(FuelAstarParams), _vp, _i32, _vp, _i32, _vp,
                                          _vp]),
    "fuelgpu_view_cost_batch": (C.c_int, [_vp, _i32, _vp, _vp, _vp, _vp, _vp, C.POINTER(FuelViewCostParams), _vp, _i32,
                                          _vp]),
    "fuelgpu_view_cost_batch_dev": (C.c_int, [_vp, _i32, _vp, _vp, _vp, _vp, _vp, C.POINTER(FuelViewCostParams), _vp,
                                              _i32, _vp]),
    "fuelgpu_local_tour_batch": (C.c_int, [_vp, _i32, _vp, _vp, _vp, _vp, _vp, _vp, _vp, C.POINTER(FuelLocalTourParams),
                                           _vp, _i32, _vp, _i32, _vp, _vp]),
    "fuelgpu_local_tour_batch_dev": (C.c_int, [_vp, _i32, _vp, _vp, _vp, _vp, _vp, _vp, _vp,
                                               C.POINTER(FuelLocalTourParams), _vp, _i32, _vp, _i32, _vp, _vp]),
    "fuelgpu_global_tour_batch": (C.c_int, [_vp, _i32, _vp, _vp, _vp, _vp]),
    "fuelgpu_global_tour_batch_dev": (C.c_int, [_vp, _i32, _vp, _vp, _vp, _vp]),
    "fuelgpu_kino_search_batch": (C.c_int, [_vp, _i32, _vp, _vp, _vp, _vp, C.POINTER(FuelKinoParams), _vp, _vp, _vp,
                                            _vp, _i32, _vp, _vp]),
    "fuelgpu_kino_search_batch_dev": (C.c_int, [_vp, _i32, _vp, _vp, _vp, _vp, _vp, C.POINTER(FuelKinoParams), _vp,
                                                _vp, _vp, _vp, _i32, _vp, _vp]),
}

_lib = None


def lib():
    """Load libfuelgpu.so; raise loudly if it has not been built (no fallback)."""
    global _lib
    if _lib is None:
        if not os.path.exists(SO):
            raise FuelGpuError(ENODEVICE, "libfuelgpu.so is not built (run `python -m fuel_b200.build` "
                               "or __graft_entry__.build()); there is no CPU fallback")
        L = C.CDLL(SO)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(L, name)  # AttributeError = the library does not export what the header declares
            fn.restype = res
            fn.argtypes = args
        _lib = L
    return _lib


def check(rc, handle=None):
    if rc != 0:
        msg = lib().fuelgpu_last_error(handle)
        raise FuelGpuError(rc, msg.decode() if msg else "")
    return rc


def ptr(a):
    """numpy array (or None) -> void*"""
    if a is None:
        return None
    return a.ctypes.data_as(C.c_void_p)
