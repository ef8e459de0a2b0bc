"""Host-side mirror of fast_planner::SDFMap and EDTEnvironment over the C ABI.

Same method names, argument meaning and sentinel behaviour as
plan_env/include/plan_env/sdf_map.h:27-84 and plan_env/include/plan_env/edt_environment.h:21-51
(file:line under /root/reference/fuel_planner/).  All voxel-scale work runs in libfuelgpu
(hand-written sm_90a CUDA); this class owns the host copies the reference's random
single-point readers need (occupancy bytes, and the ESDF after `download()`).
"""
import ctypes as C
import math

import numpy as np

from . import _lib
from ._lib import FuelGridDesc, check, lib, ptr


def logit(p):
    return math.log(p / (1 - p))  # sdf_map.cpp:50


class SDFMap:
    UNKNOWN, FREE, OCCUPIED = 0, 1, 2  # sdf_map.h:32

    def __init__(self, voxel_num, resolution, origin, box_min=None, box_max=None, optimistic=False,
                 signed_dist=False, p_min=0.12, p_occ=0.80, default_dist=0.0, device=0, map_size=None):
        """initMap (sdf_map.cpp:12-93) with the ROS parameters passed explicitly.

        voxel_num = map_voxel_num_, origin = map_origin_, box_min/box_max = box_mind_/box_maxd_
        in metres (default: the whole map, sdf_map.cpp:79-82)."""
        self.map_voxel_num_ = np.asarray(voxel_num, dtype=np.int32)
        self.resolution_ = float(resolution)
        self.resolution_inv_ = 1 / self.resolution_
        self.map_origin_ = np.asarray(origin, dtype=np.float64)
        self.map_min_boundary_ = self.map_origin_.copy()
        # map_size_ (sdf_map/map_size_x,y,z, sdf_map.cpp:34): map_max_boundary_ = origin + map_size_, which need not equal
        # n * resolution bit for bit (n = ceil(size / resolution)); default: n * resolution
        self.map_size_ = (self.map_voxel_num_ * self.resolution_ if map_size is None
                          else np.asarray(map_size, dtype=np.float64))
        self.map_max_boundary_ = self.map_origin_ + self.map_size_
        self.box_mind_ = np.asarray(self.map_min_boundary_ if box_min is None else box_min, dtype=np.float64)
        self.box_maxd_ = np.asarray(self.map_max_boundary_ if box_max is None else box_max, dtype=np.float64)
        self.box_min_ = self.posToIndex(self.box_mind_)
        self.box_max_ = self.posToIndex(self.box_maxd_)
        self.optimistic_ = bool(optimistic)
        self.signed_dist_ = bool(signed_dist)
        self.clamp_min_log_ = logit(p_min)
        self.min_occupancy_log_ = logit(p_occ)
        self.default_dist_ = float(default_dist)
        shape = tuple(int(v) for v in self.map_voxel_num_)
        self.shape = shape
        # host mirrors of MapData (sdf_map.h:107-125)
        self.occupancy_buffer_inflate_ = np.zeros(shape, dtype=np.int8)
        self.occupancy_tri_ = np.zeros(shape, dtype=np.uint8)  # getOccupancy() of occupancy_buffer_
        self.distance_buffer_ = None  # filled by download()
        self.local_bound_min_ = np.zeros(3, dtype=np.int32)
        self.local_bound_max_ = self.map_voxel_num_ - 1
        self.update_min_ = np.zeros(3)
        self.update_max_ = np.zeros(3)
        self.reset_updated_box_ = True
        self._fusion = None
        self._camera = None
        self._fused = False

        d = FuelGridDesc()
        for i in range(3):
            d.n[i] = shape[i]
            d.origin[i] = self.map_origin_[i]
            d.box_mind[i] = self.box_mind_[i]
            d.box_maxd[i] = self.box_maxd_[i]
            d.map_size[i] = 0.0 if map_size is None else float(self.map_size_[i])
        d.resolution = self.resolution_
        self._desc = d
        h = C.c_void_p()
        check(lib().fuelgpu_map_create(C.byref(d), int(device), C.byref(h)))
        self._h = h
        self.device = int(device)
        # the occupancy mirrors are sized once here (initMap): page-lock them for the H2D leg
        self._pinned = []
        for a in (self.occupancy_buffer_inflate_, self.occupancy_tri_):
            self.pin(a)

    def pin(self, arr):
        """cudaHostRegister a long-lived numpy buffer (full PCIe rate for upload/download)."""
        if lib().fuelgpu_host_register(ptr(arr), arr.nbytes) == 0:
            self._pinned.append(arr)

    # ---- lifetime -------------------------------------------------------------------
    def close(self):
        if getattr(self, "_h", None):
            for a in getattr(self, "_pinned", []):
                lib().fuelgpu_host_unregister(ptr(a))
            self._pinned = []
            lib().fuelgpu_map_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @property
    def handle(self):
        return self._h

    def set_stream(self, cuda_stream):
        check(lib().fuelgpu_map_set_stream(self._h, C.c_void_p(cuda_stream)), self._h)

    def synchronize(self):
        check(lib().fuelgpu_map_synchronize(self._h), self._h)

    def last_timing(self):
        ms = (C.c_float * 8)()
        check(lib().fuelgpu_map_last_timing(self._h, ms), self._h)
        return dict(esdf=ms[0], frontier=ms[1], bspline=ms[2], upload=ms[3], download=ms[4], check=ms[5], param=ms[6], poly=ms[7])

    def last_timeline(self):
        """(start, end) in ms after the start of the last upload, per stage."""
        t0, t1 = (C.c_float * 8)(), (C.c_float * 8)()
        check(lib().fuelgpu_map_last_timeline(self._h, t0, t1), self._h)
        names = ("esdf", "frontier", "bspline", "upload", "download", "check", "param", "poly")
        return {k: (t0[i], t1[i]) for i, k in enumerate(names)}

    def launch_count(self):
        n = C.c_int64()
        check(lib().fuelgpu_map_launch_count(self._h, C.byref(n)), self._h)
        return n.value

    def device_ptrs(self):
        occ, dist, flag = C.c_void_p(), C.c_void_p(), C.c_void_p()
        check(lib().fuelgpu_map_device_ptrs(self._h, C.byref(occ), C.byref(dist), C.byref(flag)), self._h)
        return occ.value, dist.value, flag.value

    # ---- index helpers (sdf_map.h:127-192) ---------------------------------------------
    def posToIndex(self, pos):
        return np.floor((np.asarray(pos, dtype=np.float64) - self.map_origin_) *
                        self.resolution_inv_).astype(np.int32)

    def indexToPos(self, idx):
        return (np.asarray(idx) + 0.5) * self.resolution_ + self.map_origin_

    def boundIndex(self, idx):
        return np.maximum(np.minimum(np.asarray(idx), self.map_voxel_num_ - 1), 0).astype(np.int32)

    def toAddress(self, idx):
        idx = np.asarray(idx)
        return (idx[..., 0] * self.shape[1] + idx[..., 1]) * self.shape[2] + idx[..., 2]

    def isInMap(self, p):
        p = np.asarray(p)
        if p.dtype.kind == "f":
            return bool(np.all(p >= self.map_min_boundary_ + 1e-4) and np.all(p <= self.map_max_boundary_ - 1e-4))
        return bool(np.all(p >= 0) and np.all(p <= self.map_voxel_num_ - 1))

    def isInBox(self, p):
        p = np.asarray(p)
        if p.dtype.kind == "f":
            return bool(np.all(p > self.box_mind_) and np.all(p < self.box_maxd_))
        return bool(np.all(p >= self.box_min_) and np.all(p < self.box_max_))

    def boundBox(self, low, up):
        return np.maximum(low, self.box_mind_), np.minimum(up, self.box_maxd_)

    def getResolution(self):
        return self.resolution_

    def getVoxelNum(self):
        return int(np.prod(self.map_voxel_num_))

    def getRegion(self):
        return self.map_origin_.copy(), self.map_voxel_num_ * self.resolution_

    def getBox(self):
        return self.box_mind_.copy(), self.box_maxd_.copy()

    def getUpdatedBox(self, reset=False):
        """sdf_map.cpp:491-495; once inputPointCloud has run the box lives in the device handle."""
        if self._fused:
            bmin, bmax = np.zeros(3), np.zeros(3)
            check(lib().fuelgpu_map_get_updated_box(self._h, ptr(bmin), ptr(bmax), 1 if reset else 0), self._h)
            return bmin, bmax
        bmin, bmax = self.update_min_.copy(), self.update_max_.copy()
        if reset:
            self.reset_updated_box_ = True
        return bmin, bmax

    # ---- occupancy fusion (sdf_map.cpp:259-345) ---------------------------------------------
    def setFusionParams(self, p_hit=0.65, p_miss=0.35, p_min=0.12, p_max=0.90, p_occ=0.80, max_ray_length=4.5,
                        local_bound_inflate=0.5):
        """sdf_map/* parameters read in initMap (sdf_map.cpp:19-47); defaults algorithm.xml:39-50."""
        fp = _lib.FuelFusionParams()
        fp.p_hit, fp.p_miss, fp.p_min, fp.p_max, fp.p_occ = p_hit, p_miss, p_min, p_max, p_occ
        fp.max_ray_length, fp.local_bound_inflate = max_ray_length, local_bound_inflate
        self._fusion = fp
        self.clamp_min_log_, self.min_occupancy_log_ = logit(p_min), logit(p_occ)

    def inputPointCloud(self, points, point_num, camera_pos):
        """inputPointCloud(points, point_num, camera_pos), sdf_map.cpp:259-345: fuses one depth frame into the
        device-resident log-odds volume and sets local_bound_min_/max_ for clearAndInflateLocalMap/updateESDF3d."""
        if self._fusion is None:
            self.setFusionParams()
        pts = np.ascontiguousarray(points, dtype=np.float32)
        assert pts.ndim == 2 and pts.shape[1] in (3, 4) and pts.shape[0] >= point_num  # [n,4] = pcl::PointXYZ layout
        cam = np.ascontiguousarray(camera_pos, dtype=np.float64)
        lo, hi = np.zeros(3, np.int32), np.zeros(3, np.int32)
        check(lib().fuelgpu_map_input_point_cloud(self._h, ptr(pts), int(point_num), int(pts.shape[1]), ptr(cam),
                                                  C.byref(self._fusion),
                                                  ptr(lo), ptr(hi)), self._h)
        if point_num > 0:
            self.local_bound_min_, self.local_bound_max_ = lo, hi
            self._fused = True

    def setCameraParams(self, fx=387.229248046875, fy=387.229248046875, cx=321.04638671875, cy=243.44969177246094,
                        k_depth_scaling_factor=1000.0, depth_filter_maxdist=5.0, depth_filter_mindist=0.2,
                        depth_filter_margin=2, skip_pixel=2):
        """map_ros/* parameters (map_ros.cpp:24-37); defaults exploration.launch:38-41, algorithm.xml:61-69."""
        c = _lib.FuelCameraParams()
        c.fx, c.fy, c.cx, c.cy = fx, fy, cx, cy
        c.k_depth_scaling_factor, c.depth_filter_maxdist, c.depth_filter_mindist = (
            k_depth_scaling_factor, depth_filter_maxdist, depth_filter_mindist)
        c.depth_filter_margin, c.skip_pixel = depth_filter_margin, skip_pixel
        self._camera = c

    def inputDepthImage(self, depth, camera_R, camera_pos):
        """MapROS::depthPoseCallback's proessDepthImage + inputPointCloud (map_ros.cpp:139-140,176-215) in one device
        call.  depth = uint16 [rows, cols]; camera_R = camera_q_.toRotationMatrix().  -> proj_points_cnt"""
        if self._fusion is None:
            self.setFusionParams()
        if self._camera is None:
            self.setCameraParams()
        img = np.ascontiguousarray(depth, dtype=np.uint16)
        R = np.ascontiguousarray(camera_R, dtype=np.float64).reshape(9)
        cam = np.ascontiguousarray(camera_pos, dtype=np.float64)
        lo, hi = np.zeros(3, np.int32), np.zeros(3, np.int32)
        cnt = C.c_int32(0)
        check(lib().fuelgpu_map_input_depth_image(self._h, ptr(img), img.shape[0], img.shape[1], C.byref(self._camera), ptr(R),
                                                  ptr(cam), C.byref(self._fusion), ptr(lo), ptr(hi), C.byref(cnt)), self._h)
        if cnt.value > 0:
            self.local_bound_min_, self.local_bound_max_ = lo, hi
            self._fused = True
        return cnt.value

    def getLogOdds(self):
        """occupancy_buffer_ (fp64 log-odds) from the device."""
        out = np.empty(self.shape, dtype=np.float64)
        check(lib().fuelgpu_map_get_logodds(self._h, ptr(out)), self._h)
        return out

    def setLogOdds(self, logodds):
        if self._fusion is None:
            self.setFusionParams()
        lo = np.ascontiguousarray(logodds, dtype=np.float64).reshape(self.shape)
        check(lib().fuelgpu_map_set_logodds(self._h, ptr(lo), self._fusion.p_min, self._fusion.p_occ), self._h)
        self._fused = True

    # ---- occupancy (host mirrors; offline recipe of plan_manage/test/compare_topo.cpp:122-133) --
    def resetBuffer(self):
        self.occupancy_buffer_inflate_[...] = 0  # sdf_map.cpp:95-114
        self.local_bound_min_ = np.zeros(3, dtype=np.int32)
        self.local_bound_max_ = (self.map_voxel_num_ - 1).astype(np.int32)

    def setOccupied(self, pos, occ=1):
        """sdf_map.h:210-215, vectorised over [n,3] positions."""
        pos = np.asarray(pos, dtype=np.float64).reshape(-1, 3)
        ok = np.all(pos >= self.map_min_boundary_ + 1e-4, axis=1) & np.all(
            pos <= self.map_max_boundary_ - 1e-4, axis=1)
        idx = self.posToIndex(pos[ok])
        self.occupancy_buffer_inflate_[idx[:, 0], idx[:, 1], idx[:, 2]] = occ

    def setOccupancyBuffer(self, logodds=None, tristate=None):
        """Set occupancy_buffer_ either as log-odds (thresholded like getOccupancy,
        sdf_map.h:194-200) or directly as its tri-state."""
        if (logodds is None) == (tristate is None):
            raise ValueError("give exactly one of logodds / tristate")
        if tristate is not None:
            self.occupancy_tri_[...] = np.asarray(tristate, dtype=np.uint8).reshape(self.shape)
        else:
            lo = np.asarray(logodds, dtype=np.float64).reshape(self.shape)
            t = np.full(self.shape, self.FREE, dtype=np.uint8)
            t[lo < self.clamp_min_log_ - 1e-3] = self.UNKNOWN
            t[lo > self.min_occupancy_log_] = self.OCCUPIED
            self.occupancy_tri_[...] = t

    def getOccupancy(self, p):
        idx = self.posToIndex(p) if np.asarray(p).dtype.kind == "f" else np.asarray(p)
        if not self.isInMap(idx.astype(np.int64)):
            return -1
        return int(self.occupancy_tri_[idx[0], idx[1], idx[2]])

    def getInflateOccupancy(self, p):
        idx = self.posToIndex(p) if np.asarray(p).dtype.kind == "f" else np.asarray(p)
        if not self.isInMap(idx.astype(np.int64)):
            return -1
        return int(self.occupancy_buffer_inflate_[idx[0], idx[1], idx[2]])

    def upload(self, bmin=None, bmax=None, logodds=None, wait=True):
        """H2D of the occupancy state.  With `logodds` the device thresholds the fp64 buffer
        itself (9 B/voxel ingest); otherwise the host tri-state byte is sent (2 B/voxel).
        wait=False queues the copies and returns: leave the mirrors alone until synchronize()."""
        fn = lib().fuelgpu_map_upload_occupancy if wait else lib().fuelgpu_map_upload_occupancy_async
        bmin_a = None if bmin is None else np.ascontiguousarray(bmin, dtype=np.int32)
        bmax_a = None if bmax is None else np.ascontiguousarray(bmax, dtype=np.int32)
        inf = np.ascontiguousarray(self.occupancy_buffer_inflate_)
        if logodds is not None:
            lo = np.ascontiguousarray(logodds, dtype=np.float64)
            check(fn(self._h, ptr(inf), ptr(lo), None, self.clamp_min_log_,
                                                     self.min_occupancy_log_, ptr(bmin_a), ptr(bmax_a)), self._h)
        else:
            tri = np.ascontiguousarray(self.occupancy_tri_)
            check(fn(self._h, ptr(inf), None, ptr(tri), self.clamp_min_log_,
                                                     self.min_occupancy_log_, ptr(bmin_a), ptr(bmax_a)), self._h)

    def clearAndInflateLocalMap(self, obstacles_inflation=0.199, virtual_ceil_height=-10.0):
        """sdf_map.cpp:364-472 on the resident occupancy byte over [local_bound_min_, local_bound_max_];
        defaults = exploration_manager/launch/algorithm.xml:38,51.  The host mirrors are refreshed."""
        inf_step = int(math.ceil(obstacles_inflation / self.resolution_))  # :436
        ceil_id = -1
        if virtual_ceil_height > -0.5:  # :462
            ceil_id = int(math.floor((virtual_ceil_height - self.map_origin_[2]) * self.resolution_inv_))
        bmin = np.ascontiguousarray(self.local_bound_min_, dtype=np.int32)
        bmax = np.ascontiguousarray(self.local_bound_max_, dtype=np.int32)
        check(lib().fuelgpu_map_inflate(self._h, ptr(bmin), ptr(bmax), inf_step, ceil_id), self._h)
        check(lib().fuelgpu_map_download_occupancy(self._h, ptr(self.occupancy_buffer_inflate_),
                                                   ptr(self.occupancy_tri_)), self._h)

    # ---- ESDF ------------------------------------------------------------------------------
    def updateESDF3d(self):
        """sdf_map.cpp:152-241 over [local_bound_min_, local_bound_max_]."""
        flags = (_lib.ESDF_OPTIMISTIC if self.optimistic_ else 0) | (_lib.ESDF_SIGNED if self.signed_dist_ else 0)
        bmin = np.ascontiguousarray(self.local_bound_min_, dtype=np.int32)
        bmax = np.ascontiguousarray(self.local_bound_max_, dtype=np.int32)
        check(lib().fuelgpu_esdf_update(self._h, ptr(bmin), ptr(bmax), flags), self._h)

    def download(self, bmin=None, bmax=None, dtype=np.float32, wait=True):
        """Mirror distance_buffer_ to the host for getDistance().  wait=False (float32 only) queues
        the copy behind the ESDF update and returns; the mirror is valid after synchronize()."""
        if self.distance_buffer_ is None or self.distance_buffer_.dtype != dtype:
            self.distance_buffer_ = np.full(self.shape, self.default_dist_, dtype=dtype)
            self.pin(self.distance_buffer_)
        bmin_a = None if bmin is None else np.ascontiguousarray(bmin, dtype=np.int32)
        bmax_a = None if bmax is None else np.ascontiguousarray(bmax, dtype=np.int32)
        if dtype == np.float32 and not wait:
            check(lib().fuelgpu_esdf_download_async(self._h, ptr(bmin_a), ptr(bmax_a), ptr(self.distance_buffer_)), self._h)
        elif dtype == np.float32:
            check(lib().fuelgpu_esdf_download(self._h, ptr(bmin_a), ptr(bmax_a), ptr(self.distance_buffer_), None), self._h)
        else:
            check(lib().fuelgpu_esdf_download(self._h, ptr(bmin_a), ptr(bmax_a), None, ptr(self.distance_buffer_)), self._h)
        return self.distance_buffer_

    def getDistance(self, p):
        """sdf_map.h:228-237 on the host mirror (call download() after updateESDF3d)."""
        idx = self.posToIndex(p) if np.asarray(p).dtype.kind == "f" else np.asarray(p)
        if not self.isInMap(idx.astype(np.int64)):
            return -1.0
        return float(self.distance_buffer_[idx[0], idx[1], idx[2]])

    def getDistWithGrad(self, pos):
        """sdf_map.cpp:497-536 for [n,3] positions, evaluated on the device ESDF."""
        pos = np.ascontiguousarray(pos, dtype=np.float64).reshape(-1, 3)
        n = pos.shape[0]
        d = np.empty(n, dtype=np.float64)
        g = np.empty((n, 3), dtype=np.float64)
        check(lib().fuelgpu_esdf_sample(self._h, n, ptr(pos), ptr(d), ptr(g)), self._h)
        return d, g


class EDTEnvironment:
    """edt_environment.h:21-51: the facade every consumer reaches the map through."""

    def __init__(self):
        self.sdf_map_ = None

    def setMap(self, sdf_map):
        self.sdf_map_ = sdf_map
        self.resolution_inv_ = 1 / sdf_map.getResolution()

    def evaluateEDTWithGrad(self, pos, time=-1.0):
        """edt_environment.cpp:78-87 -- pure pass-through to getDistWithGrad (`time` unused)."""
        return self.sdf_map_.getDistWithGrad(pos)

    def evaluateCoarseEDT(self, pos, time=-1.0):
        return self.sdf_map_.getDistance(np.asarray(pos, dtype=np.float64))
