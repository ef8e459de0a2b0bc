"""fuel_b200 -- H100-native (sm_90a) drop-in for FUEL's per-replan hot path.

ESDF update (SDFMap::updateESDF3d), frontier sweep / clustering / PCA split
(FrontierFinder::searchFrontiers) and the batched B-spline cost/gradient
(BsplineOptimizer::combineCost), as hand-written CUDA behind a C ABI (include/fuelgpu.h).
The classes here mirror the reference's public C++ surface for that path.  No CPU fallback:
importing works anywhere, but every operation needs libfuelgpu.so and an sm_90 device.
"""
from ._lib import FuelGpuError, lib  # noqa: F401
from .bspline_optimizer import BsplineOptimizer  # noqa: F401
from .frontier_finder import Frontier, FrontierFinder  # noqa: F401
from .non_uniform_bspline import NonUniformBspline  # noqa: F401
from .sdf_map import EDTEnvironment, SDFMap  # noqa: F401
from .view_node import ViewNode  # noqa: F401

__all__ = ["SDFMap", "EDTEnvironment", "FrontierFinder", "Frontier", "BsplineOptimizer", "NonUniformBspline", "ViewNode",
           "FuelGpuError", "lib"]
