"""discregrid_b200 -- H100-native (sm_90a) implementation of Discregrid's data-parallel hot path.

Host mirror (Python) of the reference's C++ classes over the C-ABI in include/discregrid_b200.h:
TriangleMesh, TriangleMeshDistance, CubicLagrangeDiscreteGrid.  Importing this package loads
discregrid_b200/lib/libdiscregrid_b200.so and fails if it has not been built; there is no CPU fallback.
"""
from . import _capi
from ._capi import DiscregridError, DBL_MAX, LIB_PATH
from .mesh import TriangleMesh, bumpy_torus, uv_sphere, box
from .distance import TriangleMeshDistance, MeshSignedDistance, MeshDistanceBand, NearestEntity, NearestResult, Result
from .grid import (CubicLagrangeDiscreteGrid, DensityMapFunction, VolumeMapFunction, DeviceFunction, DeviceNodePredicate, DeviceSamplePredicate, grid_desc,
                   generate_sdf_domain)

__all__ = ["TriangleMesh", "TriangleMeshDistance", "MeshSignedDistance", "MeshDistanceBand", "NearestEntity", "NearestResult", "Result",
           "CubicLagrangeDiscreteGrid", "DensityMapFunction", "VolumeMapFunction", "DeviceFunction", "DeviceSamplePredicate", "DeviceNodePredicate", "grid_desc",
           "generate_sdf_domain", "DiscregridError",
           "DBL_MAX", "LIB_PATH", "bumpy_torus", "uv_sphere", "box"]


def device_count():
    return _capi.lib.dg_device_count()


def selftest():
    _capi.check(_capi.lib.dg_selftest())


def kernel_launch_count():
    return int(_capi.lib.dg_kernel_launch_count())
