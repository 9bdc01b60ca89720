"""ctypes binding of libdiscregrid_b200.so -- the C-ABI declared in include/discregrid_b200.h.

This is the *reference-side binding a maintainer would add* in Python form (the reference itself is C++ and has
no FFI; see INTEGRATION.md for the C++ one).  There is deliberately no fallback: if the shared library is missing
the import fails, and if no CUDA device is present every compute call raises DiscregridError(DG_ERR_NO_DEVICE).
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
# DISCREGRID_B200_LIB: tuning builds of the same library (tools/build_variants.py); never a different implementation
LIB_PATH = os.environ.get("DISCREGRID_B200_LIB") or os.path.join(_HERE, "lib", "libdiscregrid_b200.so")

DG_OK, DG_ERR_INVALID, DG_ERR_NO_DEVICE, DG_ERR_CUDA, DG_ERR_NOMEM, DG_ERR_SELFTEST, DG_ERR_IO, DG_ERR_CALLBACK = 0, -1, -2, -3, -4, -5, -6, -7
DBL_MAX = 1.7976931348623157e308
DG_SIGN_PSEUDONORMAL, DG_SIGN_WINDING = 0, 1
DG_RAY_MISS, DG_RAY_ENTER, DG_RAY_LEAVE = 0, 1, 2
UINT32_MAX = 0xFFFFFFFF


class DiscregridError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f"[dg_status {code}] {msg}")
        self.code = code


class GridDesc(C.Structure):
    """dg_grid_desc"""
    _fields_ = [("domain_min", C.c_double * 3), ("domain_max", C.c_double * 3), ("resolution", C.c_uint32 * 3),
                ("_pad", C.c_uint32), ("cell_size", C.c_double * 3), ("inv_cell_size", C.c_double * 3)]


if not os.path.exists(LIB_PATH):
    raise ImportError(f"{LIB_PATH} is missing: build it with `make lib` (or __graft_entry__.build()); "
                      "discregrid_b200 has no pure-Python / CPU fallback")

lib = C.CDLL(LIB_PATH)
# The test suite can build the whole library with every kernel emulated on the CPU (tests/emu -> build/bin/libdgemu.so) to rehearse the GPU
# tests.  That build is test infrastructure: the package refuses it unless the rehearsal says so explicitly, so that no user -- and no
# benchmark -- can end up on it by accident.  There is no CPU fallback.
if hasattr(lib, "emu_mesh_create") and os.environ.get("DG_ALLOW_EMULATED_LIBRARY") != "1":
    raise ImportError(f"{LIB_PATH} is the CPU-emulated TEST build of the library (tests/emu); discregrid_b200 only runs on the CUDA build "
                      "(set DG_ALLOW_EMULATED_LIBRARY=1 only from the test rehearsal)")

# True for the CPU-emulated test build: "device" pointers are host memory there
EMULATED = hasattr(lib, "emu_mesh_create")

_dp, _u32p, _i32p, _u64p, _vp = (C.POINTER(C.c_double), C.POINTER(C.c_uint32), C.POINTER(C.c_int32),
                                 C.POINTER(C.c_uint64), C.c_void_p)
_gp = C.POINTER(GridDesc)

# the device callbacks (dg_device_function, dg_device_sample_predicate, dg_device_node_predicate); every pointer as an integer address
DEVICE_FUNCTION = C.CFUNCTYPE(C.c_int, _vp, _vp, _vp, C.c_uint64, _vp, _vp)
DEVICE_SAMPLE_PREDICATE = C.CFUNCTYPE(C.c_int, _vp, _vp, C.c_uint64, _vp, _vp)
DEVICE_NODE_PREDICATE = C.CFUNCTYPE(C.c_int, _vp, _vp, _vp, C.c_uint64, _vp, _vp)

# name -> (restype, argtypes); every symbol of include/discregrid_b200.h
SIGNATURES = {
    "dg_abi_version": (C.c_int, []),
    "dg_last_error": (C.c_char_p, []),
    "dg_device_count": (C.c_int, []),
    "dg_set_device": (C.c_int, [C.c_int]),
    "dg_selftest": (C.c_int, []),
    "dg_fp64_rate_probe": (C.c_int, [_dp]),
    "dg_kernel_launch_count": (C.c_uint64, []),
    "dg_kernel_launch_count_reset": (None, []),
    "dg_grid_init": (C.c_int, [_dp, _dp, _u32p, _gp]),
    "dg_grid_num_nodes": (C.c_int, [_u32p, _u64p]),
    "dg_generate_sdf_domain": (C.c_int, [_dp, C.c_uint64, _dp, _dp]),
    "dg_obj_read": (C.c_int, [C.c_char_p, C.POINTER(_dp), _u64p, C.POINTER(_u32p), _u64p]),
    "dg_obj_free": (None, [_dp, _u32p]),
    "dg_mesh_create": (C.c_int, [_dp, C.c_uint64, _u32p, C.c_uint64, C.POINTER(_vp)]),
    "dg_mesh_destroy": (C.c_int, [_vp]),
    "dg_mesh_info": (C.c_int, [_vp, _u64p]),
    "dg_mesh_tree": (C.c_int, [_vp, _dp, _i32p]),
    "dg_mesh_pseudonormals": (C.c_int, [_vp, _dp, _dp, _dp]),
    "dg_mesh_set_sign_mode": (C.c_int, [_vp, C.c_int, C.c_double]),
    "dg_mesh_winding_number": (C.c_int, [_vp, _dp, C.c_uint64, C.c_double, _dp]),
    "dg_mesh_winding_number_device": (C.c_int, [_vp, _vp, C.c_uint64, C.c_double, _vp, _vp]),
    "dg_mesh_refit": (C.c_int, [_vp, _dp, C.c_uint64]),
    "dg_mesh_refit_device": (C.c_int, [_vp, _vp, C.c_uint64, _vp]),
    "dg_mesh_raycast": (C.c_int, [_vp, _dp, _dp, C.c_uint64, C.c_double, C.c_double, _dp, _i32p, _dp, _i32p]),
    "dg_mesh_raycast_device": (C.c_int, [_vp, _vp, _vp, C.c_uint64, C.c_double, C.c_double, _vp, _vp, _vp, _vp, _vp]),
    "dg_mesh_distance": (C.c_int, [_vp, _dp, C.c_uint64, C.c_int, _dp, _dp, _i32p, _i32p]),
    "dg_mesh_distance_device": (C.c_int, [_vp, _vp, C.c_uint64, C.c_int, _vp, _vp, _vp, _vp, _vp]),
    "dg_mesh_distance_bary": (C.c_int, [_vp, _dp, C.c_uint64, C.c_int, _dp, _dp, _i32p, _i32p, _dp]),
    "dg_mesh_distance_bary_device": (C.c_int, [_vp, _vp, C.c_uint64, C.c_int, _vp, _vp, _vp, _vp, _vp, _vp]),
    "dg_mesh_distance_vjp": (C.c_int, [_vp, C.c_uint64, _dp, _dp, _dp, _i32p, _dp, _dp, _dp, _dp]),
    "dg_mesh_distance_vjp_device": (C.c_int, [_vp, C.c_uint64, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "dg_mesh_raycast_vjp": (C.c_int, [_vp, C.c_uint64, _dp, _dp, _i32p, _dp, _dp, _dp, _dp, _dp, _dp, _dp]),
    "dg_mesh_raycast_vjp_device": (C.c_int, [_vp, C.c_uint64, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "dg_field_raycast_vjp": (C.c_int, [_vp, C.c_uint64, _dp, _dp, _dp, _i32p, _dp, _dp, _dp, _dp, _dp]),
    "dg_field_raycast_vjp_device": (C.c_int, [_vp, C.c_uint64, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "dg_sample_sdf": (C.c_int, [_vp, _gp, C.c_double, C.c_uint64, C.c_uint64, _dp]),
    "dg_add_function_sdf": (C.c_int, [_vp, _gp, C.c_double, _dp, _u32p, _u32p, _dp]),
    "dg_mesh_group_create": (C.c_int, [_vp, C.c_int, C.POINTER(C.c_int), C.POINTER(_vp)]),
    "dg_mesh_group_destroy": (C.c_int, [_vp]),
    "dg_mesh_group_size": (C.c_int, [_vp]),
    "dg_add_function_sdf_multi": (C.c_int, [_vp, _gp, C.c_double, _dp, _u32p, _u32p, _dp]),
    "dg_sample_sdf_multi_device": (C.c_int, [_vp, _gp, C.c_double, C.POINTER(_vp)]),
    "dg_sample_sdf_device": (C.c_int, [_vp, _gp, C.c_double, C.c_uint64, C.c_uint64, _vp, _vp]),
    "dg_sample_sdf_band_device": (C.c_int, [_vp, _gp, C.c_double, C.c_double, C.c_uint64, C.c_uint64, _vp, _vp]),
    "dg_add_function_sdf_band": (C.c_int, [_vp, _gp, C.c_double, C.c_double, _dp, _u32p, _u32p, _dp]),
    "dg_slab_ranges": (C.c_int, [_gp, C.c_uint32, C.c_uint32, _u64p]),
    "dg_sample_sdf_slab_device": (C.c_int, [_vp, _gp, C.c_double, C.c_uint32, C.c_uint32, _vp, _vp]),
    "dg_interleaved_slot_elems": (C.c_int, [_gp, C.c_uint32, _u64p]),
    "dg_sample_sdf_interleaved_device": (C.c_int, [_vp, _gp, C.c_double, C.c_uint32, C.c_uint32, _vp, _vp]),
    "dg_interleaved_unpack_device": (C.c_int, [_gp, C.c_uint32, _vp, _vp, _vp]),
    "dg_interleaved_node_slots": (C.c_int, [_gp, C.c_uint32, C.c_uint64, C.c_uint64, _u32p, _u64p]),
    "dg_node_positions": (C.c_int, [_gp, C.c_uint64, C.c_uint64, _dp]),
    "dg_build_cells": (C.c_int, [_u32p, C.c_uint64, C.c_uint64, _u32p]),
    "dg_field_create": (C.c_int, [_gp, _dp, C.c_uint64, _u32p, C.c_uint64, _u32p, C.POINTER(_vp)]),
    "dg_field_create_device": (C.c_int, [_gp, _vp, C.c_uint64, _vp, C.POINTER(_vp)]),
    "dg_field_create_trainable": (C.c_int, [_gp, _dp, C.c_uint64, _u32p, C.c_uint64, _u32p, C.POINTER(_vp)]),
    "dg_field_set_nodes": (C.c_int, [_vp, _dp, C.c_uint64]),
    "dg_field_set_nodes_device": (C.c_int, [_vp, _vp, C.c_uint64, _vp]),
    "dg_interpolate_vjp": (C.c_int, [_vp, _dp, C.c_uint64, _dp, _dp, _dp]),
    "dg_interpolate_vjp_device": (C.c_int, [_vp, _vp, C.c_uint64, _vp, _vp, _vp, _vp]),
    "dg_field_destroy": (C.c_int, [_vp]),
    "dg_field_info": (C.c_int, [_vp, _u64p]),
    "dg_interpolate_batch": (C.c_int, [_vp, _dp, C.c_uint64, _dp, _dp]),
    "dg_interpolate_batch_device": (C.c_int, [_vp, _vp, C.c_uint64, _vp, _vp, _vp]),
    "dg_interpolate_hessian_batch": (C.c_int, [_vp, _dp, C.c_uint64, _dp, _dp, _dp]),
    "dg_interpolate_hessian_batch_device": (C.c_int, [_vp, _vp, C.c_uint64, _vp, _vp, _vp, _vp]),
    "dg_shape_functions": (C.c_int, [_dp, C.c_uint64, _dp, _dp]),
    "dg_density_map": (C.c_int, [_vp, C.c_double, C.c_double, C.c_int, C.c_uint64, C.c_uint64, _dp]),
    "dg_reduce_field": (C.c_int, [_gp, _dp, C.c_uint64, C.POINTER(C.c_uint8), _u32p, C.c_uint64, _u32p, C.c_uint32, _u64p, _u64p, _dp]),
    "dg_density_map_device": (C.c_int, [_vp, C.c_double, C.c_double, C.c_int, C.c_uint64, C.c_uint64, _vp, _vp]),
    "dg_volume_map": (C.c_int, [_vp, C.c_double, C.c_double, C.c_int, C.c_uint64, C.c_uint64, _dp]),
    "dg_volume_map_device": (C.c_int, [_vp, C.c_double, C.c_double, C.c_int, C.c_uint64, C.c_uint64, _vp, _vp]),
    "dg_reduced_band_create": (C.c_int, [_vp, _gp, C.c_double, C.c_double, C.c_uint32, C.POINTER(_vp), _dp]),
    "dg_reduced_band_sizes": (C.c_int, [_vp, _u64p, _u64p]),
    "dg_reduced_band_copy": (C.c_int, [_vp, _dp, _u32p, _u32p]),
    "dg_reduced_band_destroy": (C.c_int, [_vp]),
    "dg_field_create_reduced": (C.c_int, [_vp, C.POINTER(_vp)]),
    "dg_isosurface_create": (C.c_int, [_vp, C.c_double, C.c_uint32, C.POINTER(_vp), _dp]),
    "dg_isosurface_sizes": (C.c_int, [_vp, _u64p, _u64p]),
    "dg_isosurface_copy": (C.c_int, [_vp, _dp, _u32p]),
    "dg_isosurface_copy_device": (C.c_int, [_vp, _vp, _vp, _vp]),
    "dg_isosurface_destroy": (C.c_int, [_vp]),
    "dg_isosurface_copy_edges": (C.c_int, [_vp, _u64p]),
    "dg_isosurface_copy_edges_device": (C.c_int, [_vp, _vp, _vp]),
    "dg_isosurface_vjp": (C.c_int, [_vp, C.c_double, C.c_uint32, C.c_uint64, _u64p, _dp, _dp]),
    "dg_isosurface_vjp_device": (C.c_int, [_vp, C.c_double, C.c_uint32, C.c_uint64, _vp, _vp, _vp, _vp]),
    "dg_field_raycast": (C.c_int, [_vp, _dp, _dp, C.c_uint64, C.c_double, C.c_double, C.c_double, _dp, _dp, _i32p]),
    "dg_field_raycast_device": (C.c_int, [_vp, _vp, _vp, C.c_uint64, C.c_double, C.c_double, C.c_double, _vp, _vp, _vp, _vp]),
    "dg_reduced_density_map_create": (C.c_int, [_gp, _dp, C.c_uint64, _u32p, C.c_uint64, _u32p, C.c_double, C.c_double, C.c_uint32,
                                                 C.POINTER(_vp), C.POINTER(_vp), _dp]),
    "dg_reduced_volume_map_create": (C.c_int, [_gp, _dp, C.c_uint64, _u32p, C.c_uint64, _u32p, C.c_double, C.c_double, C.c_uint32,
                                                C.POINTER(_vp), C.POINTER(_vp), _dp]),
    "dg_add_function_device": (C.c_int, [_gp, DEVICE_FUNCTION, _vp, DEVICE_SAMPLE_PREDICATE, _vp, C.c_uint64, _dp, _u32p, _u32p, _dp]),
    "dg_reduced_function_create": (C.c_int, [_gp, DEVICE_FUNCTION, _vp, DEVICE_SAMPLE_PREDICATE, _vp, DEVICE_NODE_PREDICATE, _vp, C.c_uint64,
                                              C.c_uint32, C.POINTER(_vp), _dp]),
    "dg_reduce_field_device": (C.c_int, [_gp, _dp, C.c_uint64, _u32p, C.c_uint64, DEVICE_NODE_PREDICATE, _vp, C.c_uint64, C.c_uint32,
                                          C.POINTER(_vp), _dp]),
}
for _name, (_res, _args) in SIGNATURES.items():
    _f = getattr(lib, _name)          # AttributeError here = the library does not export a declared symbol
    _f.restype, _f.argtypes = _res, _args


def check(rc):
    if rc != DG_OK:
        raise DiscregridError(rc, (lib.dg_last_error() or b"").decode("utf-8", "replace"))


def ptr(a, t):
    """numpy array -> typed pointer (None -> NULL)."""
    return None if a is None else a.ctypes.data_as(t)


F64P, U32P, I32P, U64P = _dp, _u32p, _i32p, _u64p
