"""Host mirror of Discregrid::DiscreteGrid / CubicLagrangeDiscreteGrid over the C-ABI.

Keeps the reference's members (m_domain, m_resolution, m_cell_size, m_inv_cell_size, m_n_cells, m_n_fields,
m_nodes, m_cells, m_cell_map -- discrete_grid.hpp:93-98, cubic_lagrange_discrete_grid.hpp:69-71) as numpy arrays so
that save()/load() stay byte-compatible with the reference's .cdf/.cdm files
(cubic_lagrange_discrete_grid.cpp:678-778), and routes the hot path to the GPU:

  addFunction(MeshSignedDistance)        -> dg_add_function_sdf  (K1, csrc/k1_sdf.cu)
  addFunction(MeshSignedDistance, pred=MeshDistanceBand)
                                         -> dg_add_function_sdf_band (K1 narrow band: DBL_MAX outside |distance| <= band)
  addReducedBandField(MeshSignedDistance, MeshDistanceBand)
                                         -> dg_reduced_band_create (the same band, then reduceField(always true), all on the GPU)
  addFunction(DensityMapFunction, pred)  -> dg_density_map       (K3, csrc/k3_density.cu)
  addReducedDensityMap(DensityMapFunction)
                                         -> dg_reduced_density_map_create (K3, then both of GenerateDensityMap's reduceField calls, on the GPU)
  addFunction(VolumeMapFunction)         -> dg_volume_map        (K3's volume-map kernel: SPH boundary volumes, not in the reference)
  addReducedVolumeMap(VolumeMapFunction) -> dg_reduced_volume_map_create (the volume map, then reduceField(0, p0) and reduceField(id, 0 <= v))
  addFunction(DeviceFunction, pred=DeviceSamplePredicate)
                                         -> dg_add_function_device (your torch code on batches of node positions made on the GPU)
  reduceField(field_id, DeviceNodePredicate)
                                         -> dg_reduce_field_device (your predicate on the GPU, then reduceField's passes there)
  addReducedFunction(DeviceFunction, DeviceSamplePredicate, DeviceNodePredicate)
                                         -> dg_reduced_function_create (addFunction + reduceField, the dense field kept on the GPU)
  interpolate(field_id, x[, gradient])   -> dg_interpolate_batch (K2, csrc/k2_interp.cu), batched over x; a float64 CUDA tensor x
                                            -> dg_interpolate_batch_device on torch's current stream (CUDA tensors out, autograd in x)
  interpolate(field_id, x, hessian=True) -> dg_interpolate_hessian_batch[_device] (K2's Hessian mode; second-order autograd in x)
  raycast(field_id, origins, directions) -> dg_field_raycast[_device] (K7: first crossings of a level set along rays and segments)
  interpolate(field_id, x, coefficients=c) -> dg_field_set_nodes_device + K2 on a trainable field, differentiable in c through
                                            dg_interpolate_vjp_device (K11, csrc/k11_field_grad.cu)
  isosurface(field_id, iso, s, device=True, coefficients=c)
                                         -> dg_field_set_nodes_device + K6 on the trainable field, the vertices differentiable in c through
                                            dg_isosurface_vjp_device (K13, csrc/k13_isosurface_grad.cu)

The reduced calls keep the handle they get from the library until the field's first device use, which builds the interpolation
field from it on the device (dg_field_create_reduced) instead of uploading the host copy again.

The reference's addFunction takes an opaque std::function.  The two functor types the reference's own tools build are recognised
and run on the library's kernels; a function of your own runs as your own GPU code when wrapped in DeviceFunction (and its
predicates in DeviceSamplePredicate / DeviceNodePredicate).  Any other callable raises TypeError; there is no hidden host loop.
"""
import contextlib
import ctypes as C
import math
import struct

import numpy as np

from . import _capi as capi
from . import _device
from .distance import MeshDistanceBand, MeshSignedDistance


class DensityMapFunction:
    """The (density_func, predicate) pair GenerateDensityMap passes to addFunction
    (cmd/generate_density_map/main.cpp:96-133): rho0 * int gamma(x+xi) W(xi) dxi over [-h,h]^3 with 16^3 Gauss points."""

    def __init__(self, sdf_field_id=0, smoothing_length=0.1, rest_density=1000.0, no_reduction=False):
        self.field_id, self.h, self.rho0, self.no_reduction = sdf_field_id, float(smoothing_length), float(rest_density), bool(no_reduction)


class VolumeMapFunction:
    """The volume map of Bender et al. 2019 (SPlisHSPlasH's boundary representation) as a recognisable function for addFunction:
    scale * the 16^3-point Gauss quadrature of an inside indicator gamma(d(x + xi)) over the ball |xi| <= h, on the SDF in field
    `sdf_field_id`, with GenerateDensityMap's sample predicate unless no_reduction (contract: DESIGN section 3, "Volume map")."""

    def __init__(self, sdf_field_id=0, smoothing_length=0.1, scale=0.8, no_reduction=False):
        self.field_id, self.h, self.scale, self.no_reduction = sdf_field_id, float(smoothing_length), float(scale), bool(no_reduction)


class DeviceFunction:
    """A function evaluated by your own GPU code, batch by batch: fn(x, keep) -> values.
    x: float64 tensor (n, 3), the positions indexToNodePosition(l) of a chunk of node ids, made on the GPU.  keep: uint8 tensor (n,) of the
    sample predicate's decisions for the same nodes (nonzero = sampled), or None without a predicate; nodes with keep == 0 may be skipped,
    they get DBL_MAX anyway.  values: float64 tensor (n,) on the same device.  Both tensors view the library's buffers (no copy) and are only
    valid during the call.  fn runs on the library's stream (torch.cuda.ExternalStream), which first waits for the torch stream that was current
    when the grid method was called, so fn sees every tensor computed before the call; plain torch operations inside fn are ordered with the
    library's own work.  So are the library's own queries on CUDA tensors, which run on torch's current stream: fn may be a function of a
    mesh or of an existing field, e.g. lambda x, k: md.signed_distance(x).distance or lambda x, k: other.interpolate(0, x) - r.  A field
    used inside fn should have its device field before the call (one interpolate on it is enough): making it synchronises the device, and
    inside fn that would stall every chunk's queued work."""

    def __init__(self, fn):
        if not callable(fn):
            raise TypeError("DeviceFunction wraps a callable fn(x, keep) -> float64 tensor")
        self.fn = fn


class DeviceSamplePredicate:
    """addFunction's sample predicate on the GPU: fn(x) -> bool tensor (n,); DBL_MAX is stored where it is False (:817)."""

    def __init__(self, fn):
        if not callable(fn):
            raise TypeError("DeviceSamplePredicate wraps a callable fn(x) -> bool tensor")
        self.fn = fn


class DeviceNodePredicate:
    """reduceField's predicate on the GPU: fn(x, values) -> bool tensor (n,); a node is kept where it is True and its value is not
    DBL_MAX (:1069-1074).  values: float64 tensor (n,), the field's coefficients of the chunk."""

    def __init__(self, fn):
        if not callable(fn):
            raise TypeError("DeviceNodePredicate wraps a callable fn(x, values) -> bool tensor")
        self.fn = fn


class _DeviceCallbacks:
    """The ctypes trampolines of one library call.  The first exception raised inside a callback is kept (the callback returns 1, the
    library stops with DG_ERR_CALLBACK) and re-raised by check()."""

    def __init__(self, func=None, sample=None, node=None):
        import torch
        self.torch = torch
        self.error = None
        # the caller's stream at the call: the library's stream waits for it before the first callback runs (work queued on it, e.g. the
        # weights of a model just trained, must be finished before fn reads it)
        self.caller_stream = None if capi.EMULATED else torch.cuda.current_stream()
        self.func = capi.DEVICE_FUNCTION(self._func(func.fn)) if func is not None else capi.DEVICE_FUNCTION()
        self.sample = capi.DEVICE_SAMPLE_PREDICATE(self._sample(sample.fn)) if sample is not None else capi.DEVICE_SAMPLE_PREDICATE()
        self.node = capi.DEVICE_NODE_PREDICATE(self._node(node.fn)) if node is not None else capi.DEVICE_NODE_PREDICATE()

    def check(self, rc):
        if self.error is not None:
            raise self.error
        capi.check(rc)

    def _view(self, addr, shape, typestr, dtype):
        """a tensor over library memory: CUDA memory through __cuda_array_interface__, host memory under the emulated test build"""
        count = math.prod(shape)
        if capi.EMULATED:
            buf = (C.c_char * (count * dtype.itemsize)).from_address(addr)
            return self.torch.frombuffer(buf, dtype=dtype).view(shape)

        class _Cai:
            __cuda_array_interface__ = {"shape": shape, "typestr": typestr, "data": (addr, False), "version": 3, "strides": None}
        return self.torch.as_tensor(_Cai(), device="cuda")

    def _stream(self, stream):
        if capi.EMULATED:
            return contextlib.nullcontext()
        ext = self.torch.cuda.ExternalStream(stream)
        if self.caller_stream is not None:
            ext.wait_stream(self.caller_stream)                # once per call: later callbacks follow on the same stream
            self.caller_stream = None
        return self.torch.cuda.stream(ext)

    def _run(self, body, stream):
        try:
            with self._stream(stream):
                body()
            return 0
        except BaseException as e:          # noqa: BLE001 -- kept and re-raised after the library call returns
            if self.error is None:
                self.error = e
            return 1

    def _result(self, r, n, dtype, like, what):
        t = self.torch
        if not isinstance(r, t.Tensor) or r.dtype != dtype or tuple(r.shape) != (n,) or r.device != like.device:
            raise TypeError(f"{what} must return a {dtype} tensor of shape ({n},) on {like.device}, got "
                            f"{type(r).__name__ if not isinstance(r, t.Tensor) else (r.dtype, tuple(r.shape), r.device)}")
        return r

    def _func(self, fn):
        t = self.torch

        def cb(_user, x, keep, n, values, stream):
            def body():
                xs = self._view(x, (n, 3), "<f8", t.float64)
                ks = self._view(keep, (n,), "|u1", t.uint8) if keep else None
                out = self._view(values, (n,), "<f8", t.float64)
                out.copy_(self._result(fn(xs, ks), n, t.float64, out, "DeviceFunction"))
            return self._run(body, stream)
        return cb

    def _sample(self, fn):
        t = self.torch

        def cb(_user, x, n, keep, stream):
            def body():
                out = self._view(keep, (n,), "|u1", t.uint8)
                out.copy_(self._result(fn(self._view(x, (n, 3), "<f8", t.float64)), n, t.bool, out, "DeviceSamplePredicate"))
            return self._run(body, stream)
        return cb

    def _node(self, fn):
        t = self.torch

        def cb(_user, x, values, n, keep, stream):
            def body():
                out = self._view(keep, (n,), "|u1", t.uint8)
                r = fn(self._view(x, (n, 3), "<f8", t.float64), self._view(values, (n,), "<f8", t.float64))
                out.copy_(self._result(r, n, t.bool, out, "DeviceNodePredicate"))
            return self._run(body, stream)
        return cb


def _copy_reduced(h, n_grid_cells, keep=False):
    """the (nodes, cells, cell map) of a dg_reduced_band handle, which is destroyed unless keep is set"""
    try:
        n_nodes, n_cells = C.c_uint64(), C.c_uint64()
        capi.check(capi.lib.dg_reduced_band_sizes(h, C.byref(n_nodes), C.byref(n_cells)))
        f = (np.empty(n_nodes.value), np.empty((n_cells.value, 32), np.uint32), np.empty(n_grid_cells, np.uint32))
        capi.check(capi.lib.dg_reduced_band_copy(h, capi.ptr(f[0], capi.F64P), capi.ptr(f[1], capi.U32P), capi.ptr(f[2], capi.U32P)))
        return f
    finally:
        if not keep:
            capi.lib.dg_reduced_band_destroy(h)


def _copy_kept(handles, n_grid_cells):
    """the (nodes, cells, cell map) of each dg_reduced_band handle; the handles are kept for the grid's first _device_field, or all
    destroyed when a copy fails"""
    try:
        return [_copy_reduced(h, n_grid_cells, keep=True) for h in handles]
    except BaseException:
        for h in handles:
            capi.lib.dg_reduced_band_destroy(h)
        raise


_INTERPOLATE = None


def _interpolate_function():
    """the autograd Function of interpolate on CUDA tensors: phi(x) with d phi / d x = K2's gradient, first order only.  Made at first use:
    torch is only imported by callers that pass tensors."""
    global _INTERPOLATE
    if _INTERPOLATE is None:
        import torch
        from torch.autograd.function import once_differentiable

        class Interpolate(torch.autograd.Function):
            @staticmethod
            def forward(ctx, x, run):
                phi, grad = run(x, True)
                ctx.mark_non_differentiable(grad)
                ctx.save_for_backward(grad)
                return phi, grad

            @staticmethod
            @once_differentiable
            def backward(ctx, grad_phi, _grad_grad):
                (grad,) = ctx.saved_tensors
                return grad_phi[:, None] * grad, None
        _INTERPOLATE = Interpolate
    return _INTERPOLATE


_INTERPOLATE_HESSIAN = None


def _interpolate_hessian_function():
    """the autograd Function of interpolate(..., hessian=True) on CUDA tensors: one kernel launch gives phi, grad and hess.  phi is
    differentiable to second order and grad to first order: phi's backward multiplies by the grad *output* (saved as an output, so a
    create_graph backward reaches grad's own backward), and grad's backward is einsum('na,nab->nb', v, hess).  hess has no derivative:
    a gradient that reaches it -- from a loss on hess, or from differentiating grad's backward, i.e. a third derivative of phi -- raises
    RuntimeError rather than being taken as zero."""
    global _INTERPOLATE_HESSIAN
    if _INTERPOLATE_HESSIAN is None:
        import torch

        class InterpolateHessian(torch.autograd.Function):
            @staticmethod
            def forward(ctx, x, run):
                phi, grad, hess = run(x)
                ctx.set_materialize_grads(False)
                ctx.save_for_backward(grad, hess)
                return phi, grad, hess

            @staticmethod
            def backward(ctx, grad_phi, grad_grad, grad_hess):
                if grad_hess is not None:
                    raise RuntimeError("interpolate: the Hessian has no derivative (third derivatives of the interpolant are not provided)")
                grad, hess = ctx.saved_tensors
                dx = None
                if grad_phi is not None:
                    dx = grad_phi[:, None] * grad
                if grad_grad is not None:
                    v = torch.einsum("na,nab->nb", grad_grad, hess)
                    dx = v if dx is None else dx + v
                return dx, None
        _INTERPOLATE_HESSIAN = InterpolateHessian
    return _INTERPOLATE_HESSIAN


class _TrainableField:
    """A trainable device field (dg_field_create_trainable) and the token of the interpolate(coefficients=) call whose values it holds.
    The grid keeps one per field id until its device copies are dropped; the autograd graph of every call made on it keeps it too, so a
    backward runs on the field its forward used (same topology, still allocated) even after setNodes, addFunction, reduceField or load
    dropped it from the grid, or after the grid itself was collected.  The handle is destroyed with the last reference."""

    def __init__(self, handle):
        self.handle, self.holds = handle, None
        info = (C.c_uint64 * 4)()
        capi.check(capi.lib.dg_field_info(handle, info))
        self.n_nodes, self.device = int(info[0]), int(info[3])

    def __del__(self):
        try:
            capi.lib.dg_field_destroy(self.handle)
        except Exception:
            pass


_INTERPOLATE_TRAINABLE = None


def _interpolate_trainable_function():
    """the autograd Function of interpolate(field_id, x, gradient, coefficients=c): phi and grad differentiable in c through K11's VJP, phi in
    x through K2's gradient and, when the forward ran K2's Hessian mode, grad in x through einsum('na,nab->nb', v, hess).  First order
    only: a double backward raises."""
    global _INTERPOLATE_TRAINABLE
    if _INTERPOLATE_TRAINABLE is None:
        import torch
        from torch.autograd.function import once_differentiable

        class InterpolateTrainable(torch.autograd.Function):
            @staticmethod
            def forward(ctx, x, c, run, vjp):
                phi, grad, hess = run(x, c)
                ctx.set_materialize_grads(False)
                ctx.vjp = vjp
                ctx.save_for_backward(x, c, grad, hess)
                return phi, grad

            @staticmethod
            @once_differentiable
            def backward(ctx, grad_phi, grad_grad):
                x, c, grad, hess = ctx.saved_tensors
                dx = dc = None
                if ctx.needs_input_grad[0]:
                    if grad_phi is not None:
                        dx = grad_phi[:, None] * grad
                    if grad_grad is not None:
                        if hess is None:
                            raise RuntimeError("interpolate: grad is differentiable in x only when x requires grad at the forward")
                        v = torch.einsum("na,nab->nb", grad_grad, hess)
                        dx = v if dx is None else dx + v
                    if dx is None:
                        dx = torch.zeros_like(x)
                if ctx.needs_input_grad[1]:
                    dc = ctx.vjp(x, c, grad_phi, grad_grad)
                return dx, dc, None, None
        _INTERPOLATE_TRAINABLE = InterpolateTrainable
    return _INTERPOLATE_TRAINABLE


_FIELD_RAYCAST = None


def _field_raycast_function():
    """the autograd Function of the level-set ray cast on CUDA tensors (K12): t_lo and t_hi differentiable in the origins, the directions
    and, with coefficients=c, in c, through the implicit function theorem at the crossing.  First order only: a double backward raises."""
    global _FIELD_RAYCAST
    if _FIELD_RAYCAST is None:
        import torch
        from torch.autograd.function import once_differentiable

        class FieldRaycast(torch.autograd.Function):
            @staticmethod
            def forward(ctx, o, d, c, run, vjp):
                t_lo, t_hi, status = run(o, d, c)
                ctx.mark_non_differentiable(status)
                ctx.set_materialize_grads(False)
                ctx.vjp = vjp
                ctx.save_for_backward(o, d, c, t_lo, status)
                return t_lo, t_hi, status

            @staticmethod
            @once_differentiable
            def backward(ctx, grad_t_lo, grad_t_hi, _grad_status):
                o, d, c, t_lo, status = ctx.saved_tensors
                if grad_t_lo is None and grad_t_hi is None:
                    return None, None, None, None, None
                go, gd, gc = ctx.vjp(o, d, c, t_lo, status, grad_t_lo, grad_t_hi, ctx.needs_input_grad[:3])
                return go, gd, gc, None, None
        _FIELD_RAYCAST = FieldRaycast
    return _FIELD_RAYCAST


def _raycast_vjp(h, o, d, t_lo, status, g_lo, g_hi, want_o, want_d, n_nodes):
    """dg_field_raycast_vjp_device on torch's current stream: (grad_origins, grad_directions, grad_nodes), each None unless wanted"""
    import torch
    n = len(o)
    go = torch.empty((n, 3), dtype=torch.float64, device=o.device) if want_o else None
    gd = torch.empty((n, 3), dtype=torch.float64, device=o.device) if want_d else None
    gn = torch.empty(n_nodes, dtype=torch.float64, device=o.device) if n_nodes is not None else None
    glo = None if g_lo is None else g_lo.to(torch.float64).contiguous()
    ghi = None if g_hi is None else g_hi.to(torch.float64).contiguous()
    ptr = lambda a: None if a is None else a.data_ptr()
    capi.check(capi.lib.dg_field_raycast_vjp_device(h, n, o.data_ptr(), d.data_ptr(), t_lo.data_ptr(), status.data_ptr(), ptr(glo), ptr(ghi),
                                                    ptr(go), ptr(gd), ptr(gn), _device.stream(o)))
    return go, gd, gn


_ISOSURFACE = None


def _isosurface_function():
    """the autograd Function of isosurface(..., coefficients=c) (K13): the vertices differentiable in c, each moving along its lattice edge as
    its crossing parameter t = (iso - f_p) / (f_q - f_p) follows the edge's two lattice values.  The triangles and the edge ids carry no
    gradient.  First order only: a double backward raises."""
    global _ISOSURFACE
    if _ISOSURFACE is None:
        import torch
        from torch.autograd.function import once_differentiable

        class Isosurface(torch.autograd.Function):
            @staticmethod
            def forward(ctx, c, run, vjp):
                V, T, E = run(c)
                ctx.mark_non_differentiable(T, E)
                ctx.set_materialize_grads(False)
                ctx.vjp = vjp
                ctx.save_for_backward(c, E)
                return V, T, E

            @staticmethod
            @once_differentiable
            def backward(ctx, grad_V, _grad_T, _grad_E):
                if grad_V is None:
                    return None, None, None
                c, E = ctx.saved_tensors
                return ctx.vjp(c, E, grad_V), None, None
        _ISOSURFACE = Isosurface
    return _ISOSURFACE


def grid_desc(domain_min, domain_max, resolution, cell_size=None, inv_cell_size=None):
    """dg_grid_desc; cell sizes computed like the DiscreteGrid ctor (discrete_grid.hpp:22-29) unless given verbatim."""
    d = capi.GridDesc()
    mn = np.ascontiguousarray(domain_min, np.float64); mx = np.ascontiguousarray(domain_max, np.float64)
    res = np.ascontiguousarray(resolution, np.uint32)
    capi.check(capi.lib.dg_grid_init(capi.ptr(mn, capi.F64P), capi.ptr(mx, capi.F64P), capi.ptr(res, capi.U32P), C.byref(d)))
    if cell_size is not None:
        for k in range(3):
            d.cell_size[k] = float(cell_size[k]); d.inv_cell_size[k] = float(inv_cell_size[k])
    return d


def generate_sdf_domain(vertices):
    """GenerateSDF's padded bounding box (cmd/generate_sdf/main.cpp:83-91)."""
    V = np.ascontiguousarray(vertices, np.float64).reshape(-1, 3)
    mn = np.empty(3); mx = np.empty(3)
    capi.check(capi.lib.dg_generate_sdf_domain(capi.ptr(V, capi.F64P), len(V), capi.ptr(mn, capi.F64P), capi.ptr(mx, capi.F64P)))
    return mn, mx


class CubicLagrangeDiscreteGrid:
    def __init__(self, domain_or_filename=None, domain_max=None, resolution=None):
        """CubicLagrangeDiscreteGrid(filename) | CubicLagrangeDiscreteGrid(domain_min, domain_max, resolution)
        (cubic_lagrange_discrete_grid.hpp:12-14)."""
        self.m_nodes, self.m_cells, self.m_cell_map = [], [], []
        self.m_n_fields = 0
        self._fields = {}          # field_id -> device handle (cache; invalidated by addFunction/load/reduceField)
        self._reduced = {}         # field_id -> the dg_reduced_band its reduced call returned, until its first _device_field (or invalidation)
        self._trainable = {}       # field_id -> _TrainableField (interpolate(coefficients=))
        self._desc = None
        if isinstance(domain_or_filename, str):
            self.load(domain_or_filename)
        elif domain_or_filename is not None:
            self._desc = grid_desc(domain_or_filename, domain_max, resolution)
            self._sync_members()

    # ------------------------------------------------------------------ members / accessors (discrete_grid.hpp:85-98)
    def _sync_members(self):
        d = self._desc
        self.m_domain = (np.array(d.domain_min[:]), np.array(d.domain_max[:]))
        self.m_resolution = np.array(d.resolution[:], np.uint32)
        self.m_cell_size = np.array(d.cell_size[:])
        self.m_inv_cell_size = np.array(d.inv_cell_size[:])
        self.m_n_cells = int(np.prod(self.m_resolution.astype(np.uint64)))

    def domain(self):
        return self.m_domain

    def resolution(self):
        return self.m_resolution

    def cellSize(self):
        return self.m_cell_size

    def invCellSize(self):
        return self.m_inv_cell_size

    def nCells(self):
        return self.m_n_cells

    def nFields(self):
        return self.m_n_fields

    def nNodes(self):
        n = C.c_uint64()
        capi.check(capi.lib.dg_grid_num_nodes(self._desc.resolution, C.byref(n)))
        return n.value

    # discrete_grid.cpp:8-38
    def singleToMultiIndex(self, l):
        n0, n1 = int(self.m_resolution[0]), int(self.m_resolution[1])
        n01 = n0 * n1
        k, t = divmod(int(l), n01)
        j, i = divmod(t, n0)
        return (i, j, k)

    def multiToSingleIndex(self, ijk):
        n0, n1 = int(self.m_resolution[0]), int(self.m_resolution[1])
        return n1 * n0 * int(ijk[2]) + n0 * int(ijk[1]) + int(ijk[0])

    def subdomain(self, l_or_ijk):
        ijk = self.singleToMultiIndex(l_or_ijk) if np.isscalar(l_or_ijk) else l_or_ijk
        origin = self.m_domain[0] + np.array(ijk, np.float64) * self.m_cell_size
        return origin, origin + self.m_cell_size

    def nodePositions(self, l_begin=0, l_end=None):
        """indexToNodePosition for a node range (cubic_lagrange_discrete_grid.cpp:604-665), computed on the GPU."""
        l_end = self.nNodes() if l_end is None else l_end
        x = np.empty((l_end - l_begin, 3))
        capi.check(capi.lib.dg_node_positions(C.byref(self._desc), l_begin, l_end, capi.ptr(x, capi.F64P)))
        return x

    # ------------------------------------------------------------------ addFunction (cubic_lagrange_discrete_grid.cpp:780-899)
    def addFunction(self, func, verbose=False, pred=None):
        if isinstance(func, DeviceFunction) or isinstance(pred, DeviceSamplePredicate):
            if not isinstance(func, DeviceFunction) or (pred is not None and not isinstance(pred, DeviceSamplePredicate)):
                raise TypeError("a DeviceFunction takes a DeviceSamplePredicate (or none), and a DeviceSamplePredicate only goes with a DeviceFunction")
            # the whole addFunction in one call: your function on the GPU, connectivity + cell map written by the library's host threads meanwhile
            coeffs = np.empty(self.nNodes())
            cells = np.empty((self.m_n_cells, 32), np.uint32)
            cmap = np.empty(self.m_n_cells, np.uint32)
            self.last_add_function_ms = np.zeros(6)
            cb = _DeviceCallbacks(func=func, sample=pred)
            cb.check(capi.lib.dg_add_function_device(C.byref(self._desc), cb.func, None, cb.sample, None, 0, capi.ptr(coeffs, capi.F64P),
                                                     capi.ptr(cells, capi.U32P), capi.ptr(cmap, capi.U32P), capi.ptr(self.last_add_function_ms, capi.F64P)))
            if verbose:
                print(f"Construction: {len(coeffs)} nodes sampled on the GPU in {self.last_add_function_ms[0]:.1f} ms")
            self._invalidate()
            self.m_nodes.append(coeffs); self.m_cells.append(cells); self.m_cell_map.append(cmap)
            self.m_n_fields += 1
            return self.m_n_fields - 1
        if isinstance(func, MeshSignedDistance):
            if pred is not None and not isinstance(pred, MeshDistanceBand):
                raise TypeError("a sample predicate is only supported with DensityMapFunction, or as MeshDistanceBand with MeshSignedDistance")
            if pred is not None and pred.md is not func.md:
                raise TypeError("MeshDistanceBand must use the same TriangleMeshDistance as the MeshSignedDistance it restricts")
            # the whole addFunction in one call: node loop on the GPU, connectivity + cell map written by the library's host threads meanwhile
            coeffs = np.empty(self.nNodes())
            cells = np.empty((self.m_n_cells, 32), np.uint32)
            cmap = np.empty(self.m_n_cells, np.uint32)
            self.last_add_function_ms = np.zeros(6)
            out = (capi.ptr(coeffs, capi.F64P), capi.ptr(cells, capi.U32P), capi.ptr(cmap, capi.U32P), capi.ptr(self.last_add_function_ms, capi.F64P))
            if pred is None:
                capi.check(capi.lib.dg_add_function_sdf(func.md.handle, C.byref(self._desc), func.sign, *out))
            else:
                capi.check(capi.lib.dg_add_function_sdf_band(func.md.handle, C.byref(self._desc), func.sign, pred.band, *out))
            self.m_nodes.append(coeffs); self.m_cells.append(cells); self.m_cell_map.append(cmap)
            self.m_n_fields += 1
            return self.m_n_fields - 1
        elif isinstance(func, DensityMapFunction):
            coeffs = np.empty(self.nNodes())
            capi.check(capi.lib.dg_density_map(self._device_field(func.field_id), func.h, func.rho0, int(func.no_reduction), 0,
                                               len(coeffs), capi.ptr(coeffs, capi.F64P)))
        elif isinstance(func, VolumeMapFunction):
            coeffs = np.empty(self.nNodes())
            capi.check(capi.lib.dg_volume_map(self._device_field(func.field_id), func.h, func.scale, int(func.no_reduction), 0,
                                              len(coeffs), capi.ptr(coeffs, capi.F64P)))
        else:
            raise TypeError("addFunction runs on the GPU and only accepts MeshSignedDistance, DensityMapFunction, VolumeMapFunction or DeviceFunction; "
                            "wrap a function of your own that runs on the GPU (e.g. torch operations) in DeviceFunction")
        return self.addSampledFunction(coeffs)

    def addReducedBandField(self, func, pred, verbose=False):
        """addFunction(func, verbose, pred) followed by reduceField(id, always true), in one GPU call (dg_reduced_band_create): the field
        holds exactly what those two calls leave, but only the survivors and the cell map ever reach the host.  func: MeshSignedDistance,
        pred: MeshDistanceBand over the same TriangleMeshDistance.  Returns the field id.
        The library's handle on the device copy of the result is kept: the field's first interpolate (or any other device use) builds its
        interpolation field from it on the device and then releases it, with no host round trip.  Until then, or until the grid's device
        fields are invalidated (addFunction, reduceField, load, ...), the handle's arrays stay held in GPU memory -- for the 512^3 bunny band
        (49.4 M nodes, 6.28 M cells) 0.40 GB of nodes, 0.80 GB of rows and 0.54 GB of cell map.  The same holds for addReducedFunction,
        addReducedDensityMap (both fields) and reduceField with a DeviceNodePredicate."""
        if not isinstance(func, MeshSignedDistance) or not isinstance(pred, MeshDistanceBand):
            raise TypeError("addReducedBandField takes a MeshSignedDistance and a MeshDistanceBand")
        if pred.md is not func.md:
            raise TypeError("MeshDistanceBand must use the same TriangleMeshDistance as the MeshSignedDistance it restricts")
        h = C.c_void_p()
        self.last_reduced_band_ms = np.zeros(7)
        capi.check(capi.lib.dg_reduced_band_create(func.md.handle, C.byref(self._desc), func.sign, pred.band, 0, C.byref(h),
                                                   capi.ptr(self.last_reduced_band_ms, capi.F64P)))
        coeffs, cells, cmap = _copy_kept([h], self.m_n_cells)[0]
        if verbose:
            print(f"Construction: {len(coeffs)} of {self.nNodes()} nodes kept in {self.last_reduced_band_ms[6]:.1f} ms on the GPU")
        self.m_nodes.append(coeffs); self.m_cells.append(cells); self.m_cell_map.append(cmap)
        self.m_n_fields += 1
        self._keep_reduced(self.m_n_fields - 1, h)
        return self.m_n_fields - 1

    def addReducedFunction(self, func, sample_pred=None, reduce_pred=None, verbose=False):
        """addFunction(func, verbose, sample_pred) followed by reduceField(id, reduce_pred), in one call (dg_reduced_function_create): the
        field holds exactly what those two calls leave, but the dense values stay on the GPU; only the survivors and the cell map reach the
        host.  func: DeviceFunction; sample_pred: DeviceSamplePredicate or None; reduce_pred: DeviceNodePredicate or None (always true).
        Returns the field id.  The result's device copy is kept for the field's first interpolate, as in addReducedBandField."""
        if not isinstance(func, DeviceFunction) or not isinstance(sample_pred, (DeviceSamplePredicate, type(None))) \
                or not isinstance(reduce_pred, (DeviceNodePredicate, type(None))):
            raise TypeError("addReducedFunction takes a DeviceFunction, a DeviceSamplePredicate or None and a DeviceNodePredicate or None")
        h = C.c_void_p()
        self.last_reduced_function_ms = np.zeros(8)
        cb = _DeviceCallbacks(func=func, sample=sample_pred, node=reduce_pred)
        cb.check(capi.lib.dg_reduced_function_create(C.byref(self._desc), cb.func, None, cb.sample, None, cb.node, None, 0, 0, C.byref(h),
                                                     capi.ptr(self.last_reduced_function_ms, capi.F64P)))
        coeffs, cells, cmap = _copy_kept([h], self.m_n_cells)[0]
        if verbose:
            print(f"Construction: {len(coeffs)} of {self.nNodes()} nodes kept in {self.last_reduced_function_ms[6]:.1f} ms")
        self._invalidate()
        self.m_nodes.append(coeffs); self.m_cells.append(cells); self.m_cell_map.append(cmap)
        self.m_n_fields += 1
        self._keep_reduced(self.m_n_fields - 1, h)
        return self.m_n_fields - 1

    def addReducedDensityMap(self, func):
        """GenerateDensityMap with reduction in one GPU call (dg_reduced_density_map_create): leaves exactly what
        addFunction(func) followed by reduceField(func.field_id, p0) and reduceField(new_id, p1) leave, with the tool's predicates
        p0(x, v) = -6h < v + cell_diag & v - cell_diag < 2h and p1(x, v) = 0 <= v <= 3 rho0 (main.cpp:139-140).  The SDF field is replaced by
        its reduction and the reduced density field is appended; the dense density field never reaches the host.  Returns the new field id.
        The device copies of both results are kept for the fields' first interpolate, as in addReducedBandField."""
        if not isinstance(func, DensityMapFunction):
            raise TypeError("addReducedDensityMap takes a DensityMapFunction")
        if func.no_reduction:
            raise TypeError("addReducedDensityMap: the DensityMapFunction has no_reduction set (use addFunction)")
        self.last_reduced_density_ms = np.zeros(13)
        return self._add_reduced_node_map("addReducedDensityMap", capi.lib.dg_reduced_density_map_create, func.field_id, func.h, func.rho0,
                                          self.last_reduced_density_ms)

    def addReducedVolumeMap(self, func):
        """The volume map with reduction in one GPU call (dg_reduced_volume_map_create): leaves exactly what addFunction(func) followed by
        reduceField(func.field_id, p0) and reduceField(new_id, p1) leave, with GenerateDensityMap's p0 (as in addReducedDensityMap) and
        p1(x, v) = 0 <= v.  The SDF field is replaced by its reduction and the reduced volume field is appended; the dense volume field never
        reaches the host.  Returns the new field id.  The device copies of both results are kept for the fields' first interpolate."""
        if not isinstance(func, VolumeMapFunction):
            raise TypeError("addReducedVolumeMap takes a VolumeMapFunction")
        if func.no_reduction:
            raise TypeError("addReducedVolumeMap: the VolumeMapFunction has no_reduction set (use addFunction)")
        self.last_reduced_volume_ms = np.zeros(13)
        return self._add_reduced_node_map("addReducedVolumeMap", capi.lib.dg_reduced_volume_map_create, func.field_id, func.h, func.scale,
                                          self.last_reduced_volume_ms)

    def _add_reduced_node_map(self, who, entry, fid, h, param, timings):
        """the shared body of addReducedDensityMap / addReducedVolumeMap: `entry` is the library's one-call route"""
        nodes = np.ascontiguousarray(self.m_nodes[fid], np.float64)
        cells = np.ascontiguousarray(self.m_cells[fid], np.uint32)
        cmap = np.ascontiguousarray(self.m_cell_map[fid], np.uint32)
        if len(cmap) != self.m_n_cells:
            raise ValueError(f"{who}: the SDF field's cell map must cover every grid cell")
        r = (C.c_void_p(), C.c_void_p())
        capi.check(entry(C.byref(self._desc), capi.ptr(nodes, capi.F64P), len(nodes), capi.ptr(cells, capi.U32P), len(cells),
                         capi.ptr(cmap, capi.U32P), h, param, 0, C.byref(r[0]), C.byref(r[1]), capi.ptr(timings, capi.F64P)))
        out = _copy_kept(r, self.m_n_cells)
        self._invalidate()
        self.m_nodes[fid], self.m_cells[fid], self.m_cell_map[fid] = out[0]
        self.m_nodes.append(out[1][0]); self.m_cells.append(out[1][1]); self.m_cell_map.append(out[1][2])
        self.m_n_fields += 1
        self._keep_reduced(fid, r[0])
        self._keep_reduced(self.m_n_fields - 1, r[1])
        return self.m_n_fields - 1

    def addSampledFunction(self, coeffs):
        """Appends a field from node values (what addFunction's loop :806-831 produces), then builds the cell
        table (:833-886, on the GPU) and the identity cell map (:888-891).  Returns the field id (:898)."""
        coeffs = np.ascontiguousarray(coeffs, np.float64)
        if coeffs.shape != (self.nNodes(),):
            raise ValueError(f"expected {self.nNodes()} node values")
        cells = np.empty((self.m_n_cells, 32), np.uint32)
        capi.check(capi.lib.dg_build_cells(self._desc.resolution, 0, self.m_n_cells, capi.ptr(cells, capi.U32P)))
        self.m_nodes.append(coeffs)
        self.m_cells.append(cells)
        self.m_cell_map.append(np.arange(self.m_n_cells, dtype=np.uint32))
        self.m_n_fields += 1
        return self.m_n_fields - 1

    # ------------------------------------------------------------------ reduceField (cubic_lagrange_discrete_grid.cpp:1065-1174)
    def reduceField(self, field_id, pred):
        """Sparsifies a field.  pred(x[n,3], values[n]) -> bool[n] is the reference's Predicate, vectorised; nodes, cells and the
        cell map end up exactly as the reference leaves them (dg_reduce_field).  A DeviceNodePredicate runs on the GPU instead, on
        positions made there, and so does the whole reduction (dg_reduce_field_device); its device copy of the result is kept for the
        field's first interpolate, as in addReducedBandField."""
        if isinstance(pred, DeviceNodePredicate):
            nodes = np.ascontiguousarray(self.m_nodes[field_id], np.float64)
            cells = np.ascontiguousarray(self.m_cells[field_id], np.uint32)
            h = C.c_void_p()
            cb = _DeviceCallbacks(node=pred)
            cb.check(capi.lib.dg_reduce_field_device(C.byref(self._desc), capi.ptr(nodes, capi.F64P), len(nodes), capi.ptr(cells, capi.U32P),
                                                     len(cells), cb.node, None, 0, 0, C.byref(h), None))
            out = _copy_kept([h], self.m_n_cells)[0]
            self._invalidate()
            self.m_nodes[field_id], self.m_cells[field_id], self.m_cell_map[field_id] = out
            self._keep_reduced(field_id, h)
            return
        nodes = np.ascontiguousarray(self.m_nodes[field_id], np.float64).copy()
        keep = np.asarray(pred(self.nodePositions(0, len(nodes)), nodes), bool) & (nodes != np.finfo(np.float64).max)   # :1073
        keep = np.ascontiguousarray(keep, np.uint8)
        cells = np.ascontiguousarray(self.m_cells[field_id], np.uint32).copy()
        cmap = np.empty(self.m_n_cells, np.uint32)
        n_nodes, n_cells = C.c_uint64(), C.c_uint64()
        capi.check(capi.lib.dg_reduce_field(C.byref(self._desc), capi.ptr(nodes, capi.F64P), len(nodes), keep.ctypes.data_as(C.POINTER(C.c_uint8)),
                                            capi.ptr(cells, capi.U32P), len(cells), capi.ptr(cmap, capi.U32P), 0, C.byref(n_nodes), C.byref(n_cells), None))
        self._invalidate()
        self.m_nodes[field_id], self.m_cells[field_id], self.m_cell_map[field_id] = nodes[:n_nodes.value].copy(), cells[:n_cells.value].copy(), cmap

    # ------------------------------------------------------------------ device field cache
    def _device_field(self, field_id):
        """the device field of field_id, made at first use: from the reduced handle the field's reduced call kept (dg_field_create_reduced,
        device to device; the handle is released) or else by uploading the host members (dg_field_create).  Creating it synchronises the
        device."""
        if field_id not in self._fields:
            h = C.c_void_p()
            r = self._reduced.get(field_id)
            if r is not None:
                capi.check(capi.lib.dg_field_create_reduced(r, C.byref(h)))
                capi.lib.dg_reduced_band_destroy(self._reduced.pop(field_id))
            else:
                nodes, cells, cmap = self.m_nodes[field_id], self.m_cells[field_id], self.m_cell_map[field_id]
                capi.check(capi.lib.dg_field_create(C.byref(self._desc), capi.ptr(nodes, capi.F64P), len(nodes),
                                                    capi.ptr(cells, capi.U32P), len(cells), capi.ptr(cmap, capi.U32P), C.byref(h)))
            self._fields[field_id] = h
        return self._fields[field_id]

    def _keep_reduced(self, field_id, h):
        """keeps the handle a reduced call returned for field_id, so that the field's first _device_field needs no upload"""
        old = self._reduced.pop(field_id, None)
        if old is not None:
            capi.lib.dg_reduced_band_destroy(old)
        self._reduced[field_id] = h

    def _invalidate(self):
        for h in self._fields.values():
            capi.lib.dg_field_destroy(h)
        for h in self._reduced.values():
            capi.lib.dg_reduced_band_destroy(h)
        self._fields, self._reduced, self._trainable = {}, {}, {}

    def _trainable_field(self, field_id):
        """the trainable device field of field_id (dg_field_create_trainable of the host members), made at first use; it synchronises"""
        if field_id not in self._trainable:
            h = C.c_void_p()
            nodes, cells, cmap = self.m_nodes[field_id], self.m_cells[field_id], self.m_cell_map[field_id]
            nodes = np.ascontiguousarray(nodes, np.float64)
            cells = np.ascontiguousarray(cells, np.uint32)
            cmap = np.ascontiguousarray(cmap, np.uint32)
            capi.check(capi.lib.dg_field_create_trainable(C.byref(self._desc), capi.ptr(nodes, capi.F64P), len(nodes), capi.ptr(cells, capi.U32P),
                                                          len(cells), capi.ptr(cmap, capi.U32P), C.byref(h)))
            self._trainable[field_id] = _TrainableField(h)
        return self._trainable[field_id]

    def setNodes(self, field_id, values):
        """Replaces the node values of field field_id (beyond the reference): values, a numpy array or a tensor of len(m_nodes[field_id])
        values, is copied to m_nodes[field_id], and the field's device copies are dropped, so that save() and every other method see it.
        The way to keep a field trained through interpolate(..., coefficients=c): grid.setNodes(field_id, c.detach())."""
        if hasattr(values, "detach"):
            values = values.detach().cpu().numpy()
        values = np.array(values, np.float64, copy=True).reshape(-1)
        if len(values) != len(self.m_nodes[field_id]):
            raise ValueError(f"setNodes: field {field_id} has {len(self.m_nodes[field_id])} nodes (got {len(values)})")
        h = self._fields.pop(field_id, None)
        if h is not None:
            capi.lib.dg_field_destroy(h)
        r = self._reduced.pop(field_id, None)
        if r is not None:
            capi.lib.dg_reduced_band_destroy(r)
        self._trainable.pop(field_id, None)          # destroyed with the last graph that still uses it
        self.m_nodes[field_id] = values

    def __del__(self):
        try:
            self._invalidate()
        except Exception:
            pass

    # ------------------------------------------------------------------ interpolate (cubic_lagrange_discrete_grid.cpp:977-1063)
    def interpolate(self, field_id_or_x, x=None, gradient=False, hessian=False, coefficients=None):
        """interpolate(x) == interpolate(0, x) (discrete_grid.hpp:38-41).  x: (n, 3).  Returns phi[n], or
        (phi[n], grad[n,3]) when gradient=True.  Out-of-domain / removed cell / missing coefficient -> DBL_MAX, grad 0.
        A numpy array (or a CPU tensor) goes through the host pipeline and gives numpy arrays.  A float64 torch tensor (n, 3) or (3,) on
        the field's CUDA device stays there: the query runs on torch's current stream, asynchronously, and phi / grad are CUDA tensors with
        the bits of the host route.  When x requires grad (and grad mode is on), phi is differentiable in x, first order only:
        d phi / d x is K2's gradient, the reference's derivative of the interpolant (0 at DBL_MAX).  The returned grad is not differentiable.

        hessian=True (beyond the reference) returns (phi[n], grad[n,3], hess[n,3,3]) from one pass of K2's Hessian mode: phi and grad have
        the bits of gradient=True, hess is the exactly symmetric second derivative of the interpolant in x (+0.0 where phi is DBL_MAX).
        The interpolant is only C0 across cell faces, so on a face hess is that of the cell the point is assigned to.  On CUDA tensors
        that require grad, phi is differentiable to second order and grad to first order (its vector-Jacobian product is
        einsum('na,nab->nb', v, hess)), so torch.autograd.grad(..., create_graph=True) works on phi; hess has no derivative, and a
        gradient that reaches it (a third derivative of phi) raises RuntimeError.

        coefficients=c (beyond the reference) interpolates the field with the node values c instead of its own: c is a float64 CUDA tensor
        of len(m_nodes[field_id]) values on the field's device, and x must be a CUDA tensor.  The grid keeps one trainable device field
        per field id (dg_field_create_trainable, made at first use from the field's cells and cell map); each call writes c into it and runs
        K2 on torch's current stream, so phi and grad have the bits interpolate() gives on a field whose m_nodes are c.  phi and grad are
        differentiable in c (dg_interpolate_vjp_device: the transpose of K2's map, summed in a fixed order, see csrc/k11_field_grad.cu) and
        phi in x; with gradient=True and x requiring grad the forward runs K2's Hessian mode, so that grad is differentiable in x too.
        First order only (a double backward raises); hessian=True is refused.  setNodes(field_id, c.detach()) keeps the result."""
        if x is None:
            field_id, x = 0, field_id_or_x
        else:
            field_id = field_id_or_x
        if coefficients is not None:
            if hessian:
                raise ValueError("interpolate: hessian=True is not differentiable in the coefficients; drop one of the two")
            if not _device.is_device_query(x):
                raise TypeError("interpolate: coefficients= needs x as a float64 CUDA tensor")
            return self._interpolate_trainable(field_id, x, gradient, coefficients)
        if _device.is_device_query(x):
            if hessian:
                return self._interpolate_hessian_device(field_id, x)
            return self._interpolate_device(field_id, x, gradient)
        x = np.ascontiguousarray(x, np.float64).reshape(-1, 3)
        phi = np.empty(len(x))
        if hessian:
            grad, hess = np.empty((len(x), 3)), np.empty((len(x), 3, 3))
            capi.check(capi.lib.dg_interpolate_hessian_batch(self._device_field(field_id), capi.ptr(x, capi.F64P), len(x), capi.ptr(phi, capi.F64P),
                                                             capi.ptr(grad, capi.F64P), capi.ptr(hess, capi.F64P)))
            return phi, grad, hess
        grad = np.empty((len(x), 3)) if gradient else None
        capi.check(capi.lib.dg_interpolate_batch(self._device_field(field_id), capi.ptr(x, capi.F64P), len(x),
                                                 capi.ptr(phi, capi.F64P), capi.ptr(grad, capi.F64P)))
        return (phi, grad) if gradient else phi

    def _interpolate_device(self, field_id, x, gradient):
        """the CUDA-tensor route: dg_interpolate_batch_device on torch's current stream"""
        import torch
        h = self._device_field(field_id)
        info = (C.c_uint64 * 4)()
        capi.check(capi.lib.dg_field_info(h, info))
        x = _device.points(x, int(info[3]), "interpolate")

        def run(xc, with_grad):
            phi = torch.empty(len(xc), dtype=torch.float64, device=xc.device)
            grad = torch.empty((len(xc), 3), dtype=torch.float64, device=xc.device) if with_grad else None
            capi.check(capi.lib.dg_interpolate_batch_device(h, xc.data_ptr(), len(xc), phi.data_ptr(), None if grad is None else grad.data_ptr(),
                                                            _device.stream(xc)))
            return phi, grad
        if x.requires_grad and torch.is_grad_enabled():
            phi, grad = _interpolate_function().apply(x, run)
        else:
            phi, grad = run(x, gradient)
        return (phi, grad) if gradient else phi

    def _interpolate_trainable(self, field_id, x, gradient, c):
        """interpolate(..., coefficients=c): dg_field_set_nodes_device, then K2, on torch's current stream"""
        import torch
        tf = self._trainable_field(field_id)        # the closures below keep it (not the grid) alive for the backward
        h, n_nodes = tf.handle, tf.n_nodes
        x = _device.points(x, tf.device, "interpolate")
        if not isinstance(c, torch.Tensor) or c.dtype != torch.float64:
            raise TypeError(f"interpolate: coefficients must be a float64 tensor (got {type(c).__name__ if not isinstance(c, torch.Tensor) else c.dtype})")
        if tuple(c.shape) != (n_nodes,):
            raise ValueError(f"interpolate: coefficients must have shape ({n_nodes},), got {tuple(c.shape)}")
        if not capi.EMULATED and (not c.is_cuda or c.device.index != tf.device):
            raise ValueError(f"interpolate: coefficients are on {c.device} but the field lives on cuda:{tf.device}")
        c = c.contiguous()

        token = object()                   # this call's pack: the backward repacks c unless the field still holds it

        def hold(cc, again):
            if again and tf.holds is token:
                return
            capi.check(capi.lib.dg_field_set_nodes_device(h, cc.data_ptr(), n_nodes, _device.stream(cc)))
            tf.holds = token

        x_grad = x.requires_grad and torch.is_grad_enabled()
        with_hess = gradient and x_grad

        def run(xc, cc):
            hold(cc, False)
            n = len(xc)
            phi = torch.empty(n, dtype=torch.float64, device=xc.device)
            grad = torch.empty((n, 3), dtype=torch.float64, device=xc.device) if (gradient or x_grad) else None
            hess = torch.empty((n, 3, 3), dtype=torch.float64, device=xc.device) if with_hess else None
            if with_hess:
                capi.check(capi.lib.dg_interpolate_hessian_batch_device(h, xc.data_ptr(), n, phi.data_ptr(), grad.data_ptr(), hess.data_ptr(),
                                                                        _device.stream(xc)))
            else:
                capi.check(capi.lib.dg_interpolate_batch_device(h, xc.data_ptr(), n, phi.data_ptr(), None if grad is None else grad.data_ptr(),
                                                                _device.stream(xc)))
            return phi, grad, hess

        def vjp(xc, cc, grad_phi, grad_grad):
            hold(cc, True)
            gp = None if grad_phi is None else grad_phi.contiguous()
            gg = None if grad_grad is None else grad_grad.contiguous()
            out = torch.empty(n_nodes, dtype=torch.float64, device=cc.device)
            if gp is None and gg is None:
                return out.zero_()
            capi.check(capi.lib.dg_interpolate_vjp_device(h, xc.data_ptr(), len(xc), None if gp is None else gp.data_ptr(),
                                                          None if gg is None else gg.data_ptr(), out.data_ptr(), _device.stream(xc)))
            return out
        if torch.is_grad_enabled() and (x.requires_grad or c.requires_grad):
            phi, grad = _interpolate_trainable_function().apply(x, c, run, vjp)
        else:
            phi, grad, _ = run(x, c)
        return (phi, grad) if gradient else phi

    def _interpolate_hessian_device(self, field_id, x):
        """the CUDA-tensor route of hessian=True: dg_interpolate_hessian_batch_device on torch's current stream"""
        import torch
        h = self._device_field(field_id)
        info = (C.c_uint64 * 4)()
        capi.check(capi.lib.dg_field_info(h, info))
        x = _device.points(x, int(info[3]), "interpolate")

        def run(xc):
            phi = torch.empty(len(xc), dtype=torch.float64, device=xc.device)
            grad = torch.empty((len(xc), 3), dtype=torch.float64, device=xc.device)
            hess = torch.empty((len(xc), 3, 3), dtype=torch.float64, device=xc.device)
            capi.check(capi.lib.dg_interpolate_hessian_batch_device(h, xc.data_ptr(), len(xc), phi.data_ptr(), grad.data_ptr(), hess.data_ptr(),
                                                                    _device.stream(xc)))
            return phi, grad, hess
        if x.requires_grad and torch.is_grad_enabled():
            return _interpolate_hessian_function().apply(x, run)
        return run(x)

    # ------------------------------------------------------------------ level sets (beyond the reference)
    def isosurface(self, field_id=0, iso=0.0, subdivisions=1, device=False, coefficients=None, edges=False):
        """The level set {phi = iso} of a field as a triangle mesh: marching tetrahedra on a lattice that subdivides every grid cell
        `subdivisions` times (1..16), on the field's GPU (dg_isosurface_create; the contract is in csrc/k6_isosurface.cu and DESIGN §3).
        The lattice values are the bits interpolate() returns there; points where it returns DBL_MAX or a non-finite value (outside the
        domain, removed cells of a reduced field) are invalid, and tetrahedra touching them emit nothing.  Triangles are oriented from the
        negative to the non-negative side (outward for an SDF); coincident vertices are not welded, so the mesh is closed by vertex ids.
        Returns (vertices float64 (n, 3), triangles uint32 (m, 3)) as numpy arrays -- the layout TriangleMeshDistance takes.  With
        device=True they are CUDA tensors on the field's device, filled on torch's current stream, with triangles as torch.int32 (same
        values; 2^31 vertices or more are refused on this route).  A reduced field's kept device handle is used without a host round trip.
        Stage times (values, classify, scans, emit, total; ms) are left in last_isosurface_ms.

        edges=True adds a third output: the lattice edge 7 * lin(p) + d of every vertex, ascending (uint64 numpy, or torch.int64 with
        device=True; the contract's numbering).

        coefficients=c (beyond the reference) extracts the level set of the field with the node values c instead of its own, on the trainable
        device field interpolate(coefficients=) uses (same rules: c a float64 CUDA tensor of len(m_nodes[field_id]) values); it needs
        device=True (ValueError otherwise), so that the result type never changes silently.  The vertices have the bits isosurface() gives on
        a field whose m_nodes are c, and are differentiable in c (K13, csrc/k13_isosurface_grad.cu): each vertex moves along its lattice edge
        as t = (iso - f_p) / (f_q - f_p) follows the edge's lattice values, summed into the nodes in a fixed order (K11).  A vertex at a
        DBL_MAX or non-finite value, or on an edge whose two values are equal, gets 0.  The triangles and the edge ids carry no gradient; not
        differentiable in iso; first order only (a double backward raises)."""
        if coefficients is not None:
            if not device:
                raise ValueError("isosurface: coefficients= needs device=True (the vertices are then CUDA tensors differentiable in c)")
            return self._isosurface_trainable(field_id, float(iso), int(subdivisions), coefficients, edges)
        V, T, E = self._isosurface(self._device_field(field_id), float(iso), int(subdivisions), device, edges)
        return (V, T, E) if edges else (V, T)

    def _isosurface(self, h, iso, subdivisions, device, edges):
        """dg_isosurface_create on the field handle h, then its outputs: (V, T, edge ids or None) as numpy arrays or, with device=True, as
        tensors on the field's device filled on torch's current stream"""
        s = C.c_void_p()
        self.last_isosurface_ms = np.zeros(5)
        capi.check(capi.lib.dg_isosurface_create(h, iso, subdivisions, C.byref(s), capi.ptr(self.last_isosurface_ms, capi.F64P)))
        try:
            nv, nt = C.c_uint64(), C.c_uint64()
            capi.check(capi.lib.dg_isosurface_sizes(s, C.byref(nv), C.byref(nt)))
            nv, nt = nv.value, nt.value
            if not device:
                V = np.empty((nv, 3)); T = np.empty((nt, 3), np.uint32)
                capi.check(capi.lib.dg_isosurface_copy(s, capi.ptr(V, capi.F64P), capi.ptr(T, capi.U32P)))
                E = None
                if edges:
                    E = np.empty(nv, np.uint64)
                    capi.check(capi.lib.dg_isosurface_copy_edges(s, capi.ptr(E, capi.U64P)))
                return V, T, E
            import torch
            if nv >= 2 ** 31:
                raise ValueError(f"isosurface: {nv} vertices do not fit the int32 indices of the device route; use device=False")
            info = (C.c_uint64 * 4)()
            capi.check(capi.lib.dg_field_info(h, info))
            dev = torch.device("cpu") if capi.EMULATED else torch.device("cuda", int(info[3]))
            V = torch.empty((nv, 3), dtype=torch.float64, device=dev)
            T = torch.empty((nt, 3), dtype=torch.int32, device=dev)
            st = _device.stream(V)
            capi.check(capi.lib.dg_isosurface_copy_device(s, V.data_ptr(), T.data_ptr(), st))
            E = None
            if edges:
                E = torch.empty(nv, dtype=torch.int64, device=dev)
                capi.check(capi.lib.dg_isosurface_copy_edges_device(s, E.data_ptr(), st))
            if not capi.EMULATED:
                torch.cuda.current_stream(dev).synchronize()          # the copies read the handle, released below
            return V, T, E
        finally:
            capi.lib.dg_isosurface_destroy(s)

    def _isosurface_trainable(self, field_id, iso, subdivisions, c, edges):
        """isosurface(..., coefficients=c): dg_field_set_nodes_device on torch's current stream, then K6 (the route of interpolate(coefficients=))"""
        import torch
        tf = self._trainable_field(field_id)        # the closures below keep it (not the grid) alive for the backward
        h, n_nodes = tf.handle, tf.n_nodes
        if not isinstance(c, torch.Tensor) or c.dtype != torch.float64:
            raise TypeError(f"isosurface: coefficients must be a float64 tensor (got {type(c).__name__ if not isinstance(c, torch.Tensor) else c.dtype})")
        if tuple(c.shape) != (n_nodes,):
            raise ValueError(f"isosurface: coefficients must have shape ({n_nodes},), got {tuple(c.shape)}")
        if not capi.EMULATED and (not c.is_cuda or c.device.index != tf.device):
            raise ValueError(f"isosurface: coefficients are on {c.device} but the field lives on cuda:{tf.device}")
        c = c.contiguous()

        token = object()                   # this call's pack: the backward repacks c unless the field still holds it

        def hold(cc, again):
            if again and tf.holds is token:
                return
            capi.check(capi.lib.dg_field_set_nodes_device(h, cc.data_ptr(), n_nodes, _device.stream(cc)))
            tf.holds = token

        def run(cc):
            hold(cc, False)
            if not capi.EMULATED:
                torch.cuda.current_stream(cc.device).synchronize()   # dg_isosurface_create runs on the legacy default stream
            return self._isosurface(h, iso, subdivisions, True, True)

        def vjp(cc, E, grad_V):
            hold(cc, True)
            gV = grad_V.to(torch.float64).contiguous()
            out = torch.empty(n_nodes, dtype=torch.float64, device=cc.device)
            capi.check(capi.lib.dg_isosurface_vjp_device(h, iso, subdivisions, len(E), E.data_ptr(), gV.data_ptr(), out.data_ptr(),
                                                         _device.stream(cc)))
            return out
        if torch.is_grad_enabled() and c.requires_grad:
            V, T, E = _isosurface_function().apply(c, run, vjp)
        else:
            V, T, E = run(c)
        return (V, T, E) if edges else (V, T)

    def raycast(self, field_id, origins, directions, iso=0.0, t_min=0.0, t_max=math.inf, coefficients=None):
        """The first crossing of {phi = iso} along rays x(t) = origin + t * direction, t in [t_min, t_max] clipped to the domain, on the
        field's GPU (dg_field_raycast; the contract is in csrc/k7_raycast.cu and DESIGN §3).  The crossing is isolated cell by cell with
        Bernstein bounds of the interpolant along the line, so features thinner than any step are not missed, on any field (SDF, density
        map, reduced band, user function).  A segment x0 -> x1 (continuous collision detection of a step) is raycast(f, x0, x1 - x0,
        t_min=0, t_max=1).  The values along the ray are the bits interpolate() returns there; DBL_MAX and non-finite values (outside the
        domain, removed cells) are never crossed.
        Returns (t_lo, t_hi, status): the final bisection bracket and DG_RAY_ENTER (1: phi(x(t_lo)) >= iso > phi(x(t_hi))), DG_RAY_LEAVE (2:
        the reverse; a ray that starts inside reports its first LEAVE) or DG_RAY_MISS (0, with t_lo = t_hi = inf).  numpy inputs (n, 3)
        give numpy arrays (float64, float64, int32).  float64 CUDA tensors (n, 3) on the field's device stay there: the cast runs on
        torch's current stream and returns CUDA tensors.  A reduced field's kept device handle is used directly.

        Gradients (K12, contract in csrc/k12_raycast_grad.cu): on CUDA tensors under grad mode, t_lo and t_hi are differentiable in the
        origins and the directions, by the implicit function theorem at x_c = x(t_lo): dt = -(grad phi . dx) / (grad phi . d), with both
        ends of the bracket following the crossing.  coefficients=c casts against the field with the node values c instead of its own, on
        the trainable device field interpolate(coefficients=) uses (same rules: c a float64 CUDA tensor of len(m_nodes[field_id]) values),
        and makes t_lo and t_hi differentiable in c as well, summed in a fixed order (K11).  A miss, a crossing at DBL_MAX or a ray tangent
        to the level set gets 0.  status carries no gradient.  First order only: a double backward raises.  Not differentiable in iso,
        t_min or t_max."""
        iso, t_min, t_max = float(iso), float(t_min), float(t_max)
        if coefficients is not None:
            if not (_device.is_device_query(origins) and _device.is_device_query(directions)):
                raise TypeError("raycast: coefficients= needs origins and directions as float64 CUDA tensors")
            return self._raycast_trainable(field_id, origins, directions, iso, t_min, t_max, coefficients)
        h = self._device_field(field_id)
        if _device.is_device_query(origins) or _device.is_device_query(directions):
            import torch
            info = (C.c_uint64 * 4)()
            capi.check(capi.lib.dg_field_info(h, info))
            o = _device.points(origins, int(info[3]), "raycast")
            d = _device.points(directions, int(info[3]), "raycast")
            if o.shape != d.shape:
                raise ValueError(f"raycast: origins {tuple(o.shape)} and directions {tuple(d.shape)} differ in shape")

            def run(oc, dc, _c):
                return self._raycast_device(h, oc, dc, iso, t_min, t_max)

            def vjp(oc, dc, _c, t_lo, status, g_lo, g_hi, needs):
                if self._fields.get(field_id) is not h:
                    raise RuntimeError(f"raycast: field {field_id} was replaced since the forward (setNodes, addFunction, reduceField or load); "
                                       "cast with coefficients= to keep a differentiable field")
                go, gd, _ = _raycast_vjp(h, oc, dc, t_lo, status, g_lo, g_hi, needs[0], needs[1], None)
                return go, gd, None
            if torch.is_grad_enabled() and (o.requires_grad or d.requires_grad):
                return _field_raycast_function().apply(o, d, None, run, vjp)
            return run(o, d, None)
        o = np.ascontiguousarray(origins, np.float64).reshape(-1, 3)
        d = np.ascontiguousarray(directions, np.float64).reshape(-1, 3)
        if o.shape != d.shape:
            raise ValueError(f"raycast: origins {o.shape} and directions {d.shape} differ in shape")
        t_lo, t_hi, status = np.empty(len(o)), np.empty(len(o)), np.empty(len(o), np.int32)
        capi.check(capi.lib.dg_field_raycast(h, capi.ptr(o, capi.F64P), capi.ptr(d, capi.F64P), len(o), iso, t_min, t_max,
                                             capi.ptr(t_lo, capi.F64P), capi.ptr(t_hi, capi.F64P), capi.ptr(status, capi.I32P)))
        return t_lo, t_hi, status

    @staticmethod
    def _raycast_device(h, o, d, iso, t_min, t_max):
        """dg_field_raycast_device on torch's current stream; o, d contiguous float64 (n, 3) tensors on the field's device"""
        import torch
        n = len(o)
        t_lo = torch.empty(n, dtype=torch.float64, device=o.device)
        t_hi = torch.empty(n, dtype=torch.float64, device=o.device)
        status = torch.empty(n, dtype=torch.int32, device=o.device)
        capi.check(capi.lib.dg_field_raycast_device(h, o.data_ptr(), d.data_ptr(), n, iso, t_min, t_max, t_lo.data_ptr(), t_hi.data_ptr(),
                                                    status.data_ptr(), _device.stream(o)))
        return t_lo, t_hi, status

    def _raycast_trainable(self, field_id, origins, directions, iso, t_min, t_max, c):
        """raycast(..., coefficients=c): dg_field_set_nodes_device, then K7, on torch's current stream (the route of interpolate(coefficients=))"""
        import torch
        tf = self._trainable_field(field_id)        # the closures below keep it (not the grid) alive for the backward
        h, n_nodes = tf.handle, tf.n_nodes
        o = _device.points(origins, tf.device, "raycast")
        d = _device.points(directions, tf.device, "raycast")
        if o.shape != d.shape:
            raise ValueError(f"raycast: origins {tuple(o.shape)} and directions {tuple(d.shape)} differ in shape")
        if not isinstance(c, torch.Tensor) or c.dtype != torch.float64:
            raise TypeError(f"raycast: coefficients must be a float64 tensor (got {type(c).__name__ if not isinstance(c, torch.Tensor) else c.dtype})")
        if tuple(c.shape) != (n_nodes,):
            raise ValueError(f"raycast: coefficients must have shape ({n_nodes},), got {tuple(c.shape)}")
        if not capi.EMULATED and (not c.is_cuda or c.device.index != tf.device):
            raise ValueError(f"raycast: coefficients are on {c.device} but the field lives on cuda:{tf.device}")
        c = c.contiguous()

        token = object()                   # this call's pack: the backward repacks c unless the field still holds it

        def hold(cc, again):
            if again and tf.holds is token:
                return
            capi.check(capi.lib.dg_field_set_nodes_device(h, cc.data_ptr(), n_nodes, _device.stream(cc)))
            tf.holds = token

        def run(oc, dc, cc):
            hold(cc, False)
            return self._raycast_device(h, oc, dc, iso, t_min, t_max)

        def vjp(oc, dc, cc, t_lo, status, g_lo, g_hi, needs):
            hold(cc, True)
            return _raycast_vjp(h, oc, dc, t_lo, status, g_lo, g_hi, needs[0], needs[1], n_nodes if needs[2] else None)
        if torch.is_grad_enabled() and (o.requires_grad or d.requires_grad or c.requires_grad):
            return _field_raycast_function().apply(o, d, c, run, vjp)
        return run(o, d, c)

    # ------------------------------------------------------------------ save / load (cubic_lagrange_discrete_grid.cpp:678-778)
    def save(self, filename):
        d = self._desc
        with open(filename, "wb") as fh:
            fh.write(struct.pack("<6d", *d.domain_min[:], *d.domain_max[:]))        # AlignedBox3d: min, max
            fh.write(struct.pack("<3I", *d.resolution[:]))
            fh.write(struct.pack("<3d", *d.cell_size[:]))
            fh.write(struct.pack("<3d", *d.inv_cell_size[:]))
            fh.write(struct.pack("<QQ", self.m_n_cells, self.m_n_fields))
            for arrs in (self.m_nodes, self.m_cells, self.m_cell_map):
                fh.write(struct.pack("<Q", len(arrs)))
                for a in arrs:
                    fh.write(struct.pack("<Q", len(a)))
                    fh.write(np.ascontiguousarray(a).tobytes())

    def load(self, filename):
        self._invalidate()
        try:
            fh = open(filename, "rb")
        except OSError:
            # reference: message on std::cerr, object left empty (:725-729)
            import sys
            print("ERROR: Discrete grid can not be loaded. Input file does not exist!", file=sys.stderr)
            return
        with fh:
            head = fh.read(48 + 12 + 24 + 24 + 16)
            mn_mx = struct.unpack_from("<6d", head, 0)
            res = struct.unpack_from("<3I", head, 48)
            cell = struct.unpack_from("<3d", head, 60)
            inv = struct.unpack_from("<3d", head, 84)
            n_cells, n_fields = struct.unpack_from("<QQ", head, 108)
            self._desc = grid_desc(mn_mx[:3], mn_mx[3:], res, cell, inv)     # cell sizes verbatim from the file
            self._sync_members()
            self.m_n_cells, self.m_n_fields = n_cells, n_fields

            def read_nested(dtype, width):
                (outer,) = struct.unpack("<Q", fh.read(8))
                out = []
                for _ in range(outer):
                    (n,) = struct.unpack("<Q", fh.read(8))
                    a = np.frombuffer(fh.read(n * width * np.dtype(dtype).itemsize), dtype=dtype).copy()
                    out.append(a.reshape(n, width) if width > 1 else a)
                return out

            self.m_nodes = read_nested(np.float64, 1)
            self.m_cells = read_nested(np.uint32, 32)
            self.m_cell_map = read_nested(np.uint32, 1)
