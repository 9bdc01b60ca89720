"""Host mirror of Discregrid::TriangleMeshDistance (geometry/TriangleMeshDistance.h:93-208) over the C-ABI.

Same surface -- construct from a TriangleMesh or from (vertices, triangles), signed_distance / unsigned_distance
returning Result(distance, nearest_point, nearest_entity, triangle_id) -- but batched: the argument is an (n, 3)
array of points (a single point is promoted) and each Result field is an array.  All queries run in the sm_90a
kernel of csrc/k1_sdf.cu; there is no host implementation.  Points given as a float64 CUDA tensor stay on the device and the
Result holds CUDA tensors.
"""
import ctypes as C
import math
from collections import namedtuple
from enum import IntEnum

import numpy as np

from . import _capi as capi
from . import _device
from .mesh import TriangleMesh


class NearestEntity(IntEnum):          # TriangleMeshDistance.h:75
    V0 = 0
    V1 = 1
    V2 = 2
    E01 = 3
    E12 = 4
    E02 = 5
    F = 6


Result = namedtuple("Result", ["distance", "nearest_point", "nearest_entity", "triangle_id"])   # :80-86
# Result with the barycentric weights (n, 3) of the nearest point on its triangle's vertices (beyond the reference)
NearestResult = namedtuple("NearestResult", ["distance", "nearest_point", "nearest_entity", "triangle_id", "barycentric"])

_MESH_DISTANCE = None


def _mesh_distance_function():
    """the autograd Function of the mesh distance on CUDA tensors (K10): distance(x, V) with d/dx = (x - p) / d and d/dV[F[t][i]] = -w_i d/dx,
    first order only.  The backward reads the saved forward outputs and the mesh's triangles, never its vertex positions.  Made at first
    use: torch is only imported by callers that pass tensors."""
    global _MESH_DISTANCE
    if _MESH_DISTANCE is None:
        import torch
        from torch.autograd.function import once_differentiable

        class MeshDistance(torch.autograd.Function):
            @staticmethod
            def forward(ctx, x, V, md, signed):
                r = md._nearest_device(x, signed)
                ctx.mark_non_differentiable(r.nearest_point, r.nearest_entity, r.triangle_id, r.barycentric)
                ctx.save_for_backward(x, r.distance, r.nearest_point, r.triangle_id, r.barycentric)
                ctx.md = md
                return tuple(r)

            @staticmethod
            @once_differentiable
            def backward(ctx, grad_distance, *_unused):
                x, dist, near, tri, bary = ctx.saved_tensors
                md = ctx.md
                n = len(x)
                if grad_distance is None:
                    grad_distance = torch.zeros(n, dtype=torch.float64, device=x.device)
                g = grad_distance.to(torch.float64).contiguous()
                gx = torch.empty((n, 3), dtype=torch.float64, device=x.device) if ctx.needs_input_grad[0] else None
                gv = torch.empty((md.n_vertices, 3), dtype=torch.float64, device=x.device) if ctx.needs_input_grad[1] else None
                capi.check(capi.lib.dg_mesh_distance_vjp_device(md.handle, n, x.data_ptr(), dist.data_ptr(), near.data_ptr(), tri.data_ptr(),
                                                                bary.data_ptr(), g.data_ptr(), None if gx is None else gx.data_ptr(),
                                                                None if gv is None else gv.data_ptr(), _device.stream(x)))
                return gx, gv, None, None
        _MESH_DISTANCE = MeshDistance
    return _MESH_DISTANCE


_MESH_RAYCAST = None


def _mesh_raycast_function():
    """the autograd Function of the mesh ray cast on CUDA tensors (K12): t and barycentric differentiable in the origins, the directions and
    the vertex positions, first order only.  The backward differentiates at the positions the forward cast against: V when it was given,
    otherwise the positions the mesh last took from construct or refit (uploaded at the first backward that needs them)."""
    global _MESH_RAYCAST
    if _MESH_RAYCAST is None:
        import torch
        from torch.autograd.function import once_differentiable

        class MeshRaycast(torch.autograd.Function):
            @staticmethod
            def forward(ctx, o, d, V, md, t_min, t_max):
                t, tid, bary, st = md._raycast_device(o, d, t_min, t_max)
                ctx.mark_non_differentiable(tid, st)
                ctx.set_materialize_grads(False)
                ctx.save_for_backward(d, t, tid, bary, V)
                ctx.md, ctx.positions = md, (None if V is not None else md._positions)
                return t, tid, bary, st

            @staticmethod
            @once_differentiable
            def backward(ctx, grad_t, _grad_tid, grad_bary, _grad_status):
                d, t, tid, bary, V = ctx.saved_tensors
                md = ctx.md
                need_o, need_d, need_v = ctx.needs_input_grad[0], ctx.needs_input_grad[1], ctx.needs_input_grad[2]
                if grad_t is None and grad_bary is None:
                    return None, None, None, None, None, None
                n = len(d)
                pos = V.detach().contiguous() if V is not None else md._positions_on(ctx.positions, d.device)
                go = torch.empty((n, 3), dtype=torch.float64, device=d.device) if need_o else None
                gd = torch.empty((n, 3), dtype=torch.float64, device=d.device) if need_d else None
                gv = torch.empty((md.n_vertices, 3), dtype=torch.float64, device=d.device) if need_v else None
                gt = None if grad_t is None else grad_t.to(torch.float64).contiguous()
                gb = None if grad_bary is None else grad_bary.to(torch.float64).contiguous()
                ptr = lambda a: None if a is None else a.data_ptr()
                capi.check(capi.lib.dg_mesh_raycast_vjp_device(md.handle, n, d.data_ptr(), t.data_ptr(), tid.data_ptr(), bary.data_ptr(),
                                                               pos.data_ptr(), ptr(gt), ptr(gb), ptr(go), ptr(gd), ptr(gv), _device.stream(d)))
                return go, gd, gv, None, None, None
        _MESH_RAYCAST = MeshRaycast
    return _MESH_RAYCAST


class TriangleMeshDistance:
    def __init__(self, mesh_or_vertices=None, triangles=None):
        self._h = None
        if mesh_or_vertices is not None:
            self.construct(mesh_or_vertices, triangles)

    # TriangleMeshDistance.h:251-267 (the std::vector overload; the raw-pointer overload's 3x over-allocation bug,
    # :232-249, is not reproduced)
    def construct(self, mesh_or_vertices, triangles=None):
        self.close()
        if isinstance(mesh_or_vertices, TriangleMesh):
            V, F = mesh_or_vertices.vertex_data(), mesh_or_vertices.face_data()
        else:
            V, F = mesh_or_vertices, triangles
        V = np.ascontiguousarray(V, dtype=np.float64).reshape(-1, 3)
        F = np.ascontiguousarray(F, dtype=np.uint32).reshape(-1, 3)
        h = C.c_void_p()
        capi.check(capi.lib.dg_mesh_create(capi.ptr(V, capi.F64P), len(V), capi.ptr(F, capi.U32P), len(F), C.byref(h)))
        self._h = h
        self._sign_mode = "pseudonormal"
        self.n_vertices, self.n_triangles = len(V), len(F)
        self._positions, self._positions_dev = V, None        # what raycast's backward differentiates at when it is not given V
        return self

    @property
    def is_constructed(self):
        return self._h is not None

    @property
    def handle(self):
        if self._h is None:
            # reference: prints "DistanceTriangleMesh error: not constructed." and exit(-1) (:318-321)
            raise capi.DiscregridError(capi.DG_ERR_INVALID, "DistanceTriangleMesh error: not constructed.")
        return self._h

    def close(self):
        if getattr(self, "_h", None) is not None:
            capi.lib.dg_mesh_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def info(self):
        a = (C.c_uint64 * 8)()
        capi.check(capi.lib.dg_mesh_info(self.handle, a))
        return {"n_vertices": a[0], "n_triangles": a[1], "stack_depth": a[2], "watertight_flags": a[3],
                "device_bytes": a[4], "build_us": a[5], "upload_us": a[6]}

    def tree(self):
        """(spheres[n,8], kids[n,2]) in the reference's node numbering (diagnostics)."""
        n = 2 * self.n_triangles - 1
        sph = np.empty((n, 8)); kids = np.empty((n, 2), np.int32)
        capi.check(capi.lib.dg_mesh_tree(self.handle, capi.ptr(sph, capi.F64P), capi.ptr(kids, capi.I32P)))
        return sph, kids

    def pseudonormals(self):
        tri = np.empty((self.n_triangles, 3)); edge = np.empty((self.n_triangles, 3, 3)); vert = np.empty((self.n_vertices, 3))
        capi.check(capi.lib.dg_mesh_pseudonormals(self.handle, capi.ptr(tri, capi.F64P), capi.ptr(edge, capi.F64P),
                                                  capi.ptr(vert, capi.F64P)))
        return tri, edge, vert

    @property
    def device(self):
        """the CUDA device the mesh lives on (the library's current device when it was constructed)"""
        a = (C.c_uint64 * 8)()
        capi.check(capi.lib.dg_mesh_info(self.handle, a))
        return int(a[7])

    def set_sign_mode(self, mode, beta=2.0):
        """Where signed distances take their sign from (beyond the reference).  "pseudonormal" (the default) is the reference's rule, the
        angle-weighted pseudonormal at the nearest entity, which is right only for closed manifold meshes.  "winding" takes it from the
        generalized winding number: inside iff winding_number(x, beta) > 0.5, which holds for open, non-manifold and self-intersecting
        meshes too.  signed_distance, MeshSignedDistance, MeshDistanceBand and the grid calls built on them follow the mode; multi-GPU
        sampling refuses the winding mode.  beta >= 1 or inf (exact).  Not to be called while another thread queries this mesh."""
        modes = {"pseudonormal": capi.DG_SIGN_PSEUDONORMAL, "winding": capi.DG_SIGN_WINDING}
        if mode not in modes:
            raise ValueError(f"sign mode must be 'pseudonormal' or 'winding' (got {mode!r})")
        capi.check(capi.lib.dg_mesh_set_sign_mode(self.handle, modes[mode], float(beta)))
        self._sign_mode = mode
        return self

    def refit(self, vertices):
        """Moves the mesh's vertices to `vertices` (n_vertices x 3, the count of the construction) and refits every device record to
        them: the sphere tree, the pseudonormals and, once used, the winding records (beyond the reference).  The triangles and the tree's
        leaf order stay those of the construction, so a large deformation loosens the tree and queries slow down; construct again then.
        A numpy array (or anything numpy converts) is uploaded first; a float64 CUDA tensor of shape (n_vertices, 3) on the mesh's device
        is read in place, on torch's current stream after the work queued there.  Returns when the refit has finished; returns self.  Not
        to be called while another call uses this mesh, on any stream."""
        if _device.is_device_query(vertices):
            x = _device.points(vertices, self.device, "refit")
            capi.check(capi.lib.dg_mesh_refit_device(self.handle, x.data_ptr(), len(x), _device.stream(x)))
            self._positions, self._positions_dev = x.detach(), None
            return self
        V = np.ascontiguousarray(vertices, dtype=np.float64)
        if V.ndim != 2 or V.shape[1] != 3:
            raise ValueError(f"refit: vertices must have shape (n_vertices, 3) (got {V.shape})")
        capi.check(capi.lib.dg_mesh_refit(self.handle, capi.ptr(V, capi.F64P), len(V)))
        self._positions, self._positions_dev = V, None
        return self

    @property
    def sign_mode(self):
        return getattr(self, "_sign_mode", "pseudonormal")

    def winding_number(self, points, beta=2.0):
        """Generalized winding number w(x) of the mesh (Barill et al. 2018) at points (n, 3) or (3,): 1 inside a closed surface, 0 outside,
        fractional near holes.  Clusters of triangles farther than beta times their radius are summed by a far-field expansion; beta = inf
        sums every triangle exactly.  A numpy array returns a numpy array; a float64 CUDA tensor on the mesh's device returns a CUDA tensor,
        computed on torch's current stream with the same bits."""
        beta = float(beta)
        if _device.is_device_query(points):
            import torch
            x = _device.points(points, self.device, "winding_number")
            w = torch.empty(len(x), dtype=torch.float64, device=x.device)
            capi.check(capi.lib.dg_mesh_winding_number_device(self.handle, x.data_ptr(), len(x), beta, w.data_ptr(), _device.stream(x)))
            return w
        x = np.ascontiguousarray(points, dtype=np.float64).reshape(-1, 3)
        w = np.empty(len(x))
        capi.check(capi.lib.dg_mesh_winding_number(self.handle, capi.ptr(x, capi.F64P), len(x), beta, capi.ptr(w, capi.F64P)))
        return w

    def raycast(self, origins, directions, t_min=0.0, t_max=math.inf, vertices=None):
        """The first hit of each ray on the mesh's triangles (beyond the reference; dg_mesh_raycast, contract in csrc/k9_mesh_raycast.cu and
        DESIGN §3).  origins and directions (n, 3) or (3,); t in [t_min, t_max].  A segment x0 -> x1 (continuous collision detection of a
        step against a deforming mesh: refit, then cast) is raycast(x0, x1 - x0, 0.0, 1.0).  The test is watertight: a ray through a shared
        edge or vertex is not lost.  Returns (t, triangle_id, barycentric, status): the least t (the lower id wins a tie), the original
        triangle index, the weights (n, 3) of that triangle's vertices 0, 1, 2, and DG_RAY_ENTER (1: crossing from the outside of an
        outward-oriented mesh) or DG_RAY_LEAVE (2); a miss gives DG_RAY_MISS (0), t = inf, id -1 and NaN weights.  numpy inputs return numpy
        arrays; float64 CUDA tensors on the mesh's device stay there and the cast runs on torch's current stream.

        Gradients (K12, contract in csrc/k12_raycast_grad.cu): on CUDA tensors under grad mode, t and barycentric are differentiable in the
        origins and the directions, and in the vertex positions: vertices=V, a float64 CUDA tensor (n_vertices, 3) on the mesh's device,
        first refits the mesh to V.detach() -- a side effect that stays, as refit(V) -- and makes the hit differentiable in V.  The backward
        differentiates at the positions the forward cast against (V, or else those the mesh last took from construct or refit), so a refit
        between forward and backward does not change it.  A miss, or a ray parallel to its triangle, gets 0; the vertex gradient is summed
        in a fixed order, the same bits on every run.  triangle_id and status carry no gradient.  First order only: a double backward
        raises.  A depth loss is loss(t); the time of impact of a step x0 -> x1 is raycast(x0, x1 - x0, 0, 1)[0]."""
        t_min, t_max = float(t_min), float(t_max)
        if vertices is not None:
            self._refit_to(vertices, "raycast")
        if _device.is_device_query(origins) or _device.is_device_query(directions):
            import torch
            o = _device.points(origins, self.device, "raycast")
            d = _device.points(directions, self.device, "raycast")
            if o.shape != d.shape:
                raise ValueError(f"raycast: origins {tuple(o.shape)} and directions {tuple(d.shape)} differ in shape")
            if torch.is_grad_enabled() and (o.requires_grad or d.requires_grad or (vertices is not None and vertices.requires_grad)):
                return _mesh_raycast_function().apply(o, d, vertices, self, t_min, t_max)
            return self._raycast_device(o, d, t_min, t_max)
        o = np.ascontiguousarray(origins, dtype=np.float64).reshape(-1, 3)
        d = np.ascontiguousarray(directions, dtype=np.float64).reshape(-1, 3)
        if o.shape != d.shape:
            raise ValueError(f"raycast: origins {o.shape} and directions {d.shape} differ in shape")
        n = len(o)
        t = np.empty(n); tid = np.empty(n, np.int32); bary = np.empty((n, 3)); st = np.empty(n, np.int32)
        capi.check(capi.lib.dg_mesh_raycast(self.handle, capi.ptr(o, capi.F64P), capi.ptr(d, capi.F64P), n, t_min, t_max, capi.ptr(t, capi.F64P),
                                            capi.ptr(tid, capi.I32P), capi.ptr(bary, capi.F64P), capi.ptr(st, capi.I32P)))
        return t, tid, bary, st

    def _raycast_device(self, o, d, t_min, t_max):
        """dg_mesh_raycast_device on torch's current stream; o, d contiguous float64 (n, 3) tensors on the mesh's device"""
        import torch
        n = len(o)
        t = torch.empty(n, dtype=torch.float64, device=o.device)
        tid = torch.empty(n, dtype=torch.int32, device=o.device)
        bary = torch.empty((n, 3), dtype=torch.float64, device=o.device)
        st = torch.empty(n, dtype=torch.int32, device=o.device)
        capi.check(capi.lib.dg_mesh_raycast_device(self.handle, o.data_ptr(), d.data_ptr(), n, t_min, t_max, t.data_ptr(), tid.data_ptr(),
                                                   bary.data_ptr(), st.data_ptr(), _device.stream(o)))
        return t, tid, bary, st

    def _positions_on(self, positions, device):
        """positions (what construct or refit last took) as a contiguous float64 tensor on `device`; a host array is uploaded once, at the
        first backward that needs it, and kept while it stays the mesh's positions"""
        import torch
        if isinstance(positions, torch.Tensor):
            return positions.to(device=device, dtype=torch.float64).contiguous()
        cached = self._positions_dev
        if cached is not None and cached[0] is positions:
            return cached[1]
        dev = torch.from_numpy(np.ascontiguousarray(positions, np.float64).reshape(-1, 3)).to(device)
        if positions is self._positions:
            self._positions_dev = (positions, dev)
        return dev

    def _query_device(self, points, signed):
        """the CUDA-tensor route: dg_mesh_distance_device on torch's current stream, asynchronous like a torch op"""
        import torch
        x = _device.points(points, self.device, "signed_distance" if signed else "unsigned_distance")
        n = len(x)
        dist = torch.empty(n, dtype=torch.float64, device=x.device)
        near = torch.empty((n, 3), dtype=torch.float64, device=x.device)
        ent = torch.empty(n, dtype=torch.int32, device=x.device)
        tri = torch.empty(n, dtype=torch.int32, device=x.device)
        capi.check(capi.lib.dg_mesh_distance_device(self.handle, x.data_ptr(), n, int(signed), dist.data_ptr(), near.data_ptr(), ent.data_ptr(),
                                                    tri.data_ptr(), _device.stream(x)))
        return Result(dist, near, ent, tri)

    def _nearest_device(self, x, signed):
        """dg_mesh_distance_bary_device on torch's current stream; x a contiguous float64 (n, 3) tensor on the mesh's device"""
        import torch
        n = len(x)
        dist = torch.empty(n, dtype=torch.float64, device=x.device)
        near = torch.empty((n, 3), dtype=torch.float64, device=x.device)
        ent = torch.empty(n, dtype=torch.int32, device=x.device)
        tri = torch.empty(n, dtype=torch.int32, device=x.device)
        bary = torch.empty((n, 3), dtype=torch.float64, device=x.device)
        capi.check(capi.lib.dg_mesh_distance_bary_device(self.handle, x.data_ptr(), n, int(signed), dist.data_ptr(), near.data_ptr(),
                                                         ent.data_ptr(), tri.data_ptr(), bary.data_ptr(), _device.stream(x)))
        return NearestResult(dist, near, ent, tri, bary)

    def nearest(self, points, signed=True):
        """The query of signed_distance (signed=True) or unsigned_distance with the barycentric weights of the nearest point (beyond the
        reference; dg_mesh_distance_bary): NearestResult(distance, nearest_point, nearest_entity, triangle_id, barycentric).  barycentric
        (n, 3) weighs the vertices F[t][0], F[t][1], F[t][2] of the nearest triangle t, so that nearest_point is their weighted sum as the
        query computes it: one-hot at a vertex, on the edge for an edge, NaN where no triangle was found (NaN points).  The other four fields
        are bit for bit those of signed_distance / unsigned_distance.  numpy in, numpy out; a float64 CUDA tensor on the mesh's device
        returns CUDA tensors, computed on torch's current stream.  No autograd (see signed_distance)."""
        if _device.is_device_query(points):
            x = _device.points(points, self.device, "nearest")
            return self._nearest_device(x.detach(), signed)
        x = np.ascontiguousarray(points, dtype=np.float64).reshape(-1, 3)
        n = len(x)
        dist = np.empty(n); near = np.empty((n, 3)); ent = np.empty(n, np.int32); tri = np.empty(n, np.int32); bary = np.empty((n, 3))
        capi.check(capi.lib.dg_mesh_distance_bary(self.handle, capi.ptr(x, capi.F64P), n, int(signed), capi.ptr(dist, capi.F64P),
                                                  capi.ptr(near, capi.F64P), capi.ptr(ent, capi.I32P), capi.ptr(tri, capi.I32P),
                                                  capi.ptr(bary, capi.F64P)))
        return NearestResult(dist, near, ent, tri, bary)

    def _differentiable(self, points, vertices, signed):
        """the autograd route of a CUDA-tensor query: None when nothing asks for a gradient"""
        import torch
        if not torch.is_grad_enabled():
            return None
        if not (points.requires_grad or (vertices is not None and vertices.requires_grad)):
            return None
        x = _device.points(points, self.device, "signed_distance" if signed else "unsigned_distance")
        dist, near, ent, tri, _bary = _mesh_distance_function().apply(x, vertices, self, signed)
        return Result(dist, near, ent, tri)

    def _refit_to(self, vertices, who):
        import torch
        if not _device.is_device_query(vertices):
            raise TypeError(f"{who}: vertices must be a float64 CUDA tensor of shape (n_vertices, 3) (got {type(vertices).__name__})")
        if vertices.dtype != torch.float64 or vertices.dim() != 2 or tuple(vertices.shape) != (self.n_vertices, 3):
            raise ValueError(f"{who}: vertices must be a float64 tensor of shape ({self.n_vertices}, 3) (got {vertices.dtype}, "
                             f"{tuple(vertices.shape)})")
        self.refit(vertices.detach())

    def _query(self, points, signed, vertices=None):
        if vertices is not None:
            self._refit_to(vertices, "signed_distance" if signed else "unsigned_distance")
        if _device.is_device_query(points):
            r = self._differentiable(points, vertices, signed)
            if r is not None:
                return r
            return self._query_device(points, signed)
        x = np.ascontiguousarray(points, dtype=np.float64).reshape(-1, 3)
        n = len(x)
        dist = np.empty(n); near = np.empty((n, 3)); ent = np.empty(n, np.int32); tri = np.empty(n, np.int32)
        capi.check(capi.lib.dg_mesh_distance(self.handle, capi.ptr(x, capi.F64P), n, int(signed), capi.ptr(dist, capi.F64P),
                                             capi.ptr(near, capi.F64P), capi.ptr(ent, capi.I32P), capi.ptr(tri, capi.I32P)))
        return Result(dist, near, ent, tri)

    def signed_distance(self, points, vertices=None):      # :269-314
        """points: (n, 3) or (3,).  A numpy array (or anything numpy converts, CPU tensors included) goes through the host pipeline and
        returns numpy arrays.  A float64 torch tensor on the mesh's CUDA device stays there: the query runs on torch's current stream,
        asynchronously, and the Result holds CUDA tensors (distance float64 (n,), nearest_point float64 (n, 3), nearest_entity and
        triangle_id int32 (n,)) with the same bits as the host route.

        Gradients (beyond the reference): when the tensor requires grad, `distance` is differentiable in the points, d/dx = (x - p) / d
        (0 where d = 0 or no triangle was found).  vertices=V, a float64 CUDA tensor (n_vertices, 3) on the mesh's device, first refits the
        mesh to V.detach() -- a side effect that stays, as refit(V) -- and makes `distance` differentiable in V as well, through the nearest
        point's barycentric weights (envelope theorem).  The vertex gradient is summed in a fixed order: the same bits on every run.  The
        backward runs on torch's current stream and reads only the forward's outputs and the triangles, so refitting the mesh again before
        backward() does not change it.  First order only: a double backward raises.  nearest_point, nearest_entity and triangle_id carry no
        gradient."""
        return self._query(points, True, vertices)

    def unsigned_distance(self, points, vertices=None):    # :316-334
        """as signed_distance, unsigned"""
        return self._query(points, False, vertices)


class MeshSignedDistance:
    """The functor GenerateSDF hands to addFunction (cmd/generate_sdf/main.cpp:94-102):
    x -> sign * md.signed_distance(x).distance, sign = -1 for --invert.  CubicLagrangeDiscreteGrid.addFunction
    recognises this type and samples it on the GPU (the reference takes an opaque std::function, which a GPU
    cannot run -- SURVEY F6/H1)."""

    def __init__(self, md, invert=False):
        self.md = md
        self.sign = -1.0 if invert else 1.0

    def __call__(self, points):
        d = self.md.signed_distance(points).distance
        return d if self.sign == 1.0 else self.sign * d


class MeshDistanceBand:
    """The narrow-band sample predicate x -> |md.signed_distance(x).distance| <= band (fp64, the reference's own distance): what a
    reference user passes as addFunction's `pred` to keep a signed distance field only near the surface.  Callable on points like the
    reference's predicate (returns bool per point).  CubicLagrangeDiscreteGrid.addFunction(MeshSignedDistance(md), pred=MeshDistanceBand(md, w))
    recognises it and samples the band on the GPU: nodes outside hold DBL_MAX, blocks of nodes provably outside are never queried."""

    def __init__(self, md, band):
        band = float(band)
        if not band >= 0.0:
            raise ValueError(f"band must be >= 0 (got {band})")
        self.md, self.band = md, band

    def __call__(self, points):
        return np.abs(self.md.signed_distance(points).distance) <= self.band
