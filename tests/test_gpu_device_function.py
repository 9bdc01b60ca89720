"""User functions on the GPU -- dg_add_function_device, dg_reduced_function_create, dg_reduce_field_device, the Python types DeviceFunction /
DeviceSamplePredicate / DeviceNodePredicate with torch callbacks, and the C++ facade -- against the reference's own fixtures
(tests/golden/make_device_function_golden.py) and against the host route (positions to the host, numpy, addSampledFunction, dg_reduce_field
with every pass on the host).  Bar: bit-exact.  Eager torch runs one kernel per operation and the sums are written as explicit adds in the
reference lambda's order, so the torch function computes the same doubles as the reference's std::sqrt((dx*dx + dy*dy) + dz*dz) - r."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from conftest import GOLDEN, ROOT, bits_equal
from test_device_function_emulated import (CASES, REFERENCE_SORT, func_np, host_route, reduce_np, same_field, sample_np)
from test_oracle_golden import read_cdf

pytestmark = pytest.mark.gpu

DEVICE_FUNCTION_CHECK = os.path.join(ROOT, "build", "bin", "device_function_check")


def lib():
    from discregrid_b200 import _capi
    return _capi.lib


# ------------------------------------------------------------------------------------------------ the analytic case in eager torch
def sqrt_t(s):
    """a correctly rounded square root, as std::sqrt: torch.sqrt on CUDA tensors; on the CPU tensors of the emulated rehearsal numpy's, since
    torch's vectorised CPU kernel is not always correctly rounded"""
    import torch
    return torch.sqrt(s) if s.is_cuda else torch.from_numpy(np.sqrt(s.numpy()))


def func_t(p):
    def f(x, keep):
        dx, dy, dz = x[:, 0] - p["centre"][0], x[:, 1] - p["centre"][1], x[:, 2] - p["centre"][2]
        return sqrt_t((dx * dx + dy * dy) + dz * dz) - p["r"]
    return f


def sample_t(p):
    return lambda x: x[:, 0] + 0.5 * x[:, 1] < p["c"]


def reduce_t(p):
    return lambda x, v: (v <= p["vmax"]) & (x[:, 2] > p["z0"])


def types_of(dg, case):
    f = dg.DeviceFunction(func_t(case))
    s = dg.DeviceSamplePredicate(sample_t(case)) if case["sample"] else None
    q = dg.DeviceNodePredicate(reduce_t(case)) if case["reduce"] else None
    return f, s, q


def new_grid(dg, case):
    return dg.CubicLagrangeDiscreteGrid(case["mn"], case["mx"], case["res"])


def field(g, k=0):
    return g.m_nodes[k], g.m_cells[k], g.m_cell_map[k]


@pytest.mark.parametrize("name", sorted(CASES))
def test_fixtures_python_types(dg, tmp_path, name):
    """addFunction(DeviceFunction, pred=DeviceSamplePredicate), reduceField(DeviceNodePredicate) and addReducedFunction write the
    reference's file byte for byte and equal the host route bit for bit"""
    case = CASES[name]
    want = open(os.path.join(GOLDEN, case["file"]), "rb").read()
    f, s, q = types_of(dg, case)
    two = new_grid(dg, case)
    assert two.addFunction(f, False, s) == 0
    dense, reduced = host_route(lib(), two._desc, lambda x, k: func_np(x, case), (lambda x: sample_np(x, case)) if s else None,
                                (lambda x, v: reduce_np(x, v, case)) if q else None)
    assert same_field(field(two), dense)
    if q is not None:
        two.reduceField(0, q)
        assert same_field(field(two), reduced[0])
    out = str(tmp_path / "two.cdf"); two.save(out)
    assert open(out, "rb").read() == want
    if q is not None:
        one = new_grid(dg, case)
        assert one.addReducedFunction(f, s, q) == 0 and one.last_reduced_function_ms[5] == reduced[1]
        out = str(tmp_path / "one.cdf"); one.save(out)
        assert open(out, "rb").read() == want


@pytest.mark.parametrize("flags", [0, REFERENCE_SORT])
@pytest.mark.parametrize("chunk", [1000, 0])
def test_capi_chunks_and_sorts(dg, flags, chunk):
    """the C-ABI with torch callbacks, a chunk size that does not divide the grid and the default, both sorts: the reference's aniso field"""
    import ctypes as C
    from discregrid_b200 import _capi
    from discregrid_b200.grid import _DeviceCallbacks, _copy_reduced
    case = CASES["aniso_reduced"]
    g = new_grid(dg, case)
    f, s, q = types_of(dg, case)
    cb = _DeviceCallbacks(func=f, sample=s, node=q)
    h, tm = C.c_void_p(), np.zeros(8)
    cb.check(lib().dg_reduced_function_create(C.byref(g._desc), cb.func, None, cb.sample, None, cb.node, None, chunk, flags, C.byref(h),
                                              _capi.ptr(tm, _capi.F64P)))
    got = _copy_reduced(h, g.m_n_cells)
    want = read_cdf(os.path.join(GOLDEN, case["file"]))
    assert bits_equal(got[0], want["nodes"][0]) and np.array_equal(got[1], want["cells"][0]) and np.array_equal(got[2], want["cmap"][0])
    assert tm[5] == 1.0 and tm[6] >= tm[7] >= 0


def test_python_rules_and_exceptions(dg):
    """an exception inside fn is re-raised after the call (the library returned DG_ERR_CALLBACK); a wrong dtype or shape is a TypeError; device
    and host types do not mix; nothing changes the grid"""
    from discregrid_b200 import DiscregridError
    case = CASES["box_reduced"]
    g = new_grid(dg, case)
    f, _, q = types_of(dg, case)

    class Boom(Exception):
        pass

    def boom(x, keep):
        raise Boom("from fn")
    with pytest.raises(Boom):
        g.addFunction(dg.DeviceFunction(boom))
    with pytest.raises(Boom):
        g.addReducedFunction(f, None, dg.DeviceNodePredicate(lambda x, v: (_ for _ in ()).throw(Boom("from pred"))))
    with pytest.raises(TypeError, match="float64"):
        g.addFunction(dg.DeviceFunction(lambda x, k: x[:, 0].float()))
    with pytest.raises(TypeError):
        g.addFunction(dg.DeviceFunction(lambda x, k: x[:, 0] > 0))
    with pytest.raises(TypeError):
        g.addFunction(f, False, lambda x: True)
    with pytest.raises(TypeError):
        g.addFunction(lambda x: 0.0, False, dg.DeviceSamplePredicate(sample_t(case)))
    with pytest.raises(TypeError):
        g.addReducedFunction(lambda x, k: x[:, 0])
    with pytest.raises(TypeError):
        dg.DeviceFunction(3.0)
    assert g.nFields() == 0
    assert g.addFunction(f) == 0
    nodes = g.m_nodes[0].copy()
    with pytest.raises(Boom):
        g.reduceField(0, dg.DeviceNodePredicate(lambda x, v: (_ for _ in ()).throw(Boom("from pred"))))
    assert bits_equal(g.m_nodes[0], nodes)
    g.reduceField(0, q)
    with pytest.raises(DiscregridError, match="already reduced"):
        g.reduceField(0, q)


def mesh_distance_function(dg, md):
    """a DeviceFunction that calls dg_mesh_distance_device on the positions, on the library's stream"""
    import torch
    from discregrid_b200 import _capi

    def f(x, keep):
        out = torch.empty(len(x), dtype=torch.float64, device=x.device)
        stream = None if _capi.EMULATED else torch.cuda.current_stream().cuda_stream
        _capi.check(_capi.lib.dg_mesh_distance_device(md.handle, x.data_ptr(), len(x), 1, out.data_ptr(), None, None, None, stream))
        return out
    return dg.DeviceFunction(f)


def mesh_case(dg, name, res):
    if name == "box":
        mesh = dg.box()
    else:
        from conftest import ref_resource
        path = ref_resource(name)
        if path is None:
            pytest.skip(f"{name} not staged (make -C oracle ref)")
        mesh = dg.TriangleMesh(path)
    md = dg.TriangleMeshDistance(mesh)
    mn, mx = dg.generate_sdf_domain(mesh.vertices)
    return md, mn, mx


def check_mesh_distance(dg, name, res):
    md, mn, mx = mesh_case(dg, name, res)
    a = dg.CubicLagrangeDiscreteGrid(mn, mx, (res, res, res))
    a.addFunction(dg.MeshSignedDistance(md))
    b = dg.CubicLagrangeDiscreteGrid(mn, mx, (res, res, res))
    b.addFunction(mesh_distance_function(dg, md))
    assert same_field(field(b), field(a))


def test_mesh_distance_callback_box(dg):
    check_mesh_distance(dg, "box", 6)


def test_full_size_mesh_distance_callback_bunny_128(dg):
    """the device route with dg_mesh_distance_device as the function gives exactly addFunction(MeshSignedDistance)'s field"""
    check_mesh_distance(dg, "bunny.obj", 128)


ANALYTIC = dict(mn=(-1.0, -1.0, -1.0), mx=(1.0, 1.0, 1.0), centre=(0.13, -0.07, 0.21), r=0.55, c=0.6, vmax=0.02, z0=-0.5, sample=True, reduce=True)


def test_full_size_analytic_256(dg):
    """256^3: addReducedFunction against addFunction + reduceField (both with device callbacks) and against the numpy host route"""
    case = dict(ANALYTIC, res=(256, 256, 256))
    f, s, q = types_of(dg, case)
    one = new_grid(dg, case)
    one.addReducedFunction(f, s, q)
    two = new_grid(dg, case)
    two.addFunction(f, False, s)
    dense, reduced = host_route(lib(), two._desc, lambda x, k: func_np(x, case), lambda x: sample_np(x, case), lambda x, v: reduce_np(x, v, case))
    assert same_field(field(two), dense)
    del dense
    two.reduceField(0, q)
    assert same_field(field(one), field(two)) and same_field(field(one), reduced[0])
    assert 0 < len(one.m_nodes[0]) < one.nNodes() // 4


def test_full_size_analytic_256_peak_rss():
    """the one-call route at 256^3 in a fresh process: what it adds to the peak RSS of a process whose torch, CUDA context and kernels are
    already up (a small grid runs first) stays below the survivors + cell map + the host sort's arrays (a 64-bit key, a 16-byte key/position
    pair and a 32-bit rank per survivor) + 512 MiB; the dense route's node positions alone would take 2.8 GB.  The process is started from a
    small probe, so that its peak does not start at this test process's own (Linux carries the peak RSS across exec)."""
    code = ("import json, resource, sys; sys.path.insert(0, sys.argv[1]); sys.path.insert(0, sys.argv[1] + '/tests'); import discregrid_b200 as dg; "
            "from test_gpu_device_function import ANALYTIC, types_of, new_grid; "
            "w = dict(ANALYTIC, res=(8, 8, 8)); new_grid(dg, w).addReducedFunction(*types_of(dg, w)); "
            "base = resource.getrusage(resource.RUSAGE_SELF).ru_maxrss; case = dict(ANALYTIC, res=(256, 256, 256)); g = new_grid(dg, case); "
            "g.addReducedFunction(*types_of(dg, case)); "
            "print(json.dumps([len(g.m_nodes[0]), len(g.m_cells[0]), g.nNodes(), g.nCells(), base, resource.getrusage(resource.RUSAGE_SELF).ru_maxrss]))")
    probe = "import subprocess, sys; r = subprocess.run(sys.argv[1:]); sys.exit(r.returncode)"
    r = subprocess.run([sys.executable, "-c", probe, sys.executable, "-c", code, ROOT], capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0, r.stderr[-3000:]
    m, c, n, nc, base_kib, peak_kib = json.loads(r.stdout.strip().splitlines()[-1])
    bound = 8 * m + 128 * c + 4 * nc + (8 + 16 + 4) * m + (512 << 20)
    assert (peak_kib - base_kib) * 1024 < bound, (base_kib, peak_kib, m, c, n, nc)


def test_cpp_facade_check(tmp_path):
    """the C++ facade's DeviceFunction / DeviceSamplePredicate / DeviceNodePredicate (callbacks that move data with cudaMemcpyAsync on the
    given stream): addReducedFunction and addFunction + reduceField write the reference's files byte for byte"""
    for name, case in sorted(CASES.items()):
        vals = [*case["mn"], *case["mx"], *case["res"], *case["centre"], case["r"], case["c"], case["vmax"], case["z0"]]
        out = str(tmp_path / name)
        r = subprocess.run([DEVICE_FUNCTION_CHECK, out] + [float.hex(float(v)) for v in vals] + [str(int(case["sample"])), str(int(case["reduce"]))],
                           capture_output=True, text=True, timeout=600)
        assert r.returncode == 0, r.stdout + r.stderr
        want = open(os.path.join(GOLDEN, case["file"]), "rb").read()
        assert open(out + "_two.cdf", "rb").read() == want, name
        if case["reduce"]:
            assert open(out + "_one.cdf", "rb").read() == want, name
        else:
            assert open(out + "_dense.cdf", "rb").read() == want, name


def _late_centre(case, stream):
    """a centre tensor whose true value is written on `stream` only after ~0.1 s of GPU work queued ahead of it: a callback that ran before
    that work finished would read zeros"""
    import torch
    centre = torch.zeros(3, dtype=torch.float64, device="cuda")
    value = torch.tensor(case["centre"], dtype=torch.float64, device="cuda")
    torch.cuda.synchronize()
    with torch.cuda.stream(stream):
        torch.cuda._sleep(200_000_000)
        centre.copy_(value)                          # device to device: queued behind the sleep, the host does not wait
    return centre


def _centre_function(centre, r):
    def f(x, keep):
        dx, dy, dz = x[:, 0] - centre[0], x[:, 1] - centre[1], x[:, 2] - centre[2]
        return sqrt_t((dx * dx + dy * dy) + dz * dz) - r
    return f


def test_callbacks_see_tensors_computed_before_the_call(dg):
    """a DeviceFunction that reads a tensor produced just before the call -- on torch's default stream and on a side stream that is current
    at the call -- sees its final value"""
    from discregrid_b200 import _capi
    if _capi.EMULATED:
        pytest.skip("stream order needs a GPU")
    import torch
    case = CASES["aniso_reduced"]
    f, s, q = types_of(dg, case)
    want = open(os.path.join(GOLDEN, case["file"]), "rb").read()
    for stream in (torch.cuda.default_stream(), torch.cuda.Stream()):
        with torch.cuda.stream(stream):
            centre = _late_centre(case, stream)
            g = new_grid(dg, case)
            g.addReducedFunction(dg.DeviceFunction(_centre_function(centre, case["r"])), s, q)
        path = os.path.join(ROOT, "build", "pytest-tmp", "late_centre.cdf")
        os.makedirs(os.path.dirname(path), exist_ok=True)
        g.save(path)
        assert open(path, "rb").read() == want, stream


def test_capi_stream_waits_for_the_legacy_default_stream(dg):
    """the C-ABI alone (callbacks that do not order anything themselves): the library's stream starts after the work queued on the legacy
    default stream before the call"""
    import ctypes as C
    from discregrid_b200 import _capi
    from discregrid_b200.grid import _DeviceCallbacks
    if _capi.EMULATED:
        pytest.skip("stream order needs a GPU")
    import torch
    case = CASES["box_reduced"]
    g = new_grid(dg, case)
    dense, _ = host_route(lib(), g._desc, lambda x, k: func_np(x, case))
    views = _DeviceCallbacks()
    centre = _late_centre(case, torch.cuda.default_stream())
    fn = _centre_function(centre, case["r"])

    def raw(_u, x, keep, n, values, stream):
        with torch.cuda.stream(torch.cuda.ExternalStream(stream)):       # no wait_stream here: the order is the library's
            views._view(values, (n,), "<f8", torch.float64).copy_(fn(views._view(x, (n, 3), "<f8", torch.float64), None))
        return 0
    cb = _capi.DEVICE_FUNCTION(raw)
    n = g.nNodes()
    nodes, cells, cmap = np.empty(n), np.empty((g.m_n_cells, 32), np.uint32), np.empty(g.m_n_cells, np.uint32)
    _capi.check(lib().dg_add_function_device(C.byref(g._desc), cb, None, _capi.DEVICE_SAMPLE_PREDICATE(), None, 0, _capi.ptr(nodes, _capi.F64P),
                                             _capi.ptr(cells, _capi.U32P), _capi.ptr(cmap, _capi.U32P), None))
    assert same_field((nodes, cells, cmap), dense)


def test_repeated_calls_reuse_cached_memory(dg):
    """calls in a row run on the same library stream, so torch's cached blocks from the callbacks of one call serve the next: the memory torch
    holds stops growing after the first calls"""
    from discregrid_b200 import _capi
    if _capi.EMULATED:
        pytest.skip("torch's CUDA caching allocator needs a GPU")
    import torch
    case = dict(ANALYTIC, res=(96, 96, 96))
    f, s, q = types_of(dg, case)
    reserved = []
    for _ in range(6):
        new_grid(dg, case).addReducedFunction(f, s, q)
        reserved.append(torch.cuda.memory_reserved())
    assert reserved[-1] == reserved[1], reserved
