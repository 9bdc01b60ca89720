"""Refusals of the C-ABI's point queries, host and device form alike, on the CPU: the product's dg_api.cu with every kernel emulated
(build/bin/libdgemu.so, tests/emu).  Each row of the table is one refused input -- a NULL handle, a NULL array, a bad range, a bad scalar --
and is run through both forms of its query: the status code must be DG_ERR_INVALID and the message must start with the name of the entry
point that was called.  The valid calls the rows are made from, and empty calls with NULL arrays, must succeed."""
import ctypes as C
import math
import os

import numpy as np
import pytest

from conftest import GOLDEN
from test_oracle_golden import read_obj
from test_isosurface_emulated import emu, make_field  # noqa: F401 (emu: fixture)

DG_ERR_INVALID = -1
NAN, INF = math.nan, math.inf
N = 4                                                   # points per call
PAST_END = lambda s: s.n_nodes + 1                      # noqa: E731 (a node range end one past the grid's nodes)


class Handles:
    """a mesh, a field and valid arrays for N points of every query"""

    def __init__(self, lib):
        V, F = read_obj(os.path.join(GOLDEN, "box.obj"))
        V = np.ascontiguousarray(V, np.float64); F = np.ascontiguousarray(F, np.uint32)
        self.mesh = C.c_void_p()
        assert lib.dg_mesh_create(V.ctypes.data_as(C.POINTER(C.c_double)), len(V), F.ctypes.data_as(C.POINTER(C.c_uint32)), len(F),
                                  C.byref(self.mesh)) == 0, lib.dg_last_error()
        self.field = make_field(lib, "sphere")
        n = C.c_uint64()
        assert lib.dg_grid_num_nodes(self.field.desc.resolution, C.byref(n)) == 0
        self.n_nodes = n.value
        rng = np.random.default_rng(0)
        self.x = rng.uniform(-0.5, 0.5, (N, 3))
        self.d = rng.standard_normal((N, 3))
        self.v = [np.empty(N) for _ in range(3)]
        self.v3 = [np.empty((N, 3)) for _ in range(2)]
        self.i = [np.empty(N, np.int32) for _ in range(2)]
        self.xi = rng.random((N, 3))
        self.shape = np.empty((N, 32)), np.empty((N, 96))


# query -> (forms, the argument list of a valid call with overrides a, the refused inputs: label -> overrides)
def _winding(s, a):
    return [a.get("mesh", s.mesh), a.get("x", s.x), a.get("n", N), a.get("beta", 2.0), a.get("w", s.v[0])]


def _distance(s, a):
    return [a.get("mesh", s.mesh), a.get("pts", s.x), a.get("n", N), 1, a.get("dist", s.v[0]), a.get("near", s.v3[0]), a.get("ent", s.i[0]),
            a.get("tri", s.i[1])]


def _density(s, a):
    return [a.get("field", s.field.h), a.get("h", 0.3), 1000.0, 0, a.get("b", 0), a.get("e", N), a.get("out", s.v[0])]


def _volume(s, a):
    return [a.get("field", s.field.h), a.get("h", 0.3), a.get("scale", 1.0), 0, a.get("b", 0), a.get("e", N), a.get("out", s.v[0])]


def _field_raycast(s, a):
    return [a.get("field", s.field.h), a.get("o", s.x), a.get("d", s.d), a.get("n", N), a.get("iso", 0.0), a.get("t_min", 0.0),
            a.get("t_max", INF), a.get("t_lo", s.v[0]), a.get("t_hi", s.v[1]), a.get("status", s.i[0])]


def _mesh_raycast(s, a):
    return [a.get("mesh", s.mesh), a.get("o", s.x), a.get("d", s.d), a.get("n", N), a.get("t_min", 0.0), a.get("t_max", INF),
            a.get("t", s.v[0]), a.get("id", s.i[0]), a.get("bary", s.v3[0]), a.get("status", s.i[1])]


def _shape(s, a):
    return [a.get("xi", s.xi), a.get("n", N), a.get("N", s.shape[0]), a.get("dN", s.shape[1])]


BOTH, HOST = ("host", "device"), ("host",)
QUERIES = {
    "dg_mesh_winding_number": (BOTH, _winding, {
        "NULL mesh": {"mesh": None}, "NULL points": {"x": None}, "NULL output": {"w": None},
        "beta < 1": {"beta": 0.5}, "beta NaN": {"beta": NAN}}),
    "dg_mesh_distance": (BOTH, _distance, {
        "NULL mesh": {"mesh": None}, "NULL points": {"pts": None}}),
    "dg_density_map": (BOTH, _density, {
        "NULL field": {"field": None}, "NULL output": {"out": None}, "begin > end": {"b": 3, "e": 2}, "end > nodes": {"e": PAST_END},
        "h = 0": {"h": 0.0}, "h < 0": {"h": -1.0}, "h NaN": {"h": NAN}}),
    "dg_volume_map": (BOTH, _volume, {
        "NULL field": {"field": None}, "NULL output": {"out": None}, "begin > end": {"b": 3, "e": 2}, "end > nodes": {"e": PAST_END},
        "h = 0": {"h": 0.0}, "h inf": {"h": INF}, "h NaN": {"h": NAN}, "scale inf": {"scale": INF}, "scale NaN": {"scale": NAN}}),
    "dg_field_raycast": (BOTH, _field_raycast, {
        "NULL field": {"field": None}, "NULL origins": {"o": None}, "NULL directions": {"d": None}, "NULL t_lo": {"t_lo": None},
        "NULL t_hi": {"t_hi": None}, "NULL status": {"status": None}, "iso NaN": {"iso": NAN}, "iso inf": {"iso": INF},
        "t_min NaN": {"t_min": NAN}, "t_max NaN": {"t_max": NAN}, "t_min > t_max": {"t_min": 1.0, "t_max": 0.5}}),
    "dg_mesh_raycast": (BOTH, _mesh_raycast, {
        "NULL mesh": {"mesh": None}, "NULL origins": {"o": None}, "NULL directions": {"d": None}, "NULL t": {"t": None},
        "NULL triangle_id": {"id": None}, "NULL status": {"status": None}, "t_min NaN": {"t_min": NAN}, "t_max NaN": {"t_max": NAN},
        "t_min > t_max": {"t_min": 1.0, "t_max": 0.5}}),
    "dg_shape_functions": (HOST, _shape, {"NULL xi": {"xi": None}, "NULL N": {"N": None}}),
}
# empty calls: NULL arrays are fine when there is nothing to read or write
EMPTY = {
    "dg_mesh_winding_number": {"n": 0, "x": None, "w": None},
    "dg_mesh_distance": {"n": 0, "pts": None, "dist": None, "near": None, "ent": None, "tri": None},
    "dg_density_map": {"b": 2, "e": 2, "out": None},
    "dg_volume_map": {"b": 2, "e": 2, "out": None},
    "dg_field_raycast": {"n": 0, "o": None, "d": None, "t_lo": None, "t_hi": None, "status": None},
    "dg_mesh_raycast": {"n": 0, "o": None, "d": None, "t": None, "id": None, "bary": None, "status": None},
    "dg_shape_functions": {"n": 0, "xi": None, "N": None, "dN": None},
}


def _call(lib, s, query, form, over):
    """calls the host form (typed pointers) or the device form (void pointers, stream NULL; device memory is host memory here)"""
    name = query if form == "host" else query + "_device"
    args = QUERIES[query][1](s, {k: (v(s) if callable(v) else v) for k, v in over.items()})
    conv = []
    for a in args:
        if isinstance(a, np.ndarray):
            a = a.ctypes.data if form == "device" else a.ctypes.data_as(C.POINTER(np.ctypeslib.as_ctypes_type(a.dtype)))
        conv.append(a)
    if form == "device":
        conv.append(None)
    return name, getattr(lib, name)(*conv)


@pytest.fixture(scope="module")
def handles(emu):  # noqa: F811 (emu: fixture)
    s = Handles(emu)
    yield s
    emu.dg_mesh_destroy(s.mesh)


ROWS = [(q, form, label) for q, (forms, _, cases) in QUERIES.items() for form in forms for label in cases]


@pytest.mark.parametrize("query,form", [(q, form) for q, (forms, _, _) in QUERIES.items() for form in forms])
def test_valid_and_empty_calls_succeed(emu, handles, query, form):  # noqa: F811
    for over in ({}, EMPTY[query]):
        name, rc = _call(emu, handles, query, form, over)
        assert rc == 0, (name, over, emu.dg_last_error())


@pytest.mark.parametrize("query,form,label", ROWS)
def test_refusal_code(emu, handles, query, form, label):  # noqa: F811
    name, rc = _call(emu, handles, query, form, QUERIES[query][2][label])
    assert rc == DG_ERR_INVALID, (name, label, rc, emu.dg_last_error())


@pytest.mark.parametrize("query,form,label", ROWS)
def test_refusal_names_the_called_entry_point(emu, handles, query, form, label):  # noqa: F811
    name, rc = _call(emu, handles, query, form, QUERIES[query][2][label])
    assert rc != 0
    msg = emu.dg_last_error().decode()
    assert msg.startswith(name + ":"), (name, label, msg)
