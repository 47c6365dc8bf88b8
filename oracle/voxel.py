"""ctypes wrapper of the VoxelGrid checkers (TEST INFRASTRUCTURE ONLY, same rules as the oracle package):
  OracleVoxelGrid   oracle/voxel_oracle.cpp, the literal restatement (always available)
  RefVoxelGrid      the reference's own voxel_grid.cpp through oracle/ref_voxel_harness.cpp (where it has been built)
Both expose the C calls of the same shapes (orv_* / rvx_*), so one class drives either.  They are built beside liboracle.so and
libmplref.so (oracle/Makefile.voxel, the same compiler flags) rather than into them, so that the existing checkers and the
fixtures recorded with them stay exactly as they are."""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_ORV = os.path.join(_HERE, "libvoxel_oracle.so")
_RVX = os.path.join(_HERE, "_ref", "libvoxelref.so")
REF_UTILS = "/root/reference/planning_ros_utils"
_LIBS = {}


def _make(target):
    subprocess.check_call(["make", "-C", _HERE, "-f", "Makefile.voxel", target], stdout=subprocess.DEVNULL)


def _stale(so, srcs):
    return not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(s) for s in srcs)


def build(force=False):
    """Builds the oracle, and the reference harness where the reference tree is present."""
    if force or _stale(_ORV, [os.path.join(_HERE, "voxel_oracle.cpp")]):
        _make("libvoxel_oracle.so")
    if os.path.isdir(REF_UTILS):
        srcs = [os.path.join(_HERE, "ref_voxel_harness.cpp")]
        for root, _, files in os.walk(os.path.join(_HERE, "shim")):
            srcs += [os.path.join(root, f) for f in files]
        if force or _stale(_RVX, srcs):
            _make("_ref/libvoxelref.so")


def ref_available():
    try:
        build()
    except Exception:
        return False
    return os.path.exists(_RVX)


def _lib(prefix):
    if prefix not in _LIBS:
        build()
        L = C.CDLL(_ORV if prefix == "orv_" else _RVX)
        VP, I64 = C.c_void_p, C.c_int64
        sig = {
            "create": (VP, [VP, VP, C.c_float]), "destroy": (None, [VP]), "allocate": (C.c_int, [VP, VP, VP]),
            "info": (None, [VP, VP, VP, VP, VP]), "clear": (None, [VP]), "add_cloud": (None, [VP, VP, I64]),
            "add_cloud_inflated": (I64, [VP, VP, I64, VP, C.c_int, VP, I64]), "decay": (None, [VP]),
            "fill": (None, [VP, VP, C.c_int, C.c_int]), "clear_columns": (None, [VP, VP, C.c_int]),
            "get_cloud": (I64, [VP, VP, I64]), "get_local_cloud": (I64, [VP, VP, VP, VP, VP, I64]),
            "get_map": (I64, [VP, C.c_int, VP, I64]),
        }
        if prefix == "orv_":
            sig["map_ray_trace"] = (I64, [VP, VP, C.c_double, VP, VP, VP, I64])
        else:
            sig.update({"mu_create": (VP, [VP, VP, C.c_double, VP]), "mu_destroy": (None, [VP]),
                        "mu_ray_trace": (I64, [VP, VP, VP, VP, I64]), "node_edit": (I64, [VP, VP, C.c_int, VP, VP, VP, I64])})
        for name, (res, args) in sig.items():
            fn = getattr(L, prefix + name)
            fn.restype, fn.argtypes = res, args
        _LIBS[prefix] = L
    return _LIBS[prefix]


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _rows3(a, dtype):
    return np.ascontiguousarray(a, dtype=dtype).reshape(-1, 3)


class OracleVoxelGrid:
    _prefix = "orv_"

    def __init__(self, origin, dim, res):
        self.L = _lib(self._prefix)
        self._f = lambda name: getattr(self.L, self._prefix + name)
        o, d = np.ascontiguousarray(origin, dtype=np.float64), np.ascontiguousarray(dim, dtype=np.float64)
        self.h = self._f("create")(_p(o), _p(d), float(np.float32(res)))
        assert self.h, "geometry rejected"

    def __del__(self):
        try:
            self._f("destroy")(self.h)
        except Exception:
            pass

    def info(self):
        dim, ori = np.zeros(3, dtype=np.int32), np.zeros(3, dtype=np.int32)
        ori_d, res = np.zeros(3, dtype=np.float64), C.c_float()
        self._f("info")(self.h, _p(dim), _p(ori), _p(ori_d), C.byref(res))
        return dim, ori, ori_d, np.float32(res.value)

    def ncell(self):
        return int(np.prod(self.info()[0].astype(np.int64)))

    def allocate(self, dim, origin):
        """1 changed, 0 unchanged (-1: geometry rejected, oracle only)"""
        d, o = np.ascontiguousarray(dim, dtype=np.float64), np.ascontiguousarray(origin, dtype=np.float64)
        return self._f("allocate")(self.h, _p(d), _p(o))

    def clear(self):
        self._f("clear")(self.h)

    def add_cloud(self, pts):
        p = _rows3(pts, np.float64)
        self._f("add_cloud")(self.h, _p(p), len(p))

    def add_cloud_inflated(self, pts, ns):
        p, n3 = _rows3(pts, np.float64), _rows3(ns, np.int32)
        cap = len(p) * len(n3)
        out = np.zeros((max(cap, 1), 3), dtype=np.int32)
        k = self._f("add_cloud_inflated")(self.h, _p(p), len(p), _p(n3), len(n3), _p(out), cap)
        return out[:k].copy()

    def decay(self):
        self._f("decay")(self.h)

    def fill(self, cells, column):
        c = _rows3(cells, np.int32)
        self._f("fill")(self.h, _p(c), len(c), int(bool(column)))

    def clear_columns(self, cells):
        c = _rows3(cells, np.int32)
        self._f("clear_columns")(self.h, _p(c), len(c))

    def _cloud(self, fn, *args):
        n = fn(self.h, *args, None, 0)
        out = np.zeros((max(n, 1), 3), dtype=np.float64)
        fn(self.h, *args, _p(out), n)
        return out[:n]

    def get_cloud(self):
        return self._cloud(self._f("get_cloud"))

    def get_local_cloud(self, pos, ori, dim):
        a = [np.ascontiguousarray(v, dtype=np.float64) for v in (pos, ori, dim)]
        return self._cloud(self._f("get_local_cloud"), *[_p(v) for v in a])

    def get_map(self, inflated=False):
        n = self.ncell()
        out = np.zeros(max(n, 1), dtype=np.int8)
        assert self._f("get_map")(self.h, int(bool(inflated)), _p(out), out.size) == n
        return out[:n]


class RefVoxelGrid(OracleVoxelGrid):
    """The reference's VoxelGrid; info() reports origin_ as INT32_MIN (the class does not expose it)."""
    _prefix = "rvx_"


def _rows(fn, *args):
    n = fn(*args, None, 0)
    out = np.zeros((max(n, 1), 3), dtype=np.int32)
    fn(*args, _p(out), n)
    return out[:n]


def ray_trace(origin, dim, res, p1, p2):
    """MapUtil::rayTrace (map_util.h:117-134) restated by the oracle"""
    a = [np.ascontiguousarray(v, dtype=np.float64) for v in (origin, p1, p2)]
    d = np.ascontiguousarray(dim, dtype=np.int32)
    return _rows(_lib("orv_").orv_map_ray_trace, _p(a[0]), _p(d), float(res), _p(a[1]), _p(a[2]))


class RefMapUtil:
    """the reference's own MPL::VoxelMapUtil (map_util.h), as map_replanner_node.cpp keeps it beside its VoxelGrid"""

    def __init__(self, origin, dim, res, data):
        self.L = _lib("rvx_")
        o, d = np.ascontiguousarray(origin, dtype=np.float64), np.ascontiguousarray(dim, dtype=np.int32)
        data = np.ascontiguousarray(data, dtype=np.int8)
        self.h = self.L.rvx_mu_create(_p(o), _p(d), float(res), _p(data))

    def __del__(self):
        try:
            self.L.rvx_mu_destroy(self.h)
        except Exception:
            pass

    def ray_trace(self, p1, p2):
        a, b = np.ascontiguousarray(p1, dtype=np.float64), np.ascontiguousarray(p2, dtype=np.float64)
        return _rows(self.L.rvx_mu_ray_trace, self.h, _p(a), _p(b))

    def node_edit(self, grid, add, p1, p2):
        """addCloudCallback (add) / clearCloudCallback of map_replanner_node.cpp:175-232 on RefVoxelGrid `grid` and this
        MapUtil, up to the planner call; returns new_obs / new_clear"""
        a, b = np.ascontiguousarray(p1, dtype=np.float64), np.ascontiguousarray(p2, dtype=np.float64)
        out = np.zeros((1 << 16, 3), dtype=np.int32)  # one call: the edit happens once
        n = self.L.rvx_node_edit(grid.h, self.h, int(bool(add)), _p(a), _p(b), _p(out), len(out))
        assert n <= len(out)
        return out[:n].copy()
