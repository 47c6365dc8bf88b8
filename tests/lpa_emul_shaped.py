"""Host build of the device LPA* core for every session kind (tests/cpp/lpa_emul_shaped.cpp) behind the LpaMixin call shapes,
with potential maps and yaw controls.  TEST INFRASTRUCTURE."""
import ctypes as C
import os
import subprocess

import numpy as np

import oracle
from oracle.lpa import LpaMixin, map_set_cells

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "cpp", "lpa_emul_shaped.cpp")
CSRC = os.path.join(HERE, "..", "mpl_ros_b200", "csrc")
DEPS = [SRC] + [os.path.join(CSRC, h) for h in ("mplb_lpa_core.h", "mplb_ref.h", "mplb_trig.cuh")]
_LIBS = {}


def lib(reverse=False):
    """reverse: the build whose lane loops run 31 .. 0 inside every phase (the result must not depend on that order)"""
    if reverse not in _LIBS:
        SO = os.path.join(HERE, "cpp", "_lpa_emul_shaped_rev.so" if reverse else "_lpa_emul_shaped.so")
        if not os.path.exists(SO) or os.path.getmtime(SO) < max(os.path.getmtime(d) for d in DEPS):
            subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-Wall", "-Wno-unknown-pragmas"] +
                                  (["-DLPA_REVERSE_LANES"] if reverse else []) + ["-o", SO + ".tmp", SRC])
            os.replace(SO + ".tmp", SO)
        L = C.CDLL(SO)
        L.emu_map_create.restype = C.c_void_p
        L.emu_map_create.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_double, C.c_void_p]
        L.emu_map_destroy.argtypes = [C.c_void_p]
        L.emu_map_free_unknown.argtypes = [C.c_void_p]
        L.emu_map_get_data.restype = C.c_int64
        L.emu_map_get_data.argtypes = [C.c_void_p, C.c_void_p, C.c_int64]
        L.emu_map_set_data.argtypes = [C.c_void_p, C.c_void_p, C.c_int64]
        L.emu_planner_create.restype = C.c_void_p
        L.emu_planner_create.argtypes = [C.c_int]
        L.emu_planner_destroy.argtypes = [C.c_void_p]
        L.emu_planner_set_map.argtypes = [C.c_void_p, C.c_void_p]
        L.emu_planner_set_param.argtypes = [C.c_void_p, C.c_char_p, C.c_double]
        L.emu_planner_set_controls.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int]
        L.emu_planner_set_potential_map.argtypes = [C.c_void_p, C.c_void_p, C.c_int64]
        L.emu_grows.argtypes = [C.c_void_p]
        L.emu_overrun.restype = C.c_char_p
        L.emu_overrun.argtypes = [C.c_void_p]
        L.emu_capacity.argtypes = [C.c_void_p, C.c_void_p]
        L.emu_lpa_cost_mismatch.argtypes = [C.c_void_p]
        _LIBS[reverse] = L
    return _LIBS[reverse]


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p)


class EmuMap:
    REV = False

    def __init__(self, origin, dim, data, res):
        self.geom = (np.ascontiguousarray(origin, dtype=np.float64), np.ascontiguousarray(dim, dtype=np.int32), float(res))
        data = np.ascontiguousarray(data, dtype=np.int8)
        self.h = lib(self.REV).emu_map_create(len(self.geom[1]), _ptr(self.geom[1]), _ptr(self.geom[0]), self.geom[2], _ptr(data))

    def free_unknown(self):
        lib(self.REV).emu_map_free_unknown(self.h)

    def set_cells(self, cells, value):
        map_set_cells(lib(self.REV), "emu_", self.h, cells, value)

    def __del__(self):
        try:
            lib(self.REV).emu_map_destroy(self.h)
        except Exception:
            pass

    def get_data(self):
        L = lib(self.REV)
        n = L.emu_map_get_data(self.h, None, 0)
        out = np.zeros(n, dtype=np.int8)
        L.emu_map_get_data(self.h, _ptr(out), n)
        return out

    def set_data(self, data):
        data = np.ascontiguousarray(data, dtype=np.int8)
        lib(self.REV).emu_map_set_data(self.h, _ptr(data), data.size)


class EmuOverrun(AssertionError):
    """the device core wrote past a capacity it was given (found by the host build's invariant check)"""


def _checked(name):
    def call(self, *a):
        out = getattr(LpaMixin, name)(self, *a)
        msg = lib(self.REV).emu_overrun(self.h).decode()
        if msg:
            raise EmuOverrun(msg)
        return out
    return call


class EmuPlanner(LpaMixin):
    """every LPA* call raises EmuOverrun as soon as the core has exceeded one of its capacities.  updatePotentialMap
    (createMask + the stamp, map_planner.cpp:286-391) is host-side preparation outside the core: the checker stamps a copy of
    the emulated map and the result becomes both the map and the potential map, as the reference does."""
    _lpa_prefix = "emu_"
    REV = False
    for _n in ("lpa_plan", "lpa_get_sub_state_space", "lpa_get_linked_nodes", "lpa_update_blocked_nodes", "lpa_update_cleared_nodes"):
        locals()[_n] = _checked(_n)
    del _n

    @classmethod
    def _lpa_lib(cls):
        return lib(cls.REV)

    def __init__(self, dim):
        self.dim = dim
        self._vec = {}
        self.h = lib(self.REV).emu_planner_create(dim)

    def __del__(self):
        try:
            lib(self.REV).emu_planner_destroy(self.h)
        except Exception:
            pass

    def set_map(self, m):
        self._map = m
        lib(self.REV).emu_planner_set_map(self.h, m.h)

    def set_param(self, key, v):
        assert lib(self.REV).emu_planner_set_param(self.h, key.encode(), float(v)) == 0, key

    def set_controls(self, U):
        U = np.ascontiguousarray(U, dtype=np.float64)
        lib(self.REV).emu_planner_set_controls(self.h, _ptr(U), U.shape[0], U.shape[1])

    def set_vec(self, key, v):
        self._vec[key] = np.array(v, dtype=np.float64)

    def update_potential_map(self, pos):
        origin, dims, res = self._map.geom
        om = oracle.OracleMap(origin, dims, self._map.get_data(), res)
        op = oracle.OraclePlanner(self.dim)
        op.set_map(om)
        for k, v in self._vec.items():
            op.set_vec(k, v)
        op.update_potential_map(np.asarray(pos, dtype=np.float64))
        dmap = np.ascontiguousarray(om.get_data(int(np.prod(dims))), dtype=np.int8)
        self._map.set_data(dmap)
        lib(self.REV).emu_planner_set_potential_map(self.h, _ptr(dmap), dmap.size)

    def cost_mismatch(self):
        """stored finite predecessor costs that differ from what get_succ gives the edge on the current maps"""
        return lib(self.REV).emu_lpa_cost_mismatch(self.h)

    def grows(self):
        return lib(self.REV).emu_grows(self.h)

    def lpa_capacity(self):
        a = np.zeros(5, dtype=np.int32)
        lib(self.REV).emu_capacity(self.h, _ptr(a))
        return dict(zip(("cap_nodes", "cap_pred", "tsize", "n_nodes_physical", "grows"), (int(x) for x in a)))


class EmuMapRev(EmuMap):
    REV = True


class EmuPlannerRev(EmuPlanner):
    REV = True
