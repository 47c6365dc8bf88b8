"""Host build of the device LPA* core (tests/cpp/lpa_emul.cpp) behind the LpaMixin call shapes.  TEST INFRASTRUCTURE."""
import ctypes as C
import os
import subprocess

import numpy as np

from oracle.lpa import LpaMixin, map_set_cells

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "cpp", "lpa_emul.cpp")
CSRC = os.path.join(HERE, "..", "mpl_ros_b200", "csrc")
DEPS = [SRC, os.path.join(CSRC, "mplb_lpa_core.h"), os.path.join(CSRC, "mplb_ref.h")]
_LIBS = {}


def lib(reverse=False):
    """reverse: the build whose lane loops run 31 .. 0 inside every phase (the result must not depend on that order)"""
    if reverse not in _LIBS:
        SO = os.path.join(HERE, "cpp", "_lpa_emul_rev.so" if reverse else "_lpa_emul.so")
        if not os.path.exists(SO) or os.path.getmtime(SO) < max(os.path.getmtime(d) for d in DEPS):
            subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-Wall"] +
                                  (["-DLPA_REVERSE_LANES"] if reverse else []) + ["-o", SO + ".tmp", SRC])
            os.replace(SO + ".tmp", SO)
        L = C.CDLL(SO)
        L.emu_map_create.restype = C.c_void_p
        L.emu_map_create.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_double, C.c_void_p]
        L.emu_map_destroy.argtypes = [C.c_void_p]
        L.emu_map_free_unknown.argtypes = [C.c_void_p]
        L.emu_planner_create.restype = C.c_void_p
        L.emu_planner_create.argtypes = [C.c_int]
        L.emu_planner_destroy.argtypes = [C.c_void_p]
        L.emu_planner_set_map.argtypes = [C.c_void_p, C.c_void_p]
        L.emu_planner_set_param.argtypes = [C.c_void_p, C.c_char_p, C.c_double]
        L.emu_planner_set_controls.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int]
        L.emu_grows.argtypes = [C.c_void_p]
        _LIBS[reverse] = L
    return _LIBS[reverse]


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p)


class EmuMap:
    REV = False

    def __init__(self, origin, dim, data, res):
        origin = np.ascontiguousarray(origin, dtype=np.float64)
        dim = np.ascontiguousarray(dim, dtype=np.int32)
        data = np.ascontiguousarray(data, dtype=np.int8)
        self.h = lib(self.REV).emu_map_create(len(dim), _ptr(dim), _ptr(origin), float(res), _ptr(data))

    def free_unknown(self):
        lib(self.REV).emu_map_free_unknown(self.h)

    def set_cells(self, cells, value):
        map_set_cells(lib(self.REV), "emu_", self.h, cells, value)


class EmuPlanner(LpaMixin):
    _lpa_prefix = "emu_"
    REV = False

    @classmethod
    def _lpa_lib(cls):
        return lib(cls.REV)

    def __init__(self, dim):
        self.dim = dim
        self.h = lib(self.REV).emu_planner_create(dim)

    def set_map(self, m):
        self._map = m
        lib(self.REV).emu_planner_set_map(self.h, m.h)

    def set_param(self, key, v):
        assert lib(self.REV).emu_planner_set_param(self.h, key.encode(), float(v)) == 0, key

    def set_controls(self, U):
        U = np.ascontiguousarray(U, dtype=np.float64)
        lib(self.REV).emu_planner_set_controls(self.h, _ptr(U), U.shape[0], U.shape[1])

    def grows(self):
        return lib(self.REV).emu_grows(self.h)


class EmuMapRev(EmuMap):
    REV = True


class EmuPlannerRev(EmuPlanner):
    REV = True
