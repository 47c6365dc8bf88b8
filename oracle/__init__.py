"""ctypes wrapper of the CPU oracle (oracle/mpl_oracle.cpp).  TEST INFRASTRUCTURE ONLY.

Only tests/, __graft_entry__.smoke() and bench.py (cpu_baseline / --impl reference) may import this
package; nothing under mpl_ros_b200/ does.  See oracle/mpl_oracle.h for the parity pin statement.
"""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None

WAYPOINT_DTYPE = np.dtype([("pos", "f8", 3), ("vel", "f8", 3), ("acc", "f8", 3), ("jrk", "f8", 3),
                           ("yaw", "f8"), ("t", "f8"), ("control", "i4"), ("enable_t", "i4")], align=True)
RESULT_DTYPE = np.dtype([("status", "i4"), ("n_seg", "i4"), ("cost", "f8"), ("pops", "i4"), ("n_nodes", "i4"),
                         ("n_open", "i4"), ("n_closed", "i4"), ("n_prims", "i8"), ("n_samples", "i8"),
                         ("n_valid", "i8"), ("pop_hash", "u8"), ("closed_hash", "u8"), ("device_ms", "f8")], align=True)
TRACE_DTYPE = np.dtype([("verdict", "i4"), ("n", "i4"), ("n_tested", "i4"), ("block_idx", "i4"), ("cost", "f8"),
                        ("succ", "f8", 13), ("key", "i4", 16)], align=True)
NODE_DTYPE = np.dtype([("state", "f8", 13), ("t", "f8"), ("g", "f8"), ("h", "f8"), ("key", "i4", 16),
                       ("opened", "i4"), ("closed", "i4")], align=True)
HEAP_DTYPE = np.dtype([("key", "i4", 16), ("f", "f8"), ("key_hash", "u8")], align=True)


def build(force=False):
    so = os.path.join(_HERE, "liboracle.so")
    srcs = [os.path.join(_HERE, f) for f in ("mpl_oracle.cpp", "poly_oracle.cpp", "mpl_oracle.h")]
    if force or not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(s) for s in srcs):
        subprocess.check_call(["make", "-C", _HERE, "liboracle.so"], stdout=subprocess.DEVNULL)
    return so


def lib():
    global _LIB
    if _LIB is None:
        L = C.CDLL(build())
        L.orc_map_create.restype = C.c_void_p
        L.orc_map_create.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_double, C.c_void_p]
        L.orc_map_destroy.argtypes = [C.c_void_p]
        L.orc_map_free_unknown.argtypes = [C.c_void_p]
        L.orc_map_float_to_int.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        L.orc_planner_create.restype = C.c_void_p
        L.orc_planner_create.argtypes = [C.c_int]
        L.orc_planner_destroy.argtypes = [C.c_void_p]
        L.orc_planner_set_map.argtypes = [C.c_void_p, C.c_void_p]
        L.orc_planner_set_param.argtypes = [C.c_void_p, C.c_char_p, C.c_double]
        L.orc_planner_set_controls.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int]
        L.orc_planner_set_vec.argtypes = [C.c_void_p, C.c_char_p, C.c_void_p]
        L.orc_planner_set_search_region.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int]
        L.orc_planner_clear_shaping.argtypes = [C.c_void_p]
        L.orc_planner_set_prior_trajectory.argtypes = [C.c_void_p, C.c_void_p]
        L.orc_planner_set_potential_map.argtypes = [C.c_void_p, C.c_void_p, C.c_int64]
        L.orc_planner_set_search_region_mask.argtypes = [C.c_void_p, C.c_void_p, C.c_int64]
        L.orc_planner_get_search_region.restype = C.c_int64
        L.orc_planner_get_search_region.argtypes = [C.c_void_p, C.c_void_p, C.c_int64]
        L.orc_planner_update_potential_map.argtypes = [C.c_void_p, C.c_void_p]
        L.orc_map_get_data.restype = C.c_int64
        L.orc_map_get_data.argtypes = [C.c_void_p, C.c_void_p, C.c_int64]
        L.orc_plan.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        L.orc_get_actions.argtypes = [C.c_void_p, C.c_void_p, C.c_int]
        L.orc_get_seg_states.argtypes = [C.c_void_p, C.c_void_p, C.c_int]
        L.orc_get_nodes.argtypes = [C.c_void_p, C.c_void_p, C.c_int]
        L.orc_get_pop_keys.argtypes = [C.c_void_p, C.c_void_p, C.c_int]
        L.orc_get_heap.argtypes = [C.c_void_p, C.c_void_p, C.c_int]
        L.orc_get_peaks.argtypes = [C.c_void_p, C.c_void_p]
        L.orc_get_peaks.restype = None
        L.orc_get_succ_trace.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int]
        L.orc_plan_batch.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int]
        L.orc_plan_batch_dyn.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int,
                                         C.c_void_p, C.c_int, C.c_void_p]
        _LIB = L
    return _LIB


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p)


def make_waypoints(n=1):
    return np.zeros(n, dtype=WAYPOINT_DTYPE)


from .lpa import LpaMixin, map_set_cells as _map_set_cells  # noqa: E402


class OracleMap:
    def set_cells(self, cells, value):
        """the caller's getMap / edit / setMap (map_replanner_node.cpp:181-196)"""
        _map_set_cells(lib(), "orc_", self.h, cells, value)

    def __init__(self, origin, dim, data, res):
        origin = np.ascontiguousarray(origin, dtype=np.float64)
        dim = np.ascontiguousarray(dim, dtype=np.int32)
        data = np.ascontiguousarray(data, dtype=np.int8)
        assert data.size == int(np.prod(dim))
        self.ndim = len(dim)
        self.h = lib().orc_map_create(self.ndim, _ptr(dim), _ptr(origin), float(res), _ptr(data))

    def free_unknown(self):
        lib().orc_map_free_unknown(self.h)

    def get_data(self, n):
        out = np.zeros(n, dtype=np.int8)
        lib().orc_map_get_data(self.h, _ptr(out), n)
        return out

    def float_to_int(self, pt):
        pt = np.ascontiguousarray(pt, dtype=np.float64)
        pn = np.zeros(3, dtype=np.int32)
        idx = lib().orc_map_float_to_int(self.h, _ptr(pt), _ptr(pn))
        return pn[:self.ndim].copy(), idx

    def __del__(self):
        try:
            lib().orc_map_destroy(self.h)
        except Exception:
            pass


class OraclePlanner(LpaMixin):
    """Mirrors the reference setters (planner_base.h:179-265) over the oracle."""
    _lpa_prefix = "orc_"

    @staticmethod
    def _lpa_lib():
        return lib()

    def lpa_last_fault(self):
        return lib().orc_lpa_last_fault(self.h)

    def lpa_actions(self):
        L = lib()
        L.orc_lpa_get_actions.argtypes = [C.c_void_p, C.c_void_p, C.c_int]
        n = L.orc_lpa_get_actions(self.h, None, 0)
        a = np.zeros(max(n, 1), dtype=np.int32)
        n = L.orc_lpa_get_actions(self.h, _ptr(a), a.size)
        return a[:n]

    def __init__(self, dim):
        self.dim = dim
        self.h = lib().orc_planner_create(dim)
        self._map = None
        self.nU = 0

    def __del__(self):
        try:
            lib().orc_planner_destroy(self.h)
        except Exception:
            pass

    def set_map(self, m):
        self._map = m
        lib().orc_planner_set_map(self.h, m.h)

    def set_param(self, key, v):
        assert lib().orc_planner_set_param(self.h, key.encode(), float(v)) == 0, key

    def set_controls(self, U):
        U = np.ascontiguousarray(U, dtype=np.float64)
        self.nU = U.shape[0]
        lib().orc_planner_set_controls(self.h, _ptr(U), U.shape[0], U.shape[1])

    # ---- cost shaping (MapPlanner members, map_planner.h:27-49)
    def set_vec(self, key, v):
        v = np.ascontiguousarray(v, dtype=np.float64)
        lib().orc_planner_set_vec(self.h, key.encode(), _ptr(v))

    def set_search_region(self, path, dense=False):
        path = np.ascontiguousarray(path, dtype=np.float64)
        lib().orc_planner_set_search_region(self.h, _ptr(path), path.shape[0], int(dense))

    def get_search_region(self, ncell):
        out = np.zeros(ncell, dtype=np.uint8)
        n = lib().orc_planner_get_search_region(self.h, _ptr(out), ncell)
        return out[:n]

    def update_potential_map(self, pos):
        pos = np.ascontiguousarray(pos, dtype=np.float64)
        lib().orc_planner_update_potential_map(self.h, _ptr(pos))

    def set_potential_map(self, pot):
        if pot is None:
            lib().orc_planner_set_potential_map(self.h, None, 0)
            return
        pot = np.ascontiguousarray(pot, dtype=np.int8).ravel()
        lib().orc_planner_set_potential_map(self.h, _ptr(pot), pot.size)

    def set_search_region_mask(self, mask):
        if mask is None:
            lib().orc_planner_set_search_region_mask(self.h, None, 0)
            return
        mask = np.ascontiguousarray(mask, dtype=np.uint8).ravel()
        lib().orc_planner_set_search_region_mask(self.h, _ptr(mask), mask.size)

    def set_prior_trajectory(self, src):
        lib().orc_planner_set_prior_trajectory(self.h, src.h if src is not None else None)

    def clear_shaping(self):
        lib().orc_planner_clear_shaping(self.h)

    def plan(self, start, goal):
        res = np.zeros(1, dtype=RESULT_DTYPE)
        lib().orc_plan(self.h, _ptr(start), _ptr(goal), _ptr(res))
        return res[0]

    def actions(self, n_seg):
        a = np.zeros(max(n_seg, 1), dtype=np.int32)
        n = lib().orc_get_actions(self.h, _ptr(a), a.size)
        return a[:n]

    def seg_states(self, n_seg):
        s = np.zeros((max(n_seg, 1), 13), dtype=np.float64)
        n = lib().orc_get_seg_states(self.h, _ptr(s), s.shape[0])
        return s[:n]

    def nodes(self, n_nodes):
        a = np.zeros(max(n_nodes, 1), dtype=NODE_DTYPE)
        n = lib().orc_get_nodes(self.h, _ptr(a), a.size)
        return a[:n]

    def pop_keys(self, pops):
        a = np.zeros((max(pops, 1), 16), dtype=np.int32)
        n = lib().orc_get_pop_keys(self.h, _ptr(a), a.shape[0])
        return a[:n]

    def heap(self):
        """pq_ of the last plan in its array order (HEAP_DTYPE: key rows, f, key hash)"""
        n = lib().orc_get_heap(self.h, None, 0)
        a = np.zeros(max(n, 1), dtype=HEAP_DTYPE)
        n = lib().orc_get_heap(self.h, _ptr(a), a.size)
        return a[:n]

    def peaks(self):
        """largest (nodes, heap, predecessor records) at the start of any expansion of the last plan (orc_get_peaks)"""
        a = np.zeros(3, dtype=np.int64)
        lib().orc_get_peaks(self.h, _ptr(a))
        return dict(nodes=int(a[0]), heap=int(a[1]), records=int(a[2]))

    def succ_trace(self, curr):
        rows = np.zeros(self.nU, dtype=TRACE_DTYPE)
        lib().orc_get_succ_trace(self.h, _ptr(curr), _ptr(rows), rows.size)
        return rows

    def plan_batch(self, starts, goals, nthreads=1, max_seg=0, order=None, pin=False, want_busy=False):
        """Threads pull plans from an atomic queue (in `order` when given); results do not depend on the schedule."""
        n = len(starts)
        res = np.zeros(n, dtype=RESULT_DTYPE)
        acts = np.full((n, max_seg), -1, dtype=np.int32) if max_seg > 0 else None
        order = None if order is None else np.ascontiguousarray(order, dtype=np.int32)
        busy = np.zeros(max(nthreads, 1), dtype=np.float64)
        lib().orc_plan_batch_dyn(self.h, _ptr(starts), _ptr(goals), n, nthreads, _ptr(res),
                                 _ptr(acts) if acts is not None else None, max_seg,
                                 _ptr(order) if order is not None else None, int(bool(pin)), _ptr(busy))
        return (res, acts, busy) if want_busy else (res, acts)


def traj_solve(dim, control, wps, dts, yaw_control=1):
    """TrajSolver<dim>(control, yaw_control): setWaypoints(wps), setDts(dts), solve() (oracle/poly_oracle.cpp).
    Returns (n_seg, dim + 1, 6) Primitive coefficient rows (axes, then yaw; highest order first)."""
    L = lib()
    L.orc_traj_solve.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    wps = np.ascontiguousarray(wps, dtype=WAYPOINT_DTYPE)
    dts = np.ascontiguousarray(dts, dtype=np.float64)
    out = np.zeros((max(len(wps) - 1, 1), dim + 1, 6), dtype=np.float64)
    n = L.orc_traj_solve(dim, int(control), int(yaw_control), len(wps), _ptr(wps), _ptr(dts), _ptr(out))
    return out[:n]


def traj_allocate_time(dim, pts, v):
    """TrajSolver::allocate_time (traj_solver.h:122-131)."""
    L = lib()
    L.orc_traj_allocate_time.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_double, C.c_void_p]
    p3 = np.zeros((len(pts), 3), dtype=np.float64)
    p3[:, :dim] = np.asarray(pts, dtype=np.float64)[:, :dim]
    dts = np.zeros(max(len(pts) - 1, 1), dtype=np.float64)
    n = L.orc_traj_allocate_time(dim, len(pts), _ptr(p3), float(v), _ptr(dts))
    return dts[:n]
