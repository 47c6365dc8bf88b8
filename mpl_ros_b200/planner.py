"""Python mirror of the reference's operator surface for the hot path, over the C ABI (include/mplb.h).

Class and method names follow the reference so that tests read like MPL/test/test_planner_2d.cpp and
mpl_test_node/src/map_planner_node.cpp:
  MapUtil        motion_primitive_library/include/mpl_collision/map_util.h:20-314
  Waypoint       include/mpl_basis/waypoint.h:22-58
  Primitive      include/mpl_basis/primitive.h:205-431   (coefficient rows only; built from (parent, U[a], dt))
  Trajectory     include/mpl_basis/trajectory.h:42-57,250-292
  MapPlanner     include/mpl_planner/planner/map_planner.h:20-125 over PlannerBase (common/planner_base.h)
Everything numerical happens in libmplb.so on the GPU; this file only marshals buffers.
"""
import ctypes as C

import numpy as np

from . import _lib
from ._lib import MplbError, PARAM, check, lib, ptr  # noqa: F401
from .maps import ACC, JRK, SNP, VEL  # noqa: F401

VELxYAW, ACCxYAW, JRKxYAW, SNPxYAW = VEL | 16, ACC | 16, JRK | 16, SNP | 16  # control.h:15-18

PLAN_OK, PLAN_START_NOT_FREE, PLAN_MAX_EXPAND, PLAN_QUEUE_EMPTY, PLAN_TRACEBACK_FAILED, PLAN_START_IS_GOAL = range(6)


class Waypoint:
    """waypoint.h:22-58.  `control` is the 5-bit union of use_pos..use_yaw (control.h:10-20)."""

    def __init__(self, dim, control=0):
        self.dim = dim
        self.pos = np.zeros(dim)
        self.vel = np.zeros(dim)
        self.acc = np.zeros(dim)
        self.jrk = np.zeros(dim)
        self.yaw = 0.0
        self.t = 0.0
        self.control = control
        self.enable_t = False

    def _flag(bit):  # noqa: N805
        def get(self):
            return bool(self.control & bit)

        def set_(self, v):
            self.control = (self.control | bit) if v else (self.control & ~bit)
        return property(get, set_)

    use_pos, use_vel, use_acc, use_jrk, use_yaw = _flag(1), _flag(2), _flag(4), _flag(8), _flag(16)

    def to_record(self, rec):
        d = self.dim
        rec["pos"][:d], rec["vel"][:d], rec["acc"][:d], rec["jrk"][:d] = self.pos, self.vel, self.acc, self.jrk
        rec["yaw"], rec["t"], rec["control"], rec["enable_t"] = self.yaw, self.t, self.control, int(self.enable_t)
        return rec


def waypoints_array(n):
    return np.zeros(n, dtype=_lib.WAYPOINT_DTYPE)


class Primitive:
    """primitive.h:205-256: per-axis coefficient rows, highest order first, from (parent state, u, dt)."""

    def __init__(self, dim, control, state13, u, t):
        self.dim, self.control, self.t_ = dim, control, float(t)
        order = {VEL: 1, ACC: 2, JRK: 3, SNP: 4}[control & 15]
        self.coeffs = np.zeros((dim, 6))
        # pr_yaw_ = Primitive1D(p.yaw, u(Dim)) for the *xYAW controls (primitive.h:236-253)
        self.yaw_coeff = np.array([0, 0, 0, 0, u[dim], state13[12]], dtype=np.float64) if control & 16 else None
        for k in range(dim):
            p, v, a, j = state13[k], state13[3 + k], state13[6 + k], state13[9 + k]
            row = {1: (0, 0, 0, 0, u[k], p), 2: (0, 0, 0, u[k], v, p), 3: (0, 0, u[k], a, v, p),
                   4: (0, u[k], j, a, v, p)}[order]
            self.coeffs[k] = row

    @classmethod
    def from_coeffs(cls, dim, coeffs, yaw_coeff, t, control):
        """Primitive(cs, t, control), primitive.h:309-313: coefficient rows given directly (TrajSolver output)."""
        pr = cls.__new__(cls)
        pr.dim, pr.control, pr.t_ = dim, control, float(t)
        pr.coeffs = np.array(coeffs, dtype=np.float64).reshape(dim, 6)
        pr.yaw_coeff = None if yaw_coeff is None else np.array(yaw_coeff, dtype=np.float64)
        return pr

    def t(self):
        return self.t_

    def evaluate(self, t):
        """pos/vel/acc/jrk at t (primitive.h:128-145,321-331), float64 numpy (host convenience only)."""
        out = Waypoint(self.dim, self.control)
        for k in range(self.dim):
            c = self.coeffs[k]
            out.pos[k] = c[0] / 120 * t ** 5 + c[1] / 24 * t ** 4 + c[2] / 6 * t ** 3 + c[3] / 2 * t * t + c[4] * t + c[5]
            out.vel[k] = c[0] / 24 * t ** 4 + c[1] / 6 * t ** 3 + c[2] / 2 * t * t + c[3] * t + c[4]
            out.acc[k] = c[0] / 6 * t ** 3 + c[1] / 2 * t * t + c[2] * t + c[3]
            out.jrk[k] = c[0] / 2 * t * t + c[1] * t + c[2]
        if self.yaw_coeff is not None:  # primitive.h:328 + math.h:15-19
            yaw = self.yaw_coeff[4] * t + self.yaw_coeff[5]
            while yaw > np.pi:
                yaw -= 2.0 * np.pi
            while yaw < -np.pi:
                yaw += 2.0 * np.pi
            out.yaw = yaw
        return out


class Trajectory:
    """trajectory.h:42-57: piecewise primitives with cumulative taus."""

    def __init__(self, segs=()):
        self.segs = list(segs)
        self.taus = [0.0]
        for pr in self.segs:
            self.taus.append(pr.t() + self.taus[-1])
        self.total_t_ = self.taus[-1]

    def getTotalTime(self):
        return self.total_t_

    def getPrimitives(self):
        return self.segs

    def getWaypoints(self):  # trajectory.h:277-289
        ws = []
        if not self.segs:
            return ws
        t = 0.0
        for seg in self.segs:
            w = seg.evaluate(0.0)
            w.t = t
            ws.append(w)
            t += seg.t()
        w = self.segs[-1].evaluate(self.segs[-1].t())
        w.t = t
        ws.append(w)
        return ws


class MapUtil:
    """map_util.h:20-314 — the grid lives on the GPU (int8 cells + occupancy bit-bricks)."""

    def __init__(self, dim):
        self.dim = dim
        self._h = None

    def setMap(self, ori, dim, map_, res):  # map_util.h:84-90
        self._destroy()
        ori = np.ascontiguousarray(ori, dtype=np.float64)
        nd = np.ascontiguousarray(dim, dtype=np.int32)
        data = np.ascontiguousarray(map_, dtype=np.int8).reshape(-1)
        if data.size != int(np.prod(nd.astype(np.int64))):
            raise MplbError("map data size does not match dim")
        h = C.c_void_p()
        check(lib().mplb_map_create(self.dim, ptr(nd), ptr(ori), float(res), ptr(data), C.byref(h)))
        self._h = h

    def setMapFromDevice(self, ori, dim, dev_ptr, res, stream=None):
        """Adopt a grid that already sits in device memory (e.g. after an NCCL broadcast)."""
        self._destroy()
        ori = np.ascontiguousarray(ori, dtype=np.float64)
        nd = np.ascontiguousarray(dim, dtype=np.int32)
        h = C.c_void_p()
        check(lib().mplb_map_create_from_device(self.dim, ptr(nd), ptr(ori), float(res), C.c_void_p(int(dev_ptr)),
                                                C.c_void_p(int(stream) if stream else None), C.byref(h)))
        self._h = h

    def setCells(self, cells, value):
        """The caller-side map edit of map_replanner_node.cpp:181-196,221-229 (getMap, write cells, setMap) done in place on
        the device grid: `cells` rows of Dim ints receive `value` (100 occupied, 0 free)."""
        c = np.asarray(cells, dtype=np.int32).reshape(len(cells), -1)
        c3 = np.zeros((len(c), 3), dtype=np.int32)
        c3[:, :c.shape[1]] = c
        check(lib().mplb_map_set_cells(self._h, ptr(c3), len(c3), int(value)))

    def getCells(self, cells):
        """Values of cells (rows of Dim ints) as int32, INT32_MIN outside: the material of isFree / isOccupied
        (map_util.h:44-80)."""
        c = np.asarray(cells, dtype=np.int32).reshape(len(cells), -1)
        c3 = np.zeros((len(c), 3), dtype=np.int32)
        c3[:, :c.shape[1]] = c
        out = np.zeros(max(len(c3), 1), dtype=np.int32)
        check(lib().mplb_map_get_cells(self._h, ptr(c3), len(c3), ptr(out)))
        return out[:len(c3)]

    def freeUnknown(self):  # map_util.h:259-276
        check(lib().mplb_map_free_unknown(self._h))

    def dilate(self, ns):  # map_util.h:221-257
        ns = np.ascontiguousarray(ns, dtype=np.int32).reshape(-1, self.dim)
        check(lib().mplb_map_dilate(self._h, ptr(ns), ns.shape[0]))

    def _info_raw(self):
        d = C.c_int32()
        nd = np.zeros(3, dtype=np.int32)
        ori = np.zeros(3, dtype=np.float64)
        res = C.c_double()
        check(lib().mplb_map_get_info(self._h, C.byref(d), ptr(nd), ptr(ori), C.byref(res)))
        return nd[:d.value].copy(), ori[:d.value].copy(), res.value

    def _info(self):
        d = C.c_int32()
        nd = np.zeros(3, dtype=np.int32)
        ori = np.zeros(3, dtype=np.float64)
        res = C.c_double()
        check(lib().mplb_map_get_info(self._h, C.byref(d), ptr(nd), ptr(ori), C.byref(res)))
        return nd[:self.dim].copy(), ori[:self.dim].copy(), res.value

    def getRes(self):
        return self._info()[2]

    def getDim(self):
        return self._info()[0]

    def getOrigin(self):
        return self._info()[1]

    def getCloud(self):  # map_util.h:137-161: centres of the occupied cells
        nd = self.getDim()
        grid = self.getMap().reshape(tuple(int(x) for x in nd[::-1]))
        idx = np.argwhere(grid == 100)[:, ::-1]  # (x, y[, z])
        idx = idx[np.lexsort(idx[:, ::-1].T)]    # the reference walks x outermost
        return (idx + 0.5) * self.getRes() + self.getOrigin()

    def getMap(self):  # map_util.h:25
        nd = self.getDim()
        out = np.zeros(int(np.prod(nd.astype(np.int64))), dtype=np.int8)
        check(lib().mplb_map_get_data(self._h, ptr(out), out.size))
        return out

    def _destroy(self):
        if self._h is not None:
            lib().mplb_map_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self._destroy()
        except Exception:
            pass


class OccMapUtil(MapUtil):
    def __init__(self):
        super().__init__(2)


class VoxelMapUtil(MapUtil):
    def __init__(self):
        super().__init__(3)


class MapPlanner:
    """MapPlanner<Dim> (map_planner.h:20-125) / PlannerBase<Dim, Waypoint<Dim>> (planner_base.h:18-345)."""

    def __init__(self, dim, verbose=False):
        self.dim = dim
        h = C.c_void_p()
        check(lib().mplb_planner_create(dim, int(verbose), C.byref(h)))
        self._h = h
        self.map_util_ = None
        self.U_ = None
        self.dt_ = 1.0
        self._last = None
        self._control = None
        self.traj_cost_ = None
        self.traj_ = Trajectory()
        self._initialized = False
        # map_planner.h:104-113
        self.search_radius_ = np.zeros(3)
        self.potential_radius_ = np.zeros(3)
        self.potential_map_range_ = np.zeros(3)
        self.pow_ = 1.0

    def __del__(self):
        try:
            lib().mplb_planner_destroy(self._h)
        except Exception:
            pass

    # ---- setters (planner_base.h:170-265, map_planner.cpp:14-18)
    def setMapUtil(self, map_util):
        check(lib().mplb_planner_set_map(self._h, map_util._h))
        self.map_util_ = map_util

    def _set(self, key, v):
        check(lib().mplb_planner_set_param(self._h, PARAM[key], float(v)))

    def setVmax(self, v): self._set("v_max", v)
    def setAmax(self, a): self._set("a_max", a)
    def setJmax(self, j): self._set("j_max", j)
    def setYawmax(self, y): self._set("yaw_max", y)
    def setWyaw(self, w): self._set("wyaw", w)  # planner_base.h:221
    def setTmax(self, t): self._set("t_max", t)
    def setW(self, w): self._set("w", w)
    def setEpsilon(self, e): self._set("epsilon", e)
    def setMaxNum(self, n): self._set("max_num", n)

    def setHeurIgnoreDynamics(self, ignore):  # planner_base.h:233 — only the default (True) is on this path
        if not ignore:
            raise MplbError("heur_ignore_dynamics = false needs the reference's polynomial root finder (env_base.h:67-211); "
                            "not part of this path")
    def setPriorTrajectory(self, traj):  # planner_base.h:249-252 (None or an empty trajectory clears)
        segs = traj.getPrimitives() if traj is not None else []
        n = len(segs)
        if n == 0:
            check(lib().mplb_planner_set_prior_trajectory(self._h, 0, None, None, 0))
            return
        cs = np.zeros((n, 4, 6))
        ts = np.zeros(n)
        for i, pr in enumerate(segs):
            cs[i, :self.dim] = pr.coeffs
            if pr.yaw_coeff is not None:
                cs[i, 3] = pr.yaw_coeff
            ts[i] = pr.t()
        check(lib().mplb_planner_set_prior_trajectory(self._h, n, ptr(cs), ptr(ts), int(segs[-1].control)))

    def setExactPreds(self, mode):  # MPLB_EXACT_PREDS: -1 auto, 0 never, 1 always (predecessor lists of graph_search.h:100-102)
        self._set("exact_preds", mode)

    def setMemFraction(self, f): self._set("mem_fraction", f)
    def setMaxSlots(self, n): self._set("max_slots", n)
    def setArenaBytes(self, n): self._set("arena_bytes", n)  # upper bound on the arena budget; 0 = unset
    def setLPAInitNodes(self, n): self._set("lpa_init_nodes", n)  # LPA* node capacity at allocation (default 65 536)
    def setLPAInitPreds(self, n): self._set("lpa_init_preds", n)  # LPA* predecessor records at allocation (default 2^20)

    def setDt(self, dt):
        self._set("dt", dt)
        self.dt_ = float(dt)

    def setTol(self, tol_pos, tol_vel=-1, tol_acc=-1):  # planner_base.h:255-265
        self._set("tol_pos", tol_pos)
        self._set("tol_vel", tol_vel)
        self._set("tol_acc", tol_acc)

    def setU(self, U):  # planner_base.h:246
        U = np.ascontiguousarray(U, dtype=np.float64)
        check(lib().mplb_planner_set_controls(self._h, ptr(U), U.shape[0], U.shape[1]))
        self.U_ = U

    def initialized(self):
        return self._initialized

    # ---- cost shaping (map_planner.h:27-54,77-87; SURVEY section 8f.1)
    def _vec3(self, v):
        out = np.zeros(3)
        v = np.asarray(v, dtype=np.float64).ravel()
        out[:len(v)] = v
        return out

    def setSearchRadius(self, radius):  # map_planner.cpp:41-43
        self.search_radius_ = self._vec3(radius)

    def setPotentialRadius(self, radius):  # map_planner.cpp:20-23
        self.potential_radius_ = self._vec3(radius)

    def setPotentialMapRange(self, rng):  # map_planner.cpp:25-28
        self.potential_map_range_ = self._vec3(rng)

    def setPotentialWeight(self, w): self._set("potential_weight", w)  # map_planner.cpp:30-33
    def setGradientWeight(self, w): self._set("gradient_weight", w)    # map_planner.cpp:35-38

    def setSearchRegion(self, path, dense=False):  # map_planner.cpp:46-95
        pts = np.zeros((len(path), 3))
        for i, q in enumerate(path):
            q = np.asarray(q, dtype=np.float64).ravel()
            pts[i, :len(q)] = q
        check(lib().mplb_planner_set_search_region_path(self._h, ptr(pts), len(pts), int(bool(dense)),
                                                        ptr(self.search_radius_)))

    def setSearchRegionMask(self, in_region):  # env_base::set_search_region, env_base.h:301-303 (None clears)
        if in_region is None:
            check(lib().mplb_planner_set_search_region(self._h, None, 0))
            return
        m = np.ascontiguousarray(in_region, dtype=np.uint8).ravel()
        check(lib().mplb_planner_set_search_region(self._h, ptr(m), m.size))

    def getSearchRegionMask(self):  # env_base::get_search_region, env_base.h:365
        n = int(lib().mplb_planner_get_search_region(self._h, None, 0))
        out = np.zeros(n, dtype=np.uint8)
        if n:
            lib().mplb_planner_get_search_region(self._h, ptr(out), n)
        return out

    def getSearchRegion(self):  # map_planner.cpp:97-114: centres of the in-region cells
        mask = self.getSearchRegionMask()
        if mask.size == 0:
            return np.zeros((0, self.dim))
        nd = np.asarray(self.map_util_.getDim())
        idx = np.flatnonzero(mask)
        cells = np.stack(np.unravel_index(idx, tuple(nd[::-1])), axis=1)[:, ::-1]  # x fastest
        cells = cells[np.lexsort(cells[:, ::-1].T)]  # the reference walks x outermost
        return (cells + 0.5) * self.map_util_.getRes() + np.asarray(self.map_util_.getOrigin())[:self.dim]

    def setPotentialMap(self, pot):  # env_map::set_potential_map, env_map.h:182 (None clears)
        if pot is None:
            check(lib().mplb_planner_set_potential_map(self._h, None, 0))
            return
        m = np.ascontiguousarray(pot, dtype=np.int8).ravel()
        check(lib().mplb_planner_set_potential_map(self._h, ptr(m), m.size))

    def updatePotentialMap(self, pos):  # map_planner.cpp:327-391 (rewrites the shared map, like the reference)
        check(lib().mplb_planner_update_potential_map(self._h, ptr(self._vec3(pos)), ptr(self.potential_radius_),
                                                      ptr(self.potential_map_range_), float(self.pow_)))

    def iterativePlan(self, start, goal, raw_traj, max_num):  # map_planner.cpp:394-434
        traj = raw_traj
        prev_cost = 0.0
        cnt = 0
        while cnt < max_num:
            cnt += 1
            self.setSearchRegion([w.pos for w in traj.getWaypoints()], False)
            if not self.plan(start, goal):
                return False
            traj = self.getTraj()
            if prev_cost == self.traj_cost_:
                break
            prev_cost = self.traj_cost_
        return True

    # ---- plan (planner_base.h:275-325)
    def plan(self, start, goal):
        s, g = start, goal
        if isinstance(start, Waypoint):
            s = waypoints_array(1)
            start.to_record(s[0])
        if isinstance(goal, Waypoint):
            g = waypoints_array(1)
            goal.to_record(g[0])
        res = np.zeros(1, dtype=_lib.RESULT_DTYPE)
        check(lib().mplb_plan(self._h, ptr(s), ptr(g), ptr(res)))
        self._last = res[0]
        self._control = int(s["control"][0])
        self._initialized = True
        self.traj_cost_ = float(res[0]["cost"])
        st = int(res[0]["status"])
        # traj_ is rewritten only where the reference writes it: recoverTraj success or failure (graph_search.h:447-451).
        # start-not-free (planner_base.h:283-287), start-is-goal (graph_search.h:44), MaxExpandStep and empty queue
        # (graph_search.h:149-161) leave the previous trajectory in place.
        if st == PLAN_OK:
            acts, seg = self.getActions(), self.getSegStates()
            self.traj_ = Trajectory([Primitive(self.dim, self._control, seg[i], self.U_[acts[i]], self.dt_) for i in range(len(acts))])
        elif st == PLAN_TRACEBACK_FAILED:
            self.traj_ = Trajectory()
        return st in (PLAN_OK, PLAN_START_IS_GOAL)

    # ---- LPA* (planner_base.h:155-176, map_planner.h:74-87; mpl_test_node/src/map_replanner_node.cpp is the caller)
    def setLPAstar(self, use_lpastar):  # planner_base.h:170-176
        check(lib().mplb_planner_set_lpastar(self._h, int(bool(use_lpastar))))

    def getSubStateSpace(self, time_step):  # planner_base.h:155 -> state_space.h:116-204
        return check(lib().mplb_get_sub_state_space(self._h, int(time_step)))

    def getLinkedNodes(self):  # map_planner.cpp:125-158
        n = check(lib().mplb_get_linked_nodes(self._h, None, 0))
        pts = np.zeros((max(n, 1), 3), dtype=np.float64)
        n = check(lib().mplb_get_linked_nodes(self._h, ptr(pts), pts.shape[0]))
        return pts[:n, :self.dim]

    def _cells3(self, pns):
        c = np.asarray(pns, dtype=np.int32).reshape(len(pns), -1)
        c3 = np.zeros((len(c), 3), dtype=np.int32)
        c3[:, :c.shape[1]] = c
        return c3

    def updateBlockedNodes(self, blocked_pns):  # map_planner.cpp:160-171
        c3 = self._cells3(blocked_pns)
        return check(lib().mplb_update_blocked_nodes(self._h, ptr(c3), len(c3)))

    def updateClearedNodes(self, cleared_pns):  # map_planner.cpp:173-185
        c3 = self._cells3(cleared_pns)
        return check(lib().mplb_update_cleared_nodes(self._h, ptr(c3), len(c3)))

    def lpaNodes(self):
        """hm_ in iteration order (state dump: key, coord, g, rhs, h, flags, list hashes)"""
        n = check(lib().mplb_lpa_get_nodes(self._h, None, 0))
        a = np.zeros(max(n, 1), dtype=_lib.LPA_NODE_DTYPE)
        n = check(lib().mplb_lpa_get_nodes(self._h, ptr(a), a.size))
        return a[:n]

    def lpaHeap(self):
        """pq_ in its internal array order"""
        n = check(lib().mplb_lpa_get_heap(self._h, None, 0))
        a = np.zeros(max(n, 1), dtype=_lib.LPA_HEAP_DTYPE)
        n = check(lib().mplb_lpa_get_heap(self._h, ptr(a), a.size))
        return a[:n]

    def lpaBestChild(self):
        """best_child_ of the last LPA* trajectory, start .. goal"""
        n = check(lib().mplb_lpa_get_best_child(self._h, None, 0))
        a = np.zeros(max(n, 1), dtype=_lib.LPA_NODE_DTYPE)
        n = check(lib().mplb_lpa_get_best_child(self._h, ptr(a), a.size))
        return a[:n]

    def lpaCapacity(self):
        """capacity of the LPA* session's device arrays (mplb_lpa_get_capacity): cap_nodes, cap_pred, tsize,
        n_nodes_physical (records in use, those a getSubStateSpace dropped from hm_ included) and grows (doublings)"""
        v = [C.c_int32() for _ in range(5)]
        check(lib().mplb_lpa_get_capacity(self._h, *[C.byref(x) for x in v]))
        return dict(zip(("cap_nodes", "cap_pred", "tsize", "n_nodes_physical", "grows"), (x.value for x in v)))

    def result(self):
        return self._last

    def getTrajCost(self):
        return self.traj_cost_

    def getExpandedNum(self):  # planner_base.h:148
        return int(self._last["pops"])

    def getActions(self):
        n = check(lib().mplb_get_actions(self._h, None, 0))
        a = np.zeros(max(n, 1), dtype=np.int32)
        check(lib().mplb_get_actions(self._h, ptr(a), a.size))
        return a[:n]

    def getSegStates(self):
        n = check(lib().mplb_get_seg_states(self._h, None, 0))
        s = np.zeros((max(n, 1), 13), dtype=np.float64)
        check(lib().mplb_get_seg_states(self._h, ptr(s), s.shape[0]))
        return s[:n]

    def getTraj(self):  # planner_base.h:28 (traj_ as last written by recoverTraj, graph_search.h:369-455)
        return self.traj_

    def getNodes(self):
        n = check(lib().mplb_get_nodes(self._h, None, 0))
        a = np.zeros(max(n, 1), dtype=_lib.NODE_DTYPE)
        check(lib().mplb_get_nodes(self._h, ptr(a), a.size))
        return a[:n]

    def getPopLog(self):
        n = check(lib().mplb_get_pop_log(self._h, None, 0))
        a = np.zeros(max(n, 1), dtype=np.int32)
        check(lib().mplb_get_pop_log(self._h, ptr(a), a.size))
        return a[:n]

    def getCloseSet(self):  # planner_base.h:84-91 (unordered positions of closed nodes)
        nodes = self.getNodes()
        return nodes["state"][nodes["closed"] != 0][:, :self.dim]

    def getOpenSet(self):  # planner_base.h:77-81
        n = check(lib().mplb_get_open(self._h, None, 0))
        ids = np.zeros(max(n, 1), dtype=np.int32)
        check(lib().mplb_get_open(self._h, ptr(ids), ids.size))
        return self.getNodes()["state"][ids[:n]][:, :self.dim]

    def getExpandedNodes(self):  # planner_base.h:140 (expanded_nodes_, pop order)
        return self.getNodes()["state"][self.getPopLog()][:, :self.dim]

    def getExpandedEdges(self):
        """planner_base.h:143-145 (env_map.h:166): the finite-cost primitives of every expanded node, in expansion order.
        Rebuilt by running get_succ (mplb_expand) over the popped states; plain-map plans only."""
        nodes = self.getNodes()
        st = nodes["state"][self.getPopLog()]
        w = waypoints_array(len(st))
        w["pos"], w["vel"], w["acc"], w["jrk"] = st[:, 0:3], st[:, 3:6], st[:, 6:9], st[:, 9:12]
        w["control"] = self._control
        rows = self.expand(w)
        prs = []
        for i in range(len(st)):
            for a in np.flatnonzero(np.isfinite(rows[i]["cost"]) & (rows[i]["verdict"] >= 3)):
                prs.append(Primitive(self.dim, self._control, st[i], self.U_[a], self.dt_))
        return prs

    def getValidPrimitives(self):
        """planner_base.h:30-51: the finite-cost predecessor edges of every node.  In A* a predecessor record is appended
        exactly when an expanded node yields a finite-cost successor (graph_search.h:81,100-102), so this is the same
        set of primitives as getExpandedEdges (the reference returns it in hash-map order)."""
        return self.getExpandedEdges()

    def getAllPrimitives(self):  # planner_base.h:54-74: A* never records an infinite-cost predecessor, same set again
        return self.getExpandedEdges()

    def reset(self):  # planner_base.h:164-167
        check(lib().mplb_planner_reset(self._h))
        self._initialized = False
        self._last = None
        self.traj_cost_ = None

    # ---- batch (north-star extension; every entry behaves like plan())
    def plan_batch(self, starts, goals, max_seg=0, want_states=False):
        n = len(starts)
        res = np.zeros(n, dtype=_lib.RESULT_DTYPE)
        acts = np.full((n, max_seg), -1, dtype=np.int32) if max_seg > 0 else None
        segs = np.zeros((n, max_seg, 13), dtype=np.float64) if (max_seg > 0 and want_states) else None
        check(lib().mplb_plan_batch(self._h, ptr(starts), ptr(goals), n, ptr(res), ptr(acts), ptr(segs), max_seg))
        return res, acts, segs

    def plan_batch_device(self, d_starts, d_goals, n, d_results, d_actions=0, d_segs=0, max_seg=0, stream=0):
        """All pointers are device addresses (ints), e.g. torch tensor .data_ptr()."""
        vp = lambda x: C.c_void_p(int(x)) if x else None  # noqa: E731
        check(lib().mplb_plan_batch_device(self._h, vp(d_starts), vp(d_goals), n, vp(d_results), vp(d_actions), vp(d_segs),
                                           max_seg, vp(stream)))

    def refine_trajectories(self, results, actions, seg_states, plan_control, control=JRK, yaw_control=VEL):
        """map_planner_node.cpp:216-227 for every plan of a batch (waypoints of the planned trajectory, interior ones flagged
        Control::VEL, the planner's dt per segment, TrajSolver<Dim>(control, yaw_control)) — gathered and solved on the GPU.
        Returns (coefs [n, max_seg, dim + 1, 6], n_segs [n])."""
        n, max_seg = int(actions.shape[0]), int(actions.shape[1])
        results = np.ascontiguousarray(results)
        actions = np.ascontiguousarray(actions, dtype=np.int32)
        seg_states = np.ascontiguousarray(seg_states, dtype=np.float64)
        coefs = np.zeros((n, max_seg, self.dim + 1, 6), dtype=np.float64)
        nseg = np.zeros(max(n, 1), dtype=np.int32)
        check(lib().mplb_refine_trajectories(self._h, ptr(results), ptr(actions), ptr(seg_states), n, max_seg, int(plan_control),
                                             int(control), int(yaw_control), ptr(coefs), ptr(nseg)))
        return coefs, nseg[:n]

    def serialize_trajectories(self, results, actions, seg_states, z=0.0, frame_id="map", seq=0, stamp=(0, 0)):
        """toTrajectoryROSMsg + ROS 1 serialisation of planning_ros_msgs/Trajectory for every plan of a batch
        (primitive_ros_utils.h:62-113, map_planner_node.cpp:55-57,206-208), written by the GPU.  Returns a list of
        `bytes`, one message per plan (None for a plan whose trajectory was truncated by max_seg)."""
        n, max_seg = int(actions.shape[0]), int(actions.shape[1])
        results = np.ascontiguousarray(results)
        actions = np.ascontiguousarray(actions, dtype=np.int32)
        seg_states = np.ascontiguousarray(seg_states, dtype=np.float64)
        fid = frame_id.encode()
        stride = int(lib().mplb_trajectory_msg_size(max_seg, fid))
        out = np.zeros((n, stride), dtype=np.uint8)
        ln = np.zeros(n, dtype=np.uint32)
        check(lib().mplb_serialize_trajectories(self._h, ptr(results), ptr(actions), ptr(seg_states), n, max_seg, float(z),
                                                int(seq), int(stamp[0]), int(stamp[1]), fid, ptr(out), stride, ptr(ln)))
        return [out[i, :ln[i]].tobytes() if ln[i] else None for i in range(n)]

    def last_batch_stats(self):
        ms, l, t = C.c_double(), C.c_int32(), C.c_int32()
        check(lib().mplb_last_batch_stats(self._h, C.byref(ms), C.byref(l), C.byref(t)))
        return dict(kernel_ms=ms.value, launches=l.value, tiers=t.value)

    def last_batch_tiers(self):
        """One dict per arena tier pass of the last batch (mplb_tier_info: cap, slots, n_work, n_overflow, hcap, load_inv,
        tsize_max, log_cap, stride_bytes, nomem, ordered, resident)."""
        n = check(lib().mplb_last_batch_tiers(self._h, None, 0))
        rows = np.zeros(max(n, 1), dtype=_lib.TIER_DTYPE)
        check(lib().mplb_last_batch_tiers(self._h, ptr(rows), rows.size))
        return [{k: int(r[k]) for k in _lib.TIER_DTYPE.names if k != "reserved"} for r in rows[:n]]

    def expand(self, states):
        """env_map::get_succ rows for arbitrary states (env_map.h:147-172): array [n, |U|] of trace records."""
        n = len(states)
        rows = np.zeros((n, self.U_.shape[0]), dtype=_lib.TRACE_DTYPE)
        check(lib().mplb_expand(self._h, ptr(states), n, ptr(rows)))
        return rows

    def probe_samples(self, states):
        """The search kernel's filtered collision sampler on arbitrary states: one row per (state, control needing
        sampling, sample time), sorted by (state, control, k).  Returns (rows, use_fast, fast_delta)."""
        n = len(states)
        uf, fd = C.c_int32(), C.c_double()
        cnt = check(lib().mplb_probe_samples(self._h, ptr(states), n, None, 0, C.byref(uf), C.byref(fd)))
        rows = np.zeros(max(cnt, 1), dtype=_lib.PROBE_DTYPE)
        got = check(lib().mplb_probe_samples(self._h, ptr(states), n, ptr(rows), rows.size, None, None))
        assert got == cnt, (got, cnt)
        rows = rows[:cnt]
        rows = rows[np.lexsort((rows["k"], rows["control"], rows["state"]))]
        return rows, int(uf.value), float(fd.value)

    def key_layout(self, control):
        """The search configuration for start waypoints of `control` (mplb_planner_key_layout): dict of key_bits,
        key_wide and use_fast.  Raises MplbError where planning with it would."""
        kb, kw, uf = C.c_int32(), C.c_int32(), C.c_int32()
        check(lib().mplb_planner_key_layout(self._h, int(control), C.byref(kb), C.byref(kw), C.byref(uf)))
        return dict(key_bits=kb.value, key_wide=kw.value, use_fast=uf.value)


class OccMapPlanner(MapPlanner):  # map_planner.h:122
    def __init__(self, verbose=False):
        super().__init__(2, verbose)


class VoxelMapPlanner(MapPlanner):  # map_planner.h:125
    def __init__(self, verbose=False):
        super().__init__(3, verbose)
