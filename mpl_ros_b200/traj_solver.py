"""Python mirror of the reference's trajectory post-processing surface over the C ABI (mplb_traj_solve_batch):
  TrajSolver<Dim>   motion_primitive_library/include/mpl_traj_solver/traj_solver.h:12-109
Method names and behaviour follow the reference (setWaypoints / setPath / setV / setDts / solve / getPath / getWaypoints /
getDts); the spline itself (PolySolver::solve, poly_solver.cpp:23-221) is solved on the GPU, one CTA per trajectory, and
`solve_batch` exposes the batch the GPU is there for.  No CPU fallback: without libmplb.so or a device the call raises."""
import numpy as np

from . import _lib
from ._lib import check, lib, ptr
from .maps import VEL
from .planner import Primitive, Trajectory, Waypoint


def solve_batch(dim, control, waypoint_lists, dts_lists, yaw_control=VEL):
    """waypoint_lists: per trajectory a WAYPOINT_DTYPE array; dts_lists: per trajectory W - 1 durations.
    Returns a list of (n_seg, dim + 1, 6) coefficient arrays (axes, then yaw; highest order first); n_seg = 0 where the
    reference returns an empty Trajectory."""
    n = len(waypoint_lists)
    off = np.zeros(n + 1, dtype=np.int32)
    for i, w in enumerate(waypoint_lists):
        off[i + 1] = off[i] + len(w)
    wps = np.zeros(max(int(off[-1]), 1), dtype=_lib.WAYPOINT_DTYPE)
    slots = [max(len(w) - 1, 0) for w in waypoint_lists]
    dts = np.zeros(max(sum(slots), 1), dtype=np.float64)
    so = 0
    for i, (w, d) in enumerate(zip(waypoint_lists, dts_lists)):
        wps[off[i]:off[i + 1]] = w
        d = np.asarray(d, dtype=np.float64)
        if len(d) != slots[i]:
            raise ValueError("trajectory %d: %d waypoints need %d durations, got %d" % (i, len(w), slots[i], len(d)))
        dts[so:so + slots[i]] = d
        so += slots[i]
    coefs = np.zeros((max(so, 1), dim + 1, 6), dtype=np.float64)
    nseg = np.zeros(max(n, 1), dtype=np.int32)
    check(lib().mplb_traj_solve_batch(dim, int(control), int(yaw_control), n, ptr(off), ptr(wps), ptr(dts), ptr(coefs), ptr(nseg)))
    out, so = [], 0
    for i in range(n):
        out.append(coefs[so:so + nseg[i]].copy())
        so += slots[i]
    return out


def last_stats():
    """What the last solve of this thread launched (mplb_traj_solve_last_stats): dict of n_traj, max_wp, pos_shared, pos_global,
    yaw_shared, yaw_global, smem_bytes and global_bytes."""
    st = np.zeros(1, dtype=_lib.TRAJ_STATS_DTYPE)
    check(lib().mplb_traj_solve_last_stats(ptr(st)))
    return {k: int(st[0][k]) for k in _lib.TRAJ_STATS_DTYPE.names}


class TrajSolver:
    """traj_solver.h:12-109."""

    def __init__(self, dim, control, yaw_control=VEL, debug=False):
        self.dim, self.control_, self.yaw_control_ = dim, int(control), int(yaw_control)
        self.path_, self.waypoints_, self.dts_, self.v_ = [], [], [], 1.0

    def setWaypoints(self, ws):  # traj_solver.h:39-43
        self.path_ = [np.array(w.pos, dtype=np.float64) for w in ws]
        self.waypoints_ = list(ws)

    def setV(self, v):  # :46
        self.v_ = float(v)

    def setDts(self, dts):  # :50
        self.dts_ = [float(d) for d in dts]

    def setPath(self, path):  # :54-70: interior waypoints Control::VEL, the two ends carry `control`
        self.path_ = [np.array(p, dtype=np.float64) for p in path]
        self.waypoints_ = []
        for p in self.path_:
            w = Waypoint(self.dim, VEL)
            w.pos[:] = p[:self.dim]
            self.waypoints_.append(w)
        if self.waypoints_:
            # control is a 5-bit field in the reference (waypoint.h:54), so the *xYAW flags survive the assignment
            self.waypoints_[0].control = self.control_
            self.waypoints_[-1].control = self.control_

    def _allocate_time(self):  # :122-131: L-inf distance over v
        if len(self.path_) < 2 or self.v_ <= 0:
            return []
        return [float(np.max(np.abs(self.path_[i][:self.dim] - self.path_[i - 1][:self.dim]))) / self.v_
                for i in range(1, len(self.path_))]

    def solve(self, verbose=False):  # :73-109
        if len(self.waypoints_) != len(self.dts_) + 1:
            self.dts_ = self._allocate_time()
        rec = np.zeros(len(self.waypoints_), dtype=_lib.WAYPOINT_DTYPE)
        for i, w in enumerate(self.waypoints_):
            w.to_record(rec[i])
        if len(rec) != len(self.dts_) + 1:
            return Trajectory()
        coefs = solve_batch(self.dim, self.control_, [rec], [self.dts_], self.yaw_control_)[0]
        control = self.waypoints_[0].control if self.waypoints_ else 0
        return Trajectory([Primitive.from_coeffs(self.dim, c[:self.dim], c[self.dim], self.dts_[i], control) for i, c in enumerate(coefs)])

    def getPath(self):
        return self.path_

    def getWaypoints(self):
        return self.waypoints_

    def getDts(self):
        return self.dts_


class TrajSolver2D(TrajSolver):
    def __init__(self, control, yaw_control=VEL, debug=False):
        super().__init__(2, control, yaw_control, debug)


class TrajSolver3D(TrajSolver):
    def __init__(self, control, yaw_control=VEL, debug=False):
        super().__init__(3, control, yaw_control, debug)
