"""LPA* replanning flows with a potential map (distance-map replanner) and with yaw controls, over any planner object with the
LpaMixin call shapes of tests/lpa_flow.py plus `set_vec` / `update_potential_map` (oracle.OraclePlanner, oracle.ref.RefPlanner,
the host build of the device core in tests/lpa_emul_shaped.py, and the CUDA path's adaptor in test_gpu_lpa_shaped.py).

Every flow: (optionally) updatePotentialMap at the start, LPA* plan, then the replanner node's edit cycle of tests/lpa_flow.py
(block cells on the path, getLinkedNodes, updateBlockedNodes, replan; clear half of them, updateClearedNodes, replan;
getSubStateSpace(1), replan from the next waypoint).  The `restamp` flows call updatePotentialMap again after every map edit,
which leaves the stored edge costs as they were (the reference never recomputes them).  Capped flows (max_num) plan until the
search gets through, as a node that re-triggers the replan does."""
import math

import numpy as np

import oracle
import lpa_emul_shaped
import lpa_flow
from helpers import load_config

VEL, ACC, JRK, SNP, YAW = 1, 3, 7, 15, 16

# name -> dict(config, control, params, u_yaw (None: rows of Dim entries), pot (None or radius / range / restamp),
#              start_yaw, rounds, capped)
FLOWS = {
    # 2-D distance-map replanner on corridor (test_distance_map_planner_2d settings), w_grad 0 and 0.3, with / without re-stamp
    "corridor_pot": dict(config="corridor", control=ACC, params=dict(potential_weight=0.5, gradient_weight=0.0),
                         pot=dict(radius=[1.0, 1.0], range=[0.0, 0.0], restamp=False)),
    "corridor_pot_grad": dict(config="corridor", control=ACC, params=dict(potential_weight=0.5, gradient_weight=0.3),
                              pot=dict(radius=[1.0, 1.0], range=[0.0, 0.0], restamp=False)),
    "corridor_pot_restamp": dict(config="corridor", control=ACC, params=dict(potential_weight=0.5, gradient_weight=0.3),
                                 pot=dict(radius=[1.0, 1.0], range=[0.0, 0.0], restamp=True)),
    # 3-D potential stamped in a local box around the start (setPotentialMapRange)
    "simple_pot_local": dict(config="simple", control=ACC, params=dict(potential_weight=0.5, gradient_weight=0.1),
                             pot=dict(radius=[1.5, 1.5, 1.0], range=[4.0, 4.0, 2.0], restamp=False)),
    # 2-D ACCxYAW replanner with the control set, yaw_max and start yaw of test_planner_2d_with_yaw
    "corridor_yaw": dict(config="corridor", control=ACC | YAW, params=dict(yaw_max=0.7), u_yaw=0.5, start_yaw=math.pi / 2),
    # potential and yaw together: test_distance_map_planner_2d_with_yaw without its search radius
    "corridor_pot_yaw": dict(config="corridor", control=ACC | YAW, params=dict(potential_weight=0.5, gradient_weight=0.0, yaw_max=0.5),
                             u_yaw=0.5, pot=dict(radius=[1.0, 1.0], range=[0.0, 0.0], restamp=False), rounds=1),
    # 3-D JRKxYAW with a max_num cap: the search stops at MaxExpandStep and continues from the kept state; it outgrows small arrays
    "skir_jrk_yaw": dict(config="skir", control=JRK | YAW, params=dict(yaw_max=1.2, max_num=600), u_yaw=0.5, capped=True),
    # 3-D SNPxYAW: the widest lattice key (12 polynomial fields + yaw = 13)
    "skir_snp_yaw": dict(config="skir", control=SNP | YAW, params=dict(yaw_max=1.2, j_max=2.0, max_num=150), u_yaw=0.5, capped=True),
}
POT_ONLY = [n for n, f in FLOWS.items() if f.get("pot") and not f["control"] & YAW]
YAW_FLOWS = [n for n, f in FLOWS.items() if f["control"] & YAW]


def controls(U, u_yaw):
    """rows (u, u_yaw) with the yaw rate innermost, `for (dyaw = -u_yaw; dyaw <= u_yaw; dyaw += u_yaw)` as the tests build them"""
    if u_yaw is None:
        return U
    ys, d = [], -u_yaw
    while d <= u_yaw:
        ys.append(d)
        d += u_yaw
    return np.array([list(r) + [y] for r in U for y in ys], dtype=np.float64)


def build(name, cls_map, cls_planner, extra=None):
    f = FLOWS[name]
    m, dim, params, U, start, goal = load_config(f["config"])
    mp_ = cls_map(m.origin, m.dim, m.data, m.res)
    mp_.free_unknown()
    pl = cls_planner(dim)
    pl.set_map(mp_)
    for k, v in dict(params, **f["params"], **(extra or {})).items():
        pl.set_param(k, v)
    pl.set_controls(controls(U, f.get("u_yaw")))
    pl._lpa_control = f["control"]
    if f.get("pot"):
        pl.set_vec("potential_radius", np.array(f["pot"]["radius"], dtype=np.float64))
        pl.set_vec("potential_map_range", np.array(f["pot"]["range"], dtype=np.float64))
    return m, mp_, pl, dim, start, goal


class _Restamp:
    """the map as the flow edits it: with `restamp`, every edit is followed by updatePotentialMap over a box of +-1.5 m around
    the edited cells.  (updatePotentialMap reads the map it rewrote before, so every cell that already carries potential
    becomes an obstacle: a re-stamp of the whole map would close the start in.)"""

    def __init__(self, m, mp_, pl, restamp):
        self.m, self.mp_, self.pl, self.restamp = m, mp_, pl, restamp

    def set_cells(self, cells, value):
        self.mp_.set_cells(cells, value)
        if self.restamp and len(cells):
            dim = cells.shape[1]
            centre = np.zeros(3)
            centre[:dim] = (cells.mean(axis=0) + 0.5) * self.m.res + self.m.origin[:dim]
            self.pl.set_vec("potential_map_range", np.full(dim, 1.5))
            self.pl.update_potential_map(centre)


def waypoints(pos, control, yaw):
    w = oracle.make_waypoints(1)
    lpa_flow.fill_waypoints(w, pos, control)
    w["yaw"] = yaw
    return w


def run_flow(name, cls_map, cls_planner, extra=None):
    """-> (snapshots, planner)"""
    f = FLOWS[name]
    m, mp_, pl, dim, start, goal = build(name, cls_map, cls_planner, extra)
    pos3 = np.zeros(3)
    pos3[:dim] = start
    if f.get("pot"):
        pl.update_potential_map(pos3)
    s = waypoints(start, f["control"], f.get("start_yaw", 0.0))
    g = waypoints(goal, f["control"], 0.0)
    if f.get("capped"):
        snaps = []
        for _ in range(4):
            res = pl.lpa_plan(s, g)
            snaps.append(lpa_flow.snapshot(pl, res))
            if res["status"] == 0:
                break
        linked = pl.lpa_get_linked_nodes()
        snaps.append(lpa_flow.snapshot(pl, None, linked))
        return snaps, pl
    edit = _Restamp(m, mp_, pl, bool(f.get("pot", {}).get("restamp")))
    return _cycle(pl, edit, m, dim, s, g, f.get("rounds", 2)), pl


def _cycle(pl, mp_, m, dim, s, g, n_rounds):
    """the edit cycle of lpa_flow.run from given start / goal waypoints (the start may carry a yaw)"""
    snaps = []
    res = pl.lpa_plan(s, g)
    snaps.append(lpa_flow.snapshot(pl, res))
    grid = m.data.reshape(-1).copy()
    lin_of = lambda c: c[:, 0] + m.dim[0] * c[:, 1] + (m.dim[0] * m.dim[1] * c[:, 2] if dim == 3 else 0)  # noqa: E731
    for rnd in range(n_rounds):
        if res["status"] != 0:
            break
        path = lpa_flow.path_of_best_child(pl, res)
        linked = pl.lpa_get_linked_nodes()
        k = int(len(path) * (0.45, 0.7)[rnd % 2])
        cand = lpa_flow.cells_on_path(m, dim, path[k:k + 1], 2)
        new_obs = cand[(grid[lin_of(cand)] >= 0) & (grid[lin_of(cand)] < 100)]
        grid[lin_of(new_obs)] = 100
        mp_.set_cells(new_obs, 100)
        pl.lpa_update_blocked_nodes(new_obs)
        snaps.append(lpa_flow.snapshot(pl, None, linked))
        res = pl.lpa_plan(s, g)
        snaps.append(lpa_flow.snapshot(pl, res))
        if res["status"] != 0:
            break
        linked = pl.lpa_get_linked_nodes()
        cleared = new_obs[: max(1, len(new_obs) // 2)]
        grid[lin_of(cleared)] = 0
        mp_.set_cells(cleared, 0)
        pl.lpa_update_cleared_nodes(cleared)
        snaps.append(lpa_flow.snapshot(pl, None, linked))
        pl._cleared_mismatch = getattr(pl, "cost_mismatch", lambda: None)()
        res = pl.lpa_plan(s, g)
        snaps.append(lpa_flow.snapshot(pl, res))
        if res["status"] != 0:
            break
        path = lpa_flow.path_of_best_child(pl, res)
        if len(path) < 3:
            break
        nxt = pl.lpa_waypoint(1)
        pl.lpa_get_sub_state_space(1)
        snaps.append(lpa_flow.snapshot(pl, None))
        s = nxt
        res = pl.lpa_plan(s, g)
        snaps.append(lpa_flow.snapshot(pl, res))
    return snaps


# ---------------------------------------------------------------- planners with potential-map support
class OraclePlanner(oracle.OraclePlanner):
    """the checker in a chosen trig mode (1 = the product's correctly rounded sin / cos, 0 = libm as the reference)"""
    TRIG = 1

    def __init__(self, dim):
        super().__init__(dim)
        self.set_param("trig_mode", self.TRIG)


class OraclePlannerLibm(OraclePlanner):
    TRIG = 0


def emu_classes(rev=False):
    """(map class, planner class) of the host build of the device core (tests/lpa_emul_shaped.py)"""
    return (lpa_emul_shaped.EmuMapRev, lpa_emul_shaped.EmuPlannerRev) if rev else (lpa_emul_shaped.EmuMap, lpa_emul_shaped.EmuPlanner)


def digest(snaps):
    return lpa_flow.digest(snaps)
