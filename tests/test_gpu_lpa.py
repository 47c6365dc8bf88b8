"""LPA* on the GPU (mplb_lpa.cu / mplb_lpa_core.h) through the reference-shaped Python surface (setLPAstar, plan,
getLinkedNodes, updateBlockedNodes / updateClearedNodes, getSubStateSpace, MapUtil edits) against the oracle, step by step
and EXACTLY (tolerance 0): result records, the state space in hm_ order with g / rhs / h / flags and the hashes of the stored
successor and predecessor lists, the priority-queue array, best_child_, the linked points — and against the fixture recorded
from the reference's own LPA* sources (tests/golden/lpa_flows.npz), which keeps the link where neither /root/reference nor
oracle/_ref exists.  The flows replay mpl_test_node/src/map_replanner_node.cpp:107-241."""
import os

import numpy as np
import pytest

import mpl_ros_b200 as mp
from mpl_ros_b200 import _lib
import oracle
from oracle.lpa import LPA_HEAP_DTYPE, LPA_NODE_DTYPE
import lpa_flow

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden", "lpa_flows.npz")


class GpuMap:
    def __init__(self, origin, dim, data, res):
        self.mu = mp.MapUtil(len(dim))
        self.mu.setMap(origin, dim, data, res)

    def free_unknown(self):
        self.mu.freeUnknown()

    def set_cells(self, cells, value):
        self.mu.setCells(cells, value)


class GpuPlanner:
    """the LpaMixin call shapes of tests/lpa_flow.py over the product's MapPlanner"""

    def __init__(self, dim):
        self.dim = dim
        self.pl = mp.MapPlanner(dim, False)
        self.pl.setLPAstar(True)

    def set_map(self, m):
        self._map = m
        self.pl.setMapUtil(m.mu)

    def set_param(self, key, v):
        if key in ("tol_pos", "tol_vel", "tol_acc", "max_num", "epsilon", "lpa_init_nodes", "lpa_init_preds"):
            self.pl._set(key, v)
        else:
            {"v_max": self.pl.setVmax, "a_max": self.pl.setAmax, "j_max": self.pl.setJmax, "dt": self.pl.setDt, "w": self.pl.setW}[key](v)

    def set_controls(self, U):
        self.pl.setU(U)

    def lpa_plan(self, s, g):
        self.ok = self.pl.plan(s, g)
        r = np.zeros(1, dtype=oracle.RESULT_DTYPE)
        for f in oracle.RESULT_DTYPE.names:
            r[f] = self.pl.result()[f]
        return r[0]

    def lpa_get_linked_nodes(self):
        p = self.pl.getLinkedNodes()
        out = np.zeros((len(p), 3))
        out[:, :self.dim] = p
        return out

    def lpa_update_blocked_nodes(self, pns):
        return self.pl.updateBlockedNodes(pns)

    def lpa_update_cleared_nodes(self, pns):
        return self.pl.updateClearedNodes(pns)

    def lpa_get_sub_state_space(self, k):
        return self.pl.getSubStateSpace(k)

    def lpa_nodes(self):
        a = self.pl.lpaNodes()
        o = np.zeros(len(a), dtype=LPA_NODE_DTYPE)
        for f in LPA_NODE_DTYPE.names:
            o[f] = a[f]
        return o

    def lpa_heap(self):
        a = self.pl.lpaHeap()
        o = np.zeros(len(a), dtype=LPA_HEAP_DTYPE)
        o["fval"], o["key_hash"] = a["fval"], a["key_hash"]
        return o

    def lpa_best_child(self):
        return self.pl.lpaBestChild()["key"].copy()

    def lpa_best_child_states(self):
        return self.pl.lpaBestChild()["state"].copy()

    def lpa_waypoint(self, k):
        st = self.lpa_best_child_states()[k]
        w = oracle.make_waypoints(1)
        w["pos"][0], w["vel"][0], w["acc"][0], w["jrk"][0], w["yaw"][0] = st[0:3], st[3:6], st[6:9], st[9:12], st[12]
        w["control"] = self._lpa_control
        return w


@pytest.mark.parametrize("name", list(lpa_flow.FLOWS))
def test_flow_equals_oracle_and_fixture(name):
    a, _ = lpa_flow.run_flow(name, oracle.OracleMap, oracle.OraclePlanner)
    b, gp = lpa_flow.run_flow(name, GpuMap, GpuPlanner)
    lpa_flow.assert_same(a, b, name)
    gold = np.load(GOLD)[name]
    d = lpa_flow.digest(b)
    assert len(d) == len(gold)
    for f in gold.dtype.names:
        assert np.array_equal(d[f], gold[f]), (name, f)
    if a[0]["res"]["status"] == 0:  # the trajectory behind getTraj(): same action ids as the oracle's recoverTraj
        assert len(gp.pl.getTraj().getPrimitives()) == a[-1]["res"]["n_seg"] or a[-1]["res"]["status"] != 0


def test_trajectory_actions_and_reset():
    m, mp_, pl, dim, start, goal = lpa_flow.build(GpuMap, GpuPlanner, "skir")
    om, omp, opl, _, _, _ = lpa_flow.build(oracle.OracleMap, oracle.OraclePlanner, "skir")
    s, g = oracle.make_waypoints(1), oracle.make_waypoints(1)
    lpa_flow.fill_waypoints(s, start, mp.ACC)
    lpa_flow.fill_waypoints(g, goal, mp.ACC)
    r, ro = pl.lpa_plan(s, g), opl.lpa_plan(s, g)
    assert r["status"] == ro["status"] == 0 and r["cost"] == ro["cost"] == 47.0 and r["pops"] == 348
    assert np.array_equal(pl.pl.getActions(), opl.lpa_actions())
    assert np.array_equal(pl.pl.getSegStates(), opl.lpa_best_child_states()[:-1])
    r2 = pl.lpa_plan(s, g)  # nothing changed: the loop condition fails at once, same trajectory
    assert r2["status"] == 0 and r2["pops"] == 0 and r2["cost"] == 47.0
    pl.pl.reset()           # PlannerBase::reset: a new state space
    r3 = pl.lpa_plan(s, g)
    assert r3["pops"] == 348 and r3["n_nodes"] == r["n_nodes"]
    with pytest.raises(mp.MplbError):  # the A* node getters do not serve an LPA* plan
        pl.pl.getNodes()


def test_batch_of_replanners():
    """one CTA per robot: mplb_lpa_plan_batch over independent planners equals planning them one by one"""
    import ctypes as C
    names = ["skir", "skir", "skir", "skir", "skir"]
    goals = [(1.5, 1.5, 5.5), (5.5, 1.5, 0.5), (1.5, 5.5, 0.5), (3.5, 3.5, 3.5), (1.5, 1.5, 5.5)]
    controls = [mp.ACC, mp.ACC, mp.ACC, mp.ACC, mp.JRK]  # the jerk replanner outgrows its arrays (76 657 nodes): the launch is
    planners, singles = [], []                             # repeated for it while the finished neighbours must stay untouched
    for nm, c in zip(names, controls):
        extra = {"max_num": 30000} if c == mp.JRK else None
        planners.append(lpa_flow.build(GpuMap, GpuPlanner, nm, extra))
        singles.append(lpa_flow.build(GpuMap, GpuPlanner, nm, extra))
    n = len(names)
    s, g = mp.waypoints_array(n), mp.waypoints_array(n)
    for i in range(n):
        s["pos"][i], g["pos"][i] = planners[i][4], goals[i]
        s["control"][i] = g["control"][i] = controls[i]
    res = np.zeros(n, dtype=_lib.RESULT_DTYPE)
    handles = (C.c_void_p * n)(*[p[2].pl._h for p in planners])
    _lib.check(_lib.lib().mplb_lpa_plan_batch(handles, n, _lib.ptr(s), _lib.ptr(g), _lib.ptr(res)))
    for i in range(n):
        r1 = singles[i][2].lpa_plan(s[i:i + 1], g[i:i + 1])
        for f in ("status", "n_seg", "cost", "pops", "n_nodes", "n_open", "n_closed", "pop_hash", "closed_hash"):
            assert res[i][f] == r1[f], (i, f)
        assert np.array_equal(planners[i][2].lpa_nodes()["g"], singles[i][2].lpa_nodes()["g"])
    assert len({float(r["cost"]) for r in res}) > 1
    assert res[4]["n_nodes"] > 65536 and res[4]["pops"] == 11945 and res[0]["pops"] == 348


def test_shaping_is_rejected_under_lpastar():
    m, mp_, pl, dim, start, goal = lpa_flow.build(GpuMap, GpuPlanner, "corridor")
    pl.pl.setSearchRadius([0.5, 0.5])
    pl.pl.setSearchRegion([start, goal])
    s, g = oracle.make_waypoints(1), oracle.make_waypoints(1)
    lpa_flow.fill_waypoints(s, start, mp.ACC)
    lpa_flow.fill_waypoints(g, goal, mp.ACC)
    with pytest.raises(mp.MplbError):
        pl.lpa_plan(s, g)
