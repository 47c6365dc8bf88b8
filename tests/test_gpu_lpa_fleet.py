"""A fleet of LPA* replanners driven one call per replan step (mplb_lpa_plan_batch, mplb_lpa_get_linked_nodes_batch,
mplb_lpa_update_nodes_batch, mplb_lpa_sub_state_space_batch through MapPlanner's static batch members), in lockstep with the
same replanners driven by the single calls and with the oracle, exactly (tolerance 0) after every batched call: result records,
hm_ dumps, heap arrays, best_child_, linked points, visited counts, sizes and array capacities.  The fleet mixes every
tests/lpa_flow.py flow but the two large jerk flows, potential and yaw flows of tests/lpa_shaped_flow.py and seeded random replanners of
test_oracle_lpa_fuzz.  Then: launch counts that do not grow with the fleet, argument errors that leave every planner as it was,
and planLPABatch's trajectories."""
import numpy as np
import pytest

import mpl_ros_b200 as mp
import oracle
import lpa_flow
import lpa_shaped_flow as F
from test_gpu_lpa import GpuMap
from test_gpu_lpa_shaped import GpuPlanner
from test_oracle_lpa_fuzz import sequence_case

pytestmark = pytest.mark.gpu


class Member:
    """one replanner three times: `b` driven by the batched calls, `s` by the single calls, `o` the oracle"""

    def __init__(self, kind, name):
        self.name, self.oracle_ok, self.dropped = name, True, []
        if kind == "flow":
            cfg, control, params, _ = lpa_flow.FLOWS[name]
            made = [lpa_flow.build(cm, cp, cfg, params) for cm, cp in ((GpuMap, GpuPlanner), (GpuMap, GpuPlanner),
                                                                        (oracle.OracleMap, oracle.OraclePlanner))]
            self.m, dim, start, goal = made[0][0], made[0][3], made[0][4], made[0][5]
            for x in made:
                x[2]._lpa_control = control
            self.s_wp, self.g_wp = self._wp(start, control), self._wp(goal, control)
        elif kind == "shaped":
            f = F.FLOWS[name]
            made = [F.build(name, cm, cp) for cm, cp in ((GpuMap, GpuPlanner), (GpuMap, GpuPlanner), (oracle.OracleMap, F.OraclePlanner))]
            self.m, dim, start, goal = made[0][0], made[0][3], made[0][4], made[0][5]
            control = f["control"]
            if f.get("pot"):
                for x in made:
                    x[2].update_potential_map(np.r_[start, np.zeros(3 - dim)])
            self.s_wp, self.g_wp = F.waypoints(start, control, f.get("start_yaw", 0.0)), F.waypoints(goal, control, 0.0)
        else:  # seeded random replanner: (seed, dim)
            seed, dim = name
            _, (nd, origin, res, data, control, U, prm, start, goal, vel) = sequence_case(seed, dim)
            made = []
            for cm, cp in ((GpuMap, GpuPlanner), (GpuMap, GpuPlanner), (oracle.OracleMap, oracle.OraclePlanner)):
                m = cm(origin, nd, data, res)
                m.free_unknown()
                p = cp(dim)
                p.set_map(m)
                for k, v in prm.items():
                    p.set_param(k, v)
                p.set_controls(U)
                p._lpa_control = control
                made.append((None, m, p))

            class M:
                pass
            self.m = M()
            self.m.origin, self.m.dim, self.m.res, self.m.data = np.asarray(origin), np.asarray(nd), res, data
            self.s_wp, self.g_wp = oracle.make_waypoints(1), oracle.make_waypoints(1)
            self.s_wp["pos"][0, :dim], self.g_wp["pos"][0, :dim], self.s_wp["vel"][0, :dim] = start, goal, vel
            self.s_wp["control"] = self.g_wp["control"] = control
        self.dim = dim
        self.maps = [x[1] for x in made]
        self.b, self.s, self.o = (x[2] for x in made)
        self.grid = np.where(self.m.data.reshape(-1) == -1, 0, self.m.data.reshape(-1)).astype(np.int8)
        self.traj = False

    @staticmethod
    def _wp(pos, control):
        w = oracle.make_waypoints(1)
        lpa_flow.fill_waypoints(w, pos, control)
        return w

    def lin(self, c):
        d = self.m.dim
        return c[:, 0] + d[0] * c[:, 1] + (d[0] * d[1] * c[:, 2] if self.dim == 3 else 0)

    def set_cells(self, cells, value):
        if len(cells):
            self.grid[self.lin(cells)] = value
            for m in self.maps:
                m.set_cells(cells, value)


def snap(p, res=None, linked=None):
    out = lpa_flow.snapshot(p, res, linked)
    out["cap"] = p.pl.lpaCapacity() if hasattr(p, "pl") else None
    return out


def same(members, what, results=None, linked=None):
    """batched copy == single copy (capacity included) == oracle (where the oracle's case is defined)"""
    for i, mb in enumerate(members):
        r = None if results is None else results[i]
        lk = None if linked is None else linked[i]
        a, b = snap(mb.b, r[0] if r else None, lk[0] if lk else None), snap(mb.s, r[1] if r else None, lk[1] if lk else None)
        lpa_flow.assert_same([a], [b], "%s %s batch/single" % (what, mb.name))
        assert a["cap"] == b["cap"], (what, mb.name)
        if mb.oracle_ok:
            c = snap(mb.o, r[2] if r else None, lk[2] if lk else None)
            lpa_flow.assert_same([c], [a], "%s %s oracle" % (what, mb.name))


def plan_all(members):
    n = len(members)
    s, g = mp.waypoints_array(n), mp.waypoints_array(n)
    for i, mb in enumerate(members):
        s[i], g[i] = mb.s_wp[0], mb.g_wp[0]
    oks = mp.MapPlanner.planLPABatch([mb.b.pl for mb in members], s, g)
    results = []
    for i, mb in enumerate(members):
        ro = mb.o.lpa_plan(mb.s_wp, mb.g_wp) if mb.oracle_ok else None
        if ro is not None and (int(ro["status"]) == 3 and int(ro["pops"]) == 0 or mb.o.lpa_last_fault() & 2):
            mb.oracle_ok = False  # the reference reads an empty heap / walks a predecessor cycle here: no verdict to compare
        rs = mb.s.lpa_plan(mb.s_wp, mb.g_wp)
        rb = np.zeros(1, dtype=oracle.RESULT_DTYPE)[0]
        for f in oracle.RESULT_DTYPE.names:
            rb[f] = mb.b.pl.result()[f]
        assert oks[i] == mb.s.ok, mb.name
        # planLPABatch keeps traj_ / traj_cost_ as plan() does
        assert mb.b.pl.getTrajCost() == mb.s.pl.getTrajCost() or (np.isinf(mb.b.pl.getTrajCost()) and np.isinf(mb.s.pl.getTrajCost()))
        pa, pb = mb.b.pl.getTraj().getPrimitives(), mb.s.pl.getTraj().getPrimitives()
        assert len(pa) == len(pb) and all(np.array_equal(x.coeffs, y.coeffs) for x, y in zip(pa, pb)), mb.name
        mb.traj = int(rs["status"]) == 0
        results.append((rb, rs, ro))
    same(members, "plan", results)
    return results


def linked_all(members):
    got = mp.MapPlanner.getLinkedNodesBatch([mb.b.pl for mb in members])
    linked = []
    for i, mb in enumerate(members):
        lb = np.zeros((len(got[i]), 3))
        lb[:, :mb.dim] = got[i]
        ls = mb.s.lpa_get_linked_nodes()
        lo = mb.o.lpa_get_linked_nodes() if mb.oracle_ok else None
        linked.append((lb, ls, lo))
    same(members, "linked", linked=linked)
    return sum(len(x[0]) for x in linked)


def update_all(members, blocked, rnd):
    lists = []
    for i, mb in enumerate(members):
        if blocked:
            cells = np.zeros((0, mb.dim), dtype=np.int32)
            if mb.traj and (i + rnd) % 4 != 3:  # every fourth planner gets an empty range
                path = mb.s.lpa_best_child_states()[:, :mb.dim]
                k = int(len(path) * (0.45, 0.7)[(i + rnd) % 2])
                cand = lpa_flow.cells_on_path(mb.m, mb.dim, path[k:k + 1], 1 + (i % 2))
                if len(cand):
                    cand = cand[(mb.grid[mb.lin(cand)] >= 0) & (mb.grid[mb.lin(cand)] < 100)]
                    cells = np.concatenate([cand, cand[:2]]).astype(np.int32)  # duplicates, as the node's lists carry
            mb.dropped.append(cells)
            mb.set_cells(cells, 100)
        else:
            cells = mb.dropped[-1][: max(1, len(mb.dropped[-1]) // 2)] if len(mb.dropped[-1]) else mb.dropped[-1]
            mb.set_cells(cells, 0)
        lists.append(cells)
    fn = mp.MapPlanner.updateBlockedNodesBatch if blocked else mp.MapPlanner.updateClearedNodesBatch
    visited = fn([mb.b.pl for mb in members], lists)
    L = mp._lib.lib()
    for i, mb in enumerate(members):
        if len(lists[i]):
            v1 = (mb.s.lpa_update_blocked_nodes if blocked else mb.s.lpa_update_cleared_nodes)(lists[i])
        else:  # an empty list through the C call itself (the reference's loops do nothing for it)
            v1 = mp._lib.check((L.mplb_update_blocked_nodes if blocked else L.mplb_update_cleared_nodes)(mb.s.pl._h, None, 0))
        assert visited[i] == v1, (mb.name, visited[i], v1)
        if mb.oracle_ok and len(lists[i]):
            vo = (mb.o.lpa_update_blocked_nodes if blocked else mb.o.lpa_update_cleared_nodes)(lists[i])
            assert vo is None or int(vo) == v1 or int(vo) < 0, (mb.name, vo, v1)
    same(members, "blocked" if blocked else "cleared")
    return visited, lists


def subtree_all(members, rnd):
    ts, nxt = [], []
    for i, mb in enumerate(members):
        n_best = len(mb.s.lpa_best_child())
        t = 0 if n_best == 0 else min((i + rnd) % 3, max(n_best - 2, 0))
        ts.append(t if n_best else 7)  # any step for a planner without a trajectory
        nxt.append(mb.s.lpa_waypoint(t) if n_best else None)
    sizes = mp.MapPlanner.getSubStateSpaceBatch([mb.b.pl for mb in members], ts)
    for i, mb in enumerate(members):
        s1 = mb.s.lpa_get_sub_state_space(ts[i]) if nxt[i] is not None else mb.s.lpa_get_sub_state_space(0)
        assert sizes[i] == s1, (mb.name, sizes[i], s1)
        if mb.oracle_ok and nxt[i] is not None:
            if mb.o.lpa_get_sub_state_space(ts[i]) < 0:
                mb.oracle_ok = False
        if nxt[i] is not None:
            mb.s_wp = nxt[i]
    same(members, "subtree")
    return ts, sizes


# Flows left out of the fleet run alone in test_gpu_lpa.py / test_gpu_lpa_shaped.py.  The two jerk flows (76 657 and ~40 000
# nodes per plan) and the whole-map potential flows would hold gigabytes of host memory on the oracle's side at once (the oracle's
# first corridor_pot_yaw plan alone takes about 1 GiB), for no branch the members below do not take: corridor_pot_grad keeps the
# whole-map potential with a gradient term, simple_pot_local a local one, corridor_yaw / skir_jrk_yaw / skir_snp_yaw the yaw sessions.
BIG = ("skir_jrk", "corridor_jrk", "corridor_pot", "corridor_pot_restamp", "corridor_pot_yaw")


def fleet():
    members = [Member("flow", n) for n in lpa_flow.FLOWS if n not in BIG]
    members += [Member("shaped", n) for n in F.FLOWS if n not in BIG]
    members += [Member("fuzz", (seed, dim)) for dim in (2, 3) for seed in range(8)]
    return members


def test_fleet_lockstep_with_single_calls_and_oracle():
    members = fleet()
    no_goal = Member("flow", "corridor_acc")  # start in the goal region: no trajectory, no state to link
    no_goal.g_wp = no_goal.s_wp.copy()
    members.insert(3, no_goal)
    plan_all(members)
    assert not no_goal.traj
    saw_empty = saw_zero_ts = False
    for rnd in range(2):
        assert linked_all(members) > 0
        visited, lists = update_all(members, True, rnd)
        saw_empty = saw_empty or any(len(c) == 0 for c in lists)
        assert sum(visited) > 0
        plan_all(members)
        update_all(members, False, rnd)
        plan_all(members)
        ts, sizes = subtree_all(members, rnd)
        saw_zero_ts = saw_zero_ts or 0 in [t for t, mb in zip(ts, members) if mb.traj]
        assert sizes[3] == 0  # no trajectory
        plan_all(members)
    assert saw_empty and saw_zero_ts
    assert sum(mb.oracle_ok for mb in members) >= len(members) - 4


def test_launches_per_call_do_not_grow_with_the_fleet():
    def group(n):
        ms = [Member("flow", "skir_acc") for _ in range(n)]
        return ms

    counts = {}
    for n in (1, 32):
        ms = group(n)
        pls = [mb.b.pl for mb in ms]
        steps = []

        def step(fn):
            c0 = mp._lib.lib().mplb_launch_count()
            fn()
            steps.append(int(mp._lib.lib().mplb_launch_count() - c0))
        s, g = mp.waypoints_array(n), mp.waypoints_array(n)
        for i, mb in enumerate(ms):
            s[i], g[i] = mb.s_wp[0], mb.g_wp[0]
        step(lambda: mp.MapPlanner.planLPABatch(pls, s, g))
        step(lambda: mp.MapPlanner.getLinkedNodesBatch(pls))
        path = ms[0].b.lpa_best_child_states()[:, :3]
        cells = lpa_flow.cells_on_path(ms[0].m, 3, path[len(path) // 2:len(path) // 2 + 1], 2)
        for mb in ms:
            mb.maps[0].set_cells(cells, 100)
        step(lambda: mp.MapPlanner.updateBlockedNodesBatch(pls, [cells] * n))   # match arrays start empty: a regrow round
        step(lambda: mp.MapPlanner.planLPABatch(pls, s, g))
        step(lambda: mp.MapPlanner.getLinkedNodesBatch(pls))
        step(lambda: mp.MapPlanner.updateBlockedNodesBatch(pls, [cells] * n))   # arrays big enough now: no regrow
        step(lambda: mp.MapPlanner.getSubStateSpaceBatch(pls, [1] * n))
        counts[n] = steps
    assert counts[1] == counts[32], counts
    # the first update matches twice (its pair array grows), the second once
    assert counts[1][2] == counts[1][5] + 1, counts


def test_errors_leave_every_planner_untouched():
    members = [Member("flow", "skir_acc"), Member("flow", "corridor_acc")]
    plan_all(members)
    pls = [mb.b.pl for mb in members]
    before = [snap(mb.b) for mb in members]
    off = mp.MapPlanner(3)  # LPA* off
    off.setMapUtil(members[0].b.pl.map_util_)
    unplanned = Member("flow", "skir_acc").b.pl  # LPA* on, never planned
    cases = [pls + [pls[0]], pls + [off], pls + [unplanned]]
    for bad in cases:
        with pytest.raises(mp.MplbError):
            mp.MapPlanner.getLinkedNodesBatch(bad)
        with pytest.raises(mp.MplbError):
            mp.MapPlanner.updateBlockedNodesBatch(bad, [np.array([[1, 1, 1]])] * len(bad))
        with pytest.raises(mp.MplbError):
            mp.MapPlanner.getSubStateSpaceBatch(bad, [0] * len(bad))
    n_best = len(members[1].b.lpa_best_child())
    with pytest.raises(mp.MplbError):
        mp.MapPlanner.getSubStateSpaceBatch(pls, [0, n_best])
    with pytest.raises(mp.MplbError):
        mp.MapPlanner.getSubStateSpaceBatch(pls, [-1, 0])
    for mb, b in zip(members, before):
        a = snap(mb.b)
        lpa_flow.assert_same([b], [a], mb.name)
        assert a["cap"] == b["cap"]
