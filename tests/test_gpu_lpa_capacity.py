"""LPA* capacity paths on the GPU (mplb_lpa.cu) against the oracle at tolerance 0: result records, hm_ in iteration order with
g / rhs / h / flags and the successor / predecessor list hashes, the heap array, best_child_ and the linked points
(lpa_flow.snapshot / assert_same).  The host code these cases reach runs only on the device path: ensure_capacity's per-array
prefixes, the key-table rebuild (k_lpa_rehash), the header and context re-uploads, the relaunch of a batch in which finished
sessions are skipped, getSubStateSpace's pool resize, the room made for a new start node, and the gather of trajectories longer
than one launch's rows.  Every case asserts through mplb_lpa_get_capacity (MapPlanner.lpaCapacity) that it took its branch, and
prints initial sizes, doublings and peak node / predecessor records.  The cases are in tests/lpa_capacity_cases.py; the host build
of the core runs the exact-fill and re-root ones in tests/test_oracle_lpa_capacity.py."""
import ctypes as C
import os
import time

import numpy as np
import pytest

import mpl_ros_b200 as mp
from mpl_ros_b200 import _lib
import oracle
import lpa_flow
import lpa_capacity_cases as K
from test_gpu_lpa import GpuMap, GpuPlanner
from test_gpu_lpa_fuzz import _blocked_cells

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden", "lpa_flows.npz")


class GpuCap(K.CapacityLog, GpuPlanner):
    def lpa_capacity(self):
        return self.pl.lpaCapacity()


def _report(capsys, what, nodes, preds, log):
    pn, pp = K.peak(log)
    with capsys.disabled():
        print("\n%-28s init nodes %6d preds %7s  grows %d  peak nodes %6d  peak preds %7d" %
              (what, nodes, preds if preds is not None else "2^20", log[-1]["grows"], pn, pp))


def _flow(name, nodes, preds=None):
    a, _ = lpa_flow.run_flow(name, oracle.OracleMap, oracle.OraclePlanner)
    b, gp = lpa_flow.run_flow(name, GpuMap, GpuCap, K.sizes(nodes, preds))
    lpa_flow.assert_same(a, b, (name, nodes, preds))
    return b, gp


@pytest.mark.parametrize("nodes", [128, 1000])
@pytest.mark.parametrize("name", list(lpa_flow.FLOWS))
def test_flows_from_small_arrays(name, nodes, capsys):
    """every flow from 128 / 1000 nodes (and 4x as many predecessor records): the oracle's states and the fixture's digests"""
    b, gp = _flow(name, nodes, 4 * nodes)
    gold = np.load(GOLD)[name]
    d = lpa_flow.digest(b)
    assert len(d) == len(gold)
    for f in gold.dtype.names:
        assert np.array_equal(d[f], gold[f]), (name, f)
    K.check_doublings(gp.cap_log, nodes)
    _report(capsys, "%s / %d" % (name, nodes), nodes, 4 * nodes, gp.cap_log)


@pytest.mark.parametrize("op,case", [("block", K.BLOCKED_GROWTH), ("clear", K.CLEARED_GROWTH)])
def test_growth_first_in_a_replan(op, case, capsys):
    name, nodes = case
    _, gp = _flow(name, nodes)
    K.check_first_growth_after(gp.cap_log, op)
    _report(capsys, "%s after %s" % (name, op), nodes, None, gp.cap_log)


def test_growth_after_reroot(capsys):
    name, nodes, preds = K.REROOT
    _, gp = _flow(name, nodes, preds)
    K.check_reroot_growth(gp.cap_log, nodes, 27)
    _report(capsys, "%s re-root" % name, nodes, preds, gp.cap_log)


def test_growth_driven_by_predecessors(capsys):
    name, nodes, preds = K.PRED_ONLY
    _, gp = _flow(name, nodes, preds)
    K.check_pred_only_growth(gp.cap_log, nodes)
    _report(capsys, "%s predecessors" % name, nodes, preds, gp.cap_log)


@pytest.mark.parametrize("dim,seed,fill", K.EXACT_FILL)
def test_exact_fill_then_new_start(dim, seed, fill, capsys):
    """the first plan's last pop fills the arrays exactly; the next plan starts off the lattice, so plan_begin creates a node
    and the host must have made room for it"""
    case = K.fuzz_case(dim, seed)
    s, g = K.random_waypoints(case, dim)
    _, gp = K.random_planner(GpuMap, GpuCap, case, dim, K.sizes(fill))
    _, orc = K.random_planner(oracle.OracleMap, oracle.OraclePlanner, case, dim)
    a = [lpa_flow.snapshot(orc, orc.lpa_plan(s, g))]
    b = [lpa_flow.snapshot(gp, gp.lpa_plan(s, g))]
    c = gp.cap_log[-1]
    assert c["grows"] == 0 and c["n_nodes_physical"] == c["cap_nodes"] == fill, c
    s2 = K.off_lattice_start(s)
    assert not (a[0]["nodes"]["key"] == K.lattice_key(s2, dim)).all(axis=1).any()
    a.append(lpa_flow.snapshot(orc, orc.lpa_plan(s2, g)))
    b.append(lpa_flow.snapshot(gp, gp.lpa_plan(s2, g)))
    assert int(a[1]["res"]["status"]) != 1
    lpa_flow.assert_same(a, b, ("exact fill", dim, seed))
    c = gp.cap_log[-1]
    assert c["grows"] >= 1 and c["cap_nodes"] == fill << c["grows"], c
    _report(capsys, "exact fill %dD seed %d" % (dim, seed), fill, None, gp.cap_log)


@pytest.mark.parametrize("dim", [2, 3])
def test_batch_sessions_grow_in_different_rounds(dim, capsys):
    """mplb_lpa_plan_batch over 8 random replanners whose arrays need 0, 1, 3 or 4 doublings: equal to planning them one by
    one and to the oracle, before and after cells on their trajectories are blocked"""
    cases = [K.fuzz_case(dim, seed) for seed, _ in K.BATCH[dim]]
    inits = []
    for cs, (seed, d) in zip(cases, K.BATCH[dim]):
        if d is None:
            inits.append(None)
            continue
        s, g = K.random_waypoints(cs, dim)
        _, orc = K.random_planner(oracle.OracleMap, oracle.OraclePlanner, cs, dim)
        orc.lpa_plan(s, g)
        n_first = len(orc.lpa_nodes())
        assert n_first >> d >= 128, (seed, n_first)
        inits.append(n_first >> d)
    assert len({len(cs[5]) for cs in cases}) == 2  # two control-set sizes in the batch
    extra = [K.sizes(i) if i else None for i in inits]
    batched = [K.random_planner(GpuMap, GpuPlanner, cs, dim, e) for cs, e in zip(cases, extra)]
    single = [K.random_planner(GpuMap, GpuPlanner, cs, dim, e) for cs, e in zip(cases, extra)]
    orc = [K.random_planner(oracle.OracleMap, oracle.OraclePlanner, cs, dim) for cs in cases]
    n = len(cases)
    s, g = mp.waypoints_array(n), mp.waypoints_array(n)
    for i, cs in enumerate(cases):
        si, gi = K.random_waypoints(cs, dim)
        s[i], g[i] = si[0], gi[0]
    handles = (C.c_void_p * n)(*[p.pl._h for _, p in batched])
    compared = 0
    for rnd in range(2):
        res = np.zeros(n, dtype=_lib.RESULT_DTYPE)
        _lib.check(_lib.lib().mplb_lpa_plan_batch(handles, n, _lib.ptr(s), _lib.ptr(g), _lib.ptr(res)))
        ok = []
        for i in range(n):
            r1 = single[i][1].lpa_plan(s[i:i + 1], g[i:i + 1])
            ro = orc[i][1].lpa_plan(s[i:i + 1], g[i:i + 1])
            snap = lpa_flow.snapshot(batched[i][1], res[i])
            lpa_flow.assert_same([lpa_flow.snapshot(single[i][1], r1)], [snap], ("batch vs single", dim, rnd, i))
            assert batched[i][1].pl.lpaCapacity() == single[i][1].pl.lpaCapacity(), (dim, rnd, i)
            if not (ro["status"] == 3 and ro["pops"] == 0):
                lpa_flow.assert_same([lpa_flow.snapshot(orc[i][1], ro)], [snap], ("batch vs oracle", dim, rnd, i))
                compared += 1
            if int(res[i]["status"]) == 0:
                assert np.array_equal(batched[i][1].pl.getActions(), orc[i][1].lpa_actions()), (dim, rnd, i)
            ok.append(int(ro["status"]) == 0)
        if rnd == 0:
            grows = [p.pl.lpaCapacity()["grows"] for _, p in batched]
            for (seed, d), gr in zip(K.BATCH[dim], grows):
                assert gr == 0 if d is None else gr >= d, (seed, d, gr)
            assert len(set(grows)) >= 3, grows  # the sessions finished in different relaunch rounds
            with capsys.disabled():
                print("\nbatch %dD: init nodes %s, grows %s" % (dim, [i or 65536 for i in inits], grows))
            for i in range(n):
                if not ok[i]:
                    continue
                cells = _blocked_cells(cases[i], orc[i][1].lpa_best_child_states(), dim)
                if len(cells) == 0:
                    continue
                for m, p in (batched[i], single[i], orc[i]):
                    m.set_cells(cells, 100)
                    p.lpa_update_blocked_nodes(cells)
    assert compared >= n + 2


def _check_trajectory(gp, orc, n_seg):
    """getActions, getSegStates, getTraj's primitives and best_child_ over all n_seg segments"""
    acts, states = orc.lpa_actions(), orc.lpa_best_child_states()
    assert len(acts) == n_seg and len(states) == n_seg + 1
    assert np.array_equal(gp.pl.getActions(), acts)
    assert np.array_equal(gp.pl.getSegStates(), states[:-1])
    bc = gp.pl.lpaBestChild()
    assert np.array_equal(bc["key"], orc.lpa_best_child()) and np.array_equal(bc["state"], states)
    U = gp.pl.U_
    prims = gp.pl.getTraj().getPrimitives()
    assert len(prims) == n_seg
    want = np.array([mp.Primitive(2, mp.VEL, states[i], U[acts[i]], K.STRIP_DT).coeffs for i in range(n_seg)])
    assert np.array_equal(np.array([p.coeffs for p in prims]), want)


@pytest.mark.parametrize("n_seg", [K.SHORT_SEG, K.LONG_SEG])
def test_long_trajectory(n_seg, capsys):
    """a 2D VEL plan of n_seg segments (dt = 0.01 s along a free strip) through plan() and through mplb_lpa_plan_batch"""
    case = K.strip_case(n_seg)
    s, g = K.random_waypoints(case, 2)
    _, orc = K.random_planner(oracle.OracleMap, oracle.OraclePlanner, case, 2)
    ro = orc.lpa_plan(s, g)
    assert int(ro["status"]) == 0 and int(ro["n_seg"]) == n_seg, ro
    _, gp = K.random_planner(GpuMap, GpuPlanner, case, 2)
    t0 = time.perf_counter()
    r = gp.lpa_plan(s, g)
    ms = (time.perf_counter() - t0) * 1e3
    lpa_flow.assert_same([lpa_flow.snapshot(orc, ro)], [lpa_flow.snapshot(gp, r)], ("strip", n_seg))
    _check_trajectory(gp, orc, n_seg)
    # the same plan for two replanners in one launch: the strip and a 4000-segment companion
    comp = K.strip_case(4000)
    cs, cg = K.random_waypoints(comp, 2)
    _, oc = K.random_planner(oracle.OracleMap, oracle.OraclePlanner, comp, 2)
    oc.lpa_plan(cs, cg)
    pair = [K.random_planner(GpuMap, GpuPlanner, case, 2)[1], K.random_planner(GpuMap, GpuPlanner, comp, 2)[1]]
    sb, gb = mp.waypoints_array(2), mp.waypoints_array(2)
    sb[0], gb[0], sb[1], gb[1] = s[0], g[0], cs[0], cg[0]
    res = np.zeros(2, dtype=_lib.RESULT_DTYPE)
    handles = (C.c_void_p * 2)(*[p.pl._h for p in pair])
    _lib.check(_lib.lib().mplb_lpa_plan_batch(handles, 2, _lib.ptr(sb), _lib.ptr(gb), _lib.ptr(res)))
    for f in ("status", "n_seg", "cost", "pops", "n_nodes", "pop_hash", "closed_hash"):
        assert res[0][f] == r[f], f
    for p, o, k in ((pair[0], orc, n_seg), (pair[1], oc, 4000)):
        assert np.array_equal(p.pl.getActions(), o.lpa_actions()) and len(p.pl.getActions()) == k
        assert np.array_equal(p.pl.getSegStates(), o.lpa_best_child_states()[:-1])
    with capsys.disabled():
        print("\nLPA* strip %d segments: %d pops, plan() %.1f ms on one warp (host clock, includes the result copies)"
              % (n_seg, int(r["pops"]), ms))
