"""LPA* with a potential map and with yaw controls on the CPU side of the parity chain, over the flows of
tests/lpa_shaped_flow.py:
(1) the checker in libm trig mode equals the reference's OWN LPA* sources (oracle/_ref, where present) state by state, and
    reproduces the fixture recorded from them (tests/golden/lpa_shaped_flows.npz);
(2) the DEVICE core compiled for the host (tests/cpp/lpa_emul_shaped.cpp, both lane orders, tiny initial arrays so that it grows)
    equals the checker in its correctly rounded trig mode, tolerance 0; the potential-only flows also equal the fixture;
(3) the two trig definitions give the same statuses, pop counts and trajectories on the yaw flows, costs within 1e-9;
(4) each flow takes the branches it exists for (potential terms, FOV rejections, decreaseCost's cost without shaping terms,
    stale costs after a re-stamp, growth)."""
import os

import numpy as np
import pytest

import oracle
from oracle import ref
import lpa_flow
import lpa_shaped_flow as F

GOLD = os.path.join(os.path.dirname(__file__), "golden", "lpa_shaped_flows.npz")
SMALL = dict(init_cap=256, init_pred=2048)
_RUNS = {}


def _run(name, kind):
    if (name, kind) not in _RUNS:
        if kind == "libm":
            r = F.run_flow(name, oracle.OracleMap, F.OraclePlannerLibm)
        elif kind == "cr":
            r = F.run_flow(name, oracle.OracleMap, F.OraclePlanner)
        else:
            cm, cp = F.emu_classes(rev=kind == "emu_rev")
            r = F.run_flow(name, cm, cp, SMALL if kind == "emu" else dict(init_cap=512, init_pred=4096))
        if kind != "emu":  # only the host build's planner is probed later; the others would hold their state spaces
            r = (r[0], None)
        _RUNS[(name, kind)] = r
    return _RUNS[(name, kind)]


def _gold(name, snaps):
    gold = np.load(GOLD)[name]
    d = F.digest(snaps)
    assert len(d) == len(gold), name
    for f in gold.dtype.names:
        assert np.array_equal(d[f], gold[f]), (name, f)


@pytest.mark.parametrize("name", list(F.FLOWS))
def test_oracle_equals_reference_sources(name):
    a, _ = _run(name, "libm")
    if ref.available():
        b, _ = F.run_flow(name, ref.RefMap, ref.RefPlanner)
        lpa_flow.assert_same(a, b, name)
        _gold(name, b)  # the fixture is what the sources return today
    _gold(name, a)


@pytest.mark.parametrize("kind", ["emu", "emu_rev"])
@pytest.mark.parametrize("name", list(F.FLOWS))
def test_device_core_equals_oracle(name, kind):
    a, _ = _run(name, "cr")
    b, emu = _run(name, kind)
    lpa_flow.assert_same(a, b, name + " (device core, host build, " + kind + ")")
    if kind == "emu":
        assert emu.grows() >= 1, emu.grows()
    if name in F.POT_ONLY:
        _gold(name, b)


@pytest.mark.parametrize("name", F.YAW_FLOWS)
def test_yaw_flows_under_both_trig_definitions(name):
    """DESIGN 4.7: libm and correctly rounded sin / cos decide the same search on these flows"""
    a, _ = _run(name, "libm")
    b, _ = _run(name, "cr")
    assert len(a) == len(b)
    for x, y in zip(a, b):
        assert np.array_equal(x["best"], y["best"])
        assert len(x["nodes"]) == len(y["nodes"])
        if x["res"] is None:
            continue
        for f in ("status", "pops", "n_seg", "n_nodes", "pop_hash", "closed_hash"):
            assert x["res"][f] == y["res"][f], (name, f)
        cx, cy = float(x["res"]["cost"]), float(y["res"]["cost"])
        assert cx == cy or abs(cx - cy) <= 1e-9 * abs(cx), (name, cx, cy)


def _traj_states(name):
    """a fresh checker after the flow's first plan, and that plan's trajectory states"""
    f = F.FLOWS[name]
    m, mp_, pl, dim, start, goal = F.build(name, oracle.OracleMap, F.OraclePlanner)
    if f.get("pot"):
        pl.update_potential_map(np.r_[start, np.zeros(3 - dim)])
    r = pl.lpa_plan(F.waypoints(start, f["control"], f.get("start_yaw", 0.0)), F.waypoints(goal, f["control"], 0.0))
    assert int(r["status"]) in (0, 2), r
    if int(r["status"]) == 0:
        return pl, pl.lpa_best_child_states()
    st = np.zeros((1, 13))  # a capped plan has no trajectory: probe from the start
    st[0, :dim], st[0, 12] = start, f.get("start_yaw", 0.0)
    return pl, st


@pytest.mark.parametrize("name", F.POT_ONLY + ["corridor_pot_yaw"])
def test_potential_terms_are_taken(name):
    """successors along the planned trajectory carry a nonzero potential term: their cost drops when the potential map goes"""
    pl, states = _traj_states(name)
    control = F.FLOWS[name]["control"]
    with_pot = [pl.succ_trace(_wp(s, control)) for s in states]
    pl.set_potential_map(None)
    without = [pl.succ_trace(_wp(s, control)) for s in states]
    diff = sum(int(np.sum((a["verdict"] >= 3) & (b["verdict"] >= 3) & (a["cost"] != b["cost"]))) for a, b in zip(with_pot, without))
    assert diff > 0


def _wp(st, control):
    w = oracle.make_waypoints(1)
    w["pos"][0], w["vel"][0], w["acc"][0], w["jrk"][0], w["yaw"][0] = st[0:3], st[3:6], st[6:9], st[9:12], st[12]
    w["control"] = control
    return w


@pytest.mark.parametrize("name", F.YAW_FLOWS)
def test_fov_rejections_are_taken(name):
    """validate_yaw rejects controls that the base control's bounds accept (n_valid < n_prims beyond the plain rejections)"""
    pl, states = _traj_states(name)
    control = F.FLOWS[name]["control"]
    rej = [int(np.sum(pl.succ_trace(_wp(s, control))["verdict"] == 1)) for s in states]
    pl.set_param("yaw_max", -1)
    rej_plain = [int(np.sum(pl.succ_trace(_wp(s, control))["verdict"] == 1)) for s in states]
    assert sum(rej) > sum(rej_plain)


@pytest.mark.parametrize("name", ["corridor_pot", "corridor_pot_grad"])
def test_decrease_cost_restores_cost_without_shaping_terms(name):
    """after updateClearedNodes, some restored edge costs J + w dt while get_succ gives it the potential term too"""
    _, emu = _run(name, "emu")
    assert emu._cleared_mismatch > 0


def test_restamp_leaves_stored_costs_stale():
    _, emu = _run("corridor_pot_restamp", "emu")
    _, plain = _run("corridor_pot_grad", "emu")
    assert emu._cleared_mismatch > plain._cleared_mismatch


def test_capped_yaw_flow_grows():
    _, emu = _run("skir_jrk_yaw", "emu")
    assert emu.lpa_capacity()["grows"] > 0
