"""LPA* capacity paths on the host build of the device core (tests/cpp/lpa_emul.cpp) against the oracle, tolerance 0: the
exact fill that leaves no room for a new start node (and what the core did before the host made room for it), growth after a
re-root, and the trajectory longer than one launch's rows.  The host build checks after every call into the core that no
counter exceeded its capacity (EmuOverrun otherwise).  tests/test_gpu_lpa_capacity.py runs the same cases on the device."""
import numpy as np
import pytest

import oracle
import lpa_emul
import lpa_flow
import lpa_capacity_cases as K


class EmuLog(K.CapacityLog, lpa_emul.EmuPlanner):
    pass


@pytest.mark.parametrize("dim,seed,fill", K.EXACT_FILL)
def test_exact_fill_then_new_start(dim, seed, fill):
    case = K.fuzz_case(dim, seed)
    s, g = K.random_waypoints(case, dim)
    _, emu = K.random_planner(lpa_emul.EmuMap, EmuLog, case, dim, K.sizes(fill))
    _, orc = K.random_planner(oracle.OracleMap, oracle.OraclePlanner, case, dim)
    a = [lpa_flow.snapshot(orc, orc.lpa_plan(s, g))]
    b = [lpa_flow.snapshot(emu, emu.lpa_plan(s, g))]
    c = emu.cap_log[-1]
    assert c["grows"] == 0 and c["n_nodes_physical"] == c["cap_nodes"] == fill, c  # the last pop filled the arrays exactly
    s2 = K.off_lattice_start(s)
    assert not (a[0]["nodes"]["key"] == K.lattice_key(s2, dim)).all(axis=1).any()  # plan_begin has to create a node
    a.append(lpa_flow.snapshot(orc, orc.lpa_plan(s2, g)))
    b.append(lpa_flow.snapshot(emu, emu.lpa_plan(s2, g)))
    assert int(a[1]["res"]["status"]) != 1
    lpa_flow.assert_same(a, b, ("exact fill", dim, seed))
    c = emu.cap_log[-1]
    assert c["grows"] >= 1 and c["cap_nodes"] == fill << c["grows"], c


@pytest.mark.parametrize("dim,seed,fill", K.EXACT_FILL)
def test_exact_fill_without_room_for_the_start_overruns(dim, seed, fill):
    """the core alone, without the host's growth before a plan, writes the new start node past the arrays"""
    case = K.fuzz_case(dim, seed)
    s, g = K.random_waypoints(case, dim)
    _, emu = K.random_planner(lpa_emul.EmuMap, lpa_emul.EmuPlanner, case, dim, dict(K.sizes(fill), no_start_room=1))
    emu.lpa_plan(s, g)
    with pytest.raises(lpa_emul.EmuOverrun, match="plan_begin: n_nodes %d " % (fill + 1)):
        emu.lpa_plan(K.off_lattice_start(s), g)


def test_reroot_growth():
    name, nodes, preds = K.REROOT
    a, _ = lpa_flow.run_flow(name, oracle.OracleMap, oracle.OraclePlanner)
    b, emu = lpa_flow.run_flow(name, lpa_emul.EmuMap, EmuLog, K.sizes(nodes, preds))
    lpa_flow.assert_same(a, b, name)
    K.check_reroot_growth(emu.cap_log, nodes, 27)


@pytest.mark.parametrize("op,case", [("block", K.BLOCKED_GROWTH), ("clear", K.CLEARED_GROWTH)])
def test_replan_growth(op, case):
    name, nodes = case
    a, _ = lpa_flow.run_flow(name, oracle.OracleMap, oracle.OraclePlanner)
    b, emu = lpa_flow.run_flow(name, lpa_emul.EmuMap, EmuLog, K.sizes(nodes))
    lpa_flow.assert_same(a, b, name)
    K.check_first_growth_after(emu.cap_log, op)


def test_pred_only_growth():
    name, nodes, preds = K.PRED_ONLY
    a, _ = lpa_flow.run_flow(name, oracle.OracleMap, oracle.OraclePlanner)
    b, emu = lpa_flow.run_flow(name, lpa_emul.EmuMap, EmuLog, K.sizes(nodes, preds))
    lpa_flow.assert_same(a, b, name)
    K.check_pred_only_growth(emu.cap_log, nodes)


@pytest.mark.parametrize("n_seg", [K.SHORT_SEG, K.LONG_SEG])
def test_strip_trajectory(n_seg):
    """the long-trajectory case is what it claims: n_seg segments, the same actions and parent states as the oracle"""
    case = K.strip_case(n_seg)
    s, g = K.random_waypoints(case, 2)
    _, emu = K.random_planner(lpa_emul.EmuMap, lpa_emul.EmuPlanner, case, 2)
    _, orc = K.random_planner(oracle.OracleMap, oracle.OraclePlanner, case, 2)
    ro, re = orc.lpa_plan(s, g), emu.lpa_plan(s, g)
    lpa_flow.assert_same([lpa_flow.snapshot(orc, ro)], [lpa_flow.snapshot(emu, re)], ("strip", n_seg))
    assert int(ro["status"]) == 0 and int(ro["n_seg"]) == n_seg, ro
    acts = orc.lpa_actions()
    assert len(acts) == n_seg and np.array_equal(acts, emu.lpa_actions())
    assert np.array_equal(orc.lpa_best_child_states(), emu.lpa_best_child_states())
