"""LPA* on the GPU (mplb_lpa.cu) over the seeded random replanning sequences of tests/test_oracle_lpa_fuzz.py: random 2D /
3D box maps, VEL / ACC / JRK / SNP, random control sets, bounds, epsilon and max_num; rounds of blocking cells near the
trajectory, clearing some of them, re-rooting and replanning.  After every step the device's whole state (result record,
hm_ in iteration order, the priority-queue array, best_child_, the linked points) equals the oracle's.  The oracle runs
first: a sequence ends where it detects a situation the reference leaves undefined (a plan that starts on an empty queue,
a re-root onto a stored successor that left the state space), before the device is asked.  A second test plans several
sequences' replanners at once through mplb_lpa_plan_batch and compares them with the same planners run one by one."""
import ctypes as C

import numpy as np
import pytest

import oracle
import mpl_ros_b200 as mp
from mpl_ros_b200 import _lib
import lpa_flow
from test_gpu_lpa import GpuMap, GpuPlanner
from test_oracle_lpa_fuzz import run_sequence, sequence_case

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("dim", [2, 3])
def test_lpa_sequences_match_oracle(dim, capsys):
    impls = [(oracle.OracleMap, oracle.OraclePlanner, {}), (GpuMap, GpuPlanner, {})]
    total = 0
    for seed in range(24):
        n, _ = run_sequence(seed, dim, impls)
        total += n
    with capsys.disabled():
        print("\nLPA* %dD: %d steps compared over 24 sequences" % (dim, total))
    assert total > 60, total  # as many steps as the host fuzz compares


def _planner(cm, cp, case, dim):
    nd, origin, res, data, ctl, U, prm, _, _, _ = case
    m = cm(origin, nd, data, res)
    m.free_unknown()
    p = cp(dim)
    p.set_map(m)
    for k, v in prm.items():
        p.set_param(k, v)
    p.set_controls(U)
    p._lpa_control = ctl
    return m, p


def _blocked_cells(case, path, dim):
    """a 3 x 3 patch of free cells around the middle of the trajectory, the start's own cell left free"""
    nd, origin, res, data, _, _, _, start, _, _ = case
    c = np.round((path[len(path) // 2, :dim] - origin) / res - 0.5).astype(int)
    cand = np.array([[c[0] + dx, c[1] + dy] + ([c[2]] if dim == 3 else []) for dx in (-1, 0, 1) for dy in (-1, 0, 1)])
    cand = cand[np.all((cand >= 0) & (cand < nd), axis=1)]
    lin = cand[:, 0] + nd[0] * cand[:, 1] + (nd[0] * nd[1] * cand[:, 2] if dim == 3 else 0)
    cand = cand[data.reshape(-1)[lin] != 100]
    sc = np.round((start - origin) / res - 0.5).astype(int)
    return cand[np.any(cand != sc, axis=1)]


@pytest.mark.parametrize("dim", [2, 3])
def test_lpa_batch_of_random_replanners(dim):
    """one CTA per replanner: the first plan and the replan after cells on each trajectory are blocked, for 8 random
    sequences at once, equal the same planners planned one by one, and the oracle."""
    seeds = range(8)
    cases = [sequence_case(seed, dim)[1] for seed in seeds]
    batched = [_planner(GpuMap, GpuPlanner, cs, dim) for cs in cases]
    single = [_planner(GpuMap, GpuPlanner, cs, dim) for cs in cases]
    orc = [_planner(oracle.OracleMap, oracle.OraclePlanner, cs, dim) for cs in cases]
    n = len(cases)
    s, g = mp.waypoints_array(n), mp.waypoints_array(n)
    for i, cs in enumerate(cases):
        _, _, _, _, ctl, _, _, start, goal, vel = cs
        s["pos"][i, :dim], g["pos"][i, :dim], s["vel"][i, :dim] = start, goal, vel
        s["control"][i] = g["control"][i] = ctl
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
            if not (ro["status"] == 3 and ro["pops"] == 0):  # an empty queue at the start of a plan: see mplb.h
                lpa_flow.assert_same([lpa_flow.snapshot(orc[i][1], ro)], [snap], ("batch vs oracle", dim, rnd, i))
                compared += 1
            ok.append(int(ro["status"]) == 0)
        if rnd == 0:
            assert sum(ok) >= 2, ok
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
