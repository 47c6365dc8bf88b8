"""Seeded random comparison of the CUDA path with the oracle over every astar_batch_kernel instantiation (16 plain: dim
{2, 3} x VEL / ACC / JRK / SNP x |U| <= 32 / > 32; 8 shaped: potential map, search region and / or yaw controls, |U| <= 32).
The cases come from tests/fuzz_cases.py (random box maps with unknown cells, non-dyadic resolutions and origins up to 5e6 m,
every epsilon class, tolerances, max_num, start velocities; the oracle itself is fuzzed against the reference's own sources
in tests/test_oracle_fuzz_vs_reference.py).  Per case, all exact (tolerance 0):
  - one single plan: the result record, the popped keys in order, every node (stored state, g, h, opened, closed), the
    actions and segment states;
  - plain cells: the get_succ rows of mplb_expand (expand_trace_kernel) on every popped state against the oracle's;
  - one batch of 16..64 queries on the same map with a small max_seg: result records and action rows against the oracle's
    batch, segment states against single oracle plans;
  - the batch's planning_ros_msgs/Trajectory bytes against test_gpu_wire.py's serialiser fed with the oracle's plans
    (None for a truncated plan);
  - the batch refined by mplb_refine_trajectories (gather kernel + TrajSolver) for the VEL, ACC and JRK refine controls
    against oracle.traj_solve on the waypoints built from the oracle's plans (map_planner_node.cpp:216-227).
MPLB_GPU_FUZZ_CASES=<n> runs n seeds per cell instead of 4.  The last test prints one row per instantiation."""
import collections
import os
import time

import numpy as np
import pytest

import oracle
import mpl_ros_b200 as mp
import fuzz_cases as F
from helpers_gpu import assert_results_equal
from test_gpu_filters import TRACE_FIELDS
from test_gpu_wire import _ros_trajectory_bytes
from test_gpu_yaw import _full_compare

pytestmark = pytest.mark.gpu

SEEDS = int(os.environ.get("MPLB_GPU_FUZZ_CASES", "4"))
REFINE_CONTROLS = (mp.VEL, mp.ACC, mp.JRK)
STATS = {}    # cell -> Counter(plans, ok, met_obstacle)
COUNTS = collections.Counter()  # comparisons per part


def _tally(st, res):
    res = np.atleast_1d(res)
    st["plans"] += len(res)
    st["ok"] += int((res["status"] == 0).sum())
    st["met_obstacle"] += int((res["n_valid"] < res["n_prims"]).sum())


def _single(c, pl, op, st, ctx):
    sg, so = c.waypoints(c.start, vel=c.vel, yaw=c.yaw)
    gg, go = c.waypoints(c.goal)
    rg = _full_compare(pl, op, sg, gg, so, go, ctx, 3 * F.ORDER_OF_CONTROL[c.control & 15])
    _tally(st, rg)
    COUNTS["single plans"] += 1
    return rg, so


def _expand(c, pl, op, rg, so, ctx):
    """get_succ rows on every popped state (on the start when nothing was popped)."""
    if rg["pops"] > 0:
        states = pl.getNodes()["state"][pl.getPopLog()]
        w = mp.waypoints_array(len(states))
        w["pos"], w["vel"], w["acc"], w["jrk"], w["yaw"] = (states[:, 0:3], states[:, 3:6], states[:, 6:9], states[:, 9:12],
                                                            states[:, 12])
        w["control"] = c.control
    else:
        w = so.copy()
    rows = pl.expand(w)
    for i in range(len(w)):
        tr = op.succ_trace(w[i:i + 1])
        for f in TRACE_FIELDS:
            assert np.array_equal(rows[i][f], tr[f]), (ctx, "expand", i, f, rows[i][f], tr[f])
    COUNTS["expand rows"] += rows.size


def _refine_waypoints(c, op, acts, segs, ns):
    """map_planner_node.cpp:216-227: the trajectory's waypoints (segment start states, then the last primitive evaluated
    at dt, taken from the oracle's get_succ row of the last parent), interior ones VEL, the two ends the plan control."""
    d = c.dim
    w = oracle.make_waypoints(ns + 1)
    ends = np.vstack([segs[:ns], op.succ_trace(_state_waypoint(c, segs[ns - 1]))[acts[ns - 1]]["succ"]])
    for j, st in enumerate(ends):
        w["pos"][j, :d], w["vel"][j, :d], w["acc"][j, :d], w["jrk"][j, :d] = st[0:d], st[3:3 + d], st[6:6 + d], st[9:9 + d]
        w["yaw"][j] = st[12]
    w["control"] = mp.VEL
    w["control"][0] = w["control"][ns] = c.control
    return w


def _state_waypoint(c, st):
    w = oracle.make_waypoints(1)
    w["pos"][0], w["vel"][0], w["acc"][0], w["jrk"][0], w["yaw"][0] = st[0:3], st[3:6], st[6:9], st[9:12], st[12]
    w["control"] = c.control
    return w


def _batch(c, pl, op, st, seed, ctx):
    sg, gg, so, go = c.batch_waypoints(seed)
    n, max_seg, dt = len(sg), c.max_seg, c.params["dt"]
    rg, ag, segs = pl.plan_batch(sg, gg, max_seg=max_seg, want_states=True)
    ro, ao = op.plan_batch(so, go, nthreads=8, max_seg=max_seg)
    for i in range(n):
        assert_results_equal(rg[i], ro[i], (ctx, "batch", i))
    assert np.array_equal(ag, ao), (ctx, "batch actions")
    _tally(st, rg)
    COUNTS["batch plans"] += n

    z = 0.25 if c.dim == 2 else 0.0
    msgs = pl.serialize_trajectories(rg, ag, segs, z=z, frame_id="map", seq=7, stamp=(12, 345))
    refined = {rc: pl.refine_trajectories(rg, ag, segs, c.control, rc) for rc in REFINE_CONTROLS}
    ncol = 3 * F.ORDER_OF_CONTROL[c.control & 15]
    for i in range(n):
        r1 = op.plan(so[i:i + 1], go[i:i + 1])
        assert_results_equal(r1, ro[i], (ctx, "single oracle plan of batch entry", i))
        ns = int(r1["n_seg"]) if r1["status"] == 0 else 0
        acts, states = (op.actions(ns), op.seg_states(ns)) if ns else (np.zeros(0, np.int32), np.zeros((0, 13)))
        kept = ns <= max_seg
        if ns and kept:
            assert np.array_equal(segs[i, :ns, :ncol], states[:, :ncol]) and np.array_equal(segs[i, :ns, 12], states[:, 12]), \
                (ctx, "batch segment states", i)
        if kept:
            exp = _ros_trajectory_bytes(c.dim, c.control, acts, states, c.U, dt, z, "map", 7, (12, 345))
            assert msgs[i] == exp, (ctx, "wire", i)
        else:
            assert msgs[i] is None, (ctx, "wire of a truncated plan", i)
        COUNTS["wire messages"] += 1
        good = ns >= 1 and kept
        want_w = _refine_waypoints(c, op, acts, states, ns) if good else None
        for rc, (coefs, nseg) in refined.items():
            assert nseg[i] == (ns if good else 0), (ctx, "refine n_segs", rc, i)
            if not good:
                assert not coefs[i].any(), (ctx, "refine of a failed / truncated plan", rc, i)
                continue
            want = oracle.traj_solve(c.dim, rc, want_w, np.full(ns, dt))
            assert np.array_equal(coefs[i, :ns], want), (ctx, "refine", rc, i)
            assert not coefs[i, ns:].any(), (ctx, "refine tail", rc, i)
            COUNTS["refined trajectories"] += 1


def run_cell(cell):
    st = STATS[cell] = collections.Counter()
    t0 = time.perf_counter()
    for seed in range(SEEDS):
        c = F.make_case(cell, seed)
        assert c.cell == cell
        ctx = (F.cell_name(cell), seed)
        pl, op = c.build()
        rg, so = _single(c, pl, op, st, ctx)
        if not c.shaped:
            _expand(c, pl, op, rg, so, ctx)
        _batch(c, pl, op, st, seed, ctx)
    st["seconds"] = time.perf_counter() - t0


@pytest.mark.parametrize("cell", F.CELLS, ids=F.cell_name)
def test_instantiation_matches_oracle(cell):
    run_cell(cell)


def test_every_instantiation_ran(capsys):
    """Runs whatever cell the selection left out, prints the table, and asserts that every instantiation planned,
    found paths and met obstacles."""
    for cell in F.CELLS:
        if cell not in STATS:
            run_cell(cell)
    lines = ["%-24s %6s %6s %9s %7s" % ("astar_batch_kernel", "plans", "ok", "obstacle", "secs")]
    for cell in F.CELLS:
        s = STATS[cell]
        lines.append("%-24s %6d %6d %9d %7.1f" % (F.cell_name(cell), s["plans"], s["ok"], s["met_obstacle"], s["seconds"]))
    lines.append("comparisons: " + ", ".join("%s %d" % kv for kv in sorted(COUNTS.items())))
    with capsys.disabled():
        print("\n" + "\n".join(lines))
    bad = [F.cell_name(c) for c in F.CELLS if not (STATS[c]["plans"] > 0 and STATS[c]["ok"] > 0 and STATS[c]["met_obstacle"] > 0)]
    assert not bad, bad
