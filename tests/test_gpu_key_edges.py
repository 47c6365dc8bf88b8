"""The search kernel at the edges of its configuration, against the oracle with tolerance 0 (cases: key_edge_cases.py):
  - wide lattice keys (more than 96 bits: hash-table slots also compare the row's second key word) on 3D SNP, plain with
    both |U| classes and shaped with yaw, next to a 96-bit key;
  - the exact collision-sampling path (use_fast == 0) on all 16 plain instantiations, through each of its triggers, next
    to cases just inside them; up to 4096 sample divisors;
  - starts and goals outside the packable key range (unwrapped yaws; velocity, acceleration, jerk above their bound), 2D
    and 3D, plain and shaped, single plans and batches mixed with in-range queries.
Every case first asserts that the branch it is meant to cover is the one the library configured (mplb_planner_key_layout
against the restatement in key_edge_cases.py).  Per case:
  - single plans: the result record, the popped keys in order, every node (key, stored state, g, h, flags), actions and
    segment states (_full_compare of test_gpu_yaw.py);
  - plain cases: the get_succ rows of every popped state (mplb_expand);
  - one batch: result records and action rows against the oracle's batch, segment states against single oracle plans.
The last test prints one row per (instantiation, branch) and asserts that each planned, found paths and met obstacles."""
import collections
import time

import numpy as np
import pytest

import mpl_ros_b200 as mp
import key_edge_cases as K
from fuzz_cases import cell_name
from helpers_gpu import assert_results_equal
from test_gpu_fuzz import _expand, _tally
from test_gpu_yaw import _full_compare

pytestmark = pytest.mark.gpu

STATS = collections.defaultdict(collections.Counter)  # (instantiation, branch) -> plans, ok, met_obstacle
GROUPS = {"wide": K.wide_cases, "exact": K.exact_cases, "out_of_range": K.oor_cases}
RAN = set()
KEY_RANGE = 7  # MPLB_PLAN_KEY_RANGE


def _check_layout(c, pl, ctx):
    order = K.order_of(c.control)
    _, bits = K.key_layout(c.dim, order, c.map, c.params, c.U, c.shaped, bool(c.control & 16))
    want = dict(key_bits=bits, key_wide=int(bits > 96), use_fast=K.sampler(c.dim, order, c.map, c.params, c.U)["use_fast"])
    got = pl.key_layout(c.control)
    assert got == want, (ctx, got, want)
    return got


def _wide_merges(c, op, ro):
    """Some distinct nodes of the oracle's plan agree on k0 and the low 32 bits of k1: a wide compare that dropped the
    row header would merge them."""
    fields, _ = K.key_layout(c.dim, K.order_of(c.control), c.map, c.params, c.U, c.shaped, bool(c.control & 16))
    seen = collections.defaultdict(set)
    for n in op.nodes(ro["n_nodes"]):
        k0, k1 = K.pack(fields, [int(v) for v in n["key"][:n["key"][15]]])
        seen[(k0, k1 & 0xffffffff)].add(k1)
    return sum(len(v) > 1 for v in seen.values())


def _waypoints(c, pos, fields_list):
    """(GPU, oracle) waypoints at pos with the per-row field overrides of fields_list (None: none)."""
    sg, so = K.state_waypoints(c, pos)
    for i, f in enumerate(fields_list):
        for k, v in (f or {}).items():
            for w in (sg, so):
                if k == "yaw":
                    w["yaw"][i] = v
                else:
                    w[k][i, :c.dim] = v
    return sg, so


def _batch(c, pl, op, st, batch, ctx):
    S, G = c.queries(c.n_batch, c.seed + 100)
    if c.near_goals:
        G = S + np.eye(c.dim)[0] * 0.7
    n = len(S)
    sf = [batch[0][(i // 2) % len(batch[0])] if (batch and i % 2 == 0) else None for i in range(n)]
    gf = [batch[1][(i // 3) % len(batch[1])] if (batch and i % 3 == 0) else None for i in range(n)]
    sg, so = _waypoints(c, S, sf)
    gg, go = _waypoints(c, G, gf)
    rg, ag, segs = pl.plan_batch(sg, gg, max_seg=c.max_seg, want_states=True)
    ro, ao = op.plan_batch(so, go, nthreads=8, max_seg=c.max_seg)
    for i in range(n):
        assert_results_equal(rg[i], ro[i], (ctx, "batch", i))
    assert np.array_equal(ag, ao), (ctx, "batch actions")
    ncol = 3 * K.order_of(c.control)
    for i in range(n):
        ns = int(ro[i]["n_seg"]) if ro[i]["status"] == 0 else 0
        if ns and ns <= c.max_seg:
            op.plan(so[i:i + 1], go[i:i + 1])
            want = op.seg_states(ns)
            assert np.array_equal(segs[i, :ns, :ncol], want[:, :ncol]) and np.array_equal(segs[i, :ns, 12], want[:, 12]), \
                (ctx, "batch segment states", i)
    _tally(st, rg)
    return rg


def run_group(group):
    t0 = time.perf_counter()
    for name, branch, c, singles, batch in GROUPS[group]():
        inst = cell_name(c.cell)
        ctx = (inst, name)
        st = STATS[(inst, branch)]
        pl, op = c.build()
        layout = _check_layout(c, pl, ctx)
        assert layout["key_wide"] == (branch == "wide") or group != "wide", (ctx, layout)
        assert (layout["use_fast"] == 0) == branch.startswith("exact") or group != "exact", (ctx, layout)
        ns = 3 * K.order_of(c.control)
        for sfl, gfl in singles:
            sg, so = _waypoints(c, c.start, [sfl])
            gg, go = _waypoints(c, c.goal, [gfl])
            rg = _full_compare(pl, op, sg, gg, so, go, ctx + (sfl, gfl), ns)
            assert rg["status"] != KEY_RANGE, ctx
            _tally(st, rg)
            if not c.shaped:
                _expand(c, pl, op, rg, so, ctx)
            if branch == "wide":
                st["merge_pairs"] += _wide_merges(c, op, rg)
        _batch(c, pl, op, st, batch, ctx)
    RAN.add(group)
    STATS[("seconds", group)]["plans"] = int(time.perf_counter() - t0)


@pytest.mark.parametrize("group", list(GROUPS))
def test_key_edges_match_oracle(group):
    run_group(group)


def test_out_of_range_errors():
    """One step past the largest sample divisor, and a shaped plan that needs the exact sampling path, fail loudly with
    MPLB_ERR_ARG; a start the reference's (int)std::round cannot represent still ends with KEY_RANGE."""
    for c, what in ((K.too_many_samples_case(), "4096 samples"), (K.shaped_exact_case(), "positive dynamic bounds")):
        pl, _ = c.build()
        sg, _ = K.state_waypoints(c, c.start)
        gg, _ = K.state_waypoints(c, c.goal)
        for call in (lambda: pl.key_layout(c.control), lambda: pl.plan(sg, gg)):
            with pytest.raises(mp.MplbError, match="mplb error -1: .*" + what):
                call()
    c = K.oor_cases()[3][2]  # 2D ACC
    pl, _ = c.build()
    sg, _ = K.state_waypoints(c, c.start, vel=np.eye(2)[0] * 3e8)
    gg, _ = K.state_waypoints(c, c.goal)
    pl.plan(sg, gg)
    assert pl.result()["status"] == KEY_RANGE


def test_every_branch_ran(capsys):
    for group in GROUPS:
        if group not in RAN:
            run_group(group)
    lines = ["%-22s %-26s %6s %6s %9s %6s" % ("astar_batch_kernel", "branch", "plans", "ok", "obstacle", "merges")]
    keys = sorted(k for k in STATS if k[0] != "seconds")
    for k in keys:
        s = STATS[k]
        lines.append("%-22s %-26s %6d %6d %9d %6s" % (k[0], k[1], s["plans"], s["ok"], s["met_obstacle"],
                                                       s["merge_pairs"] if k[1] == "wide" else "-"))
    lines.append("seconds: " + ", ".join("%s %d" % (g, STATS[("seconds", g)]["plans"]) for g in GROUPS))
    with capsys.disabled():
        print("\n" + "\n".join(lines))
    bad = [k for k in keys if not (STATS[k]["plans"] > 0 and STATS[k]["ok"] > 0 and STATS[k]["met_obstacle"] > 0)]
    assert not bad, bad
    assert all(STATS[k]["merge_pairs"] > 0 for k in keys if k[1] == "wide"), [(k, STATS[k]["merge_pairs"]) for k in keys]
