"""GPU parity tests: the CUDA path (through the C ABI) against the oracle, bit-exact.

Bar (BASELINE.json north_star): identical voxel indices / free-occupied decisions and expanded-node sets;
costs and waypoint states are compared for exact equality here (tolerance 0), which is stricter than the
1e-6 relative the north_star allows.
"""
import numpy as np
import pytest

import oracle
import mpl_ros_b200 as mp
from mpl_ros_b200 import maps
from helpers import load_config
from helpers_gpu import RESULT_FIELDS, assert_results_equal, make_pair, waypoint_pair

pytestmark = pytest.mark.gpu


def _nodes_by_key(nodes):
    return {tuple(n["key"][:n["key"][15]]): n for n in nodes}


@pytest.mark.parametrize("name", ["corridor", "simple", "skir"])
def test_single_plan_parity(name):
    """Reference-shaped single plans: test_planner_2d.cpp (corridor KAT), map_planner_node test.launch (simple),
    test.launch.skir (skir).  Everything observable is compared: counters, pop order, every node, the trajectory."""
    m, dim, params, U, start, goal = load_config(name)
    pl, op = make_pair(m, dim, params, U)
    sg, so = waypoint_pair(start, mp.ACC)
    gg, go = waypoint_pair(goal, mp.ACC)
    ok = pl.plan(sg, gg)
    ro = op.plan(so, go)
    rg = pl.result()
    assert ok and ro["status"] == 0
    assert_results_equal(rg, ro, name)
    if name == "corridor":  # MPL/README.md:200-202
        assert rg["n_closed"] == 615 and rg["n_seg"] == 35 and rg["cost"] == 351.5
    # pop order = expanded_nodes_ order (env_map.h:154)
    gn = pl.getNodes()
    pop_keys_gpu = gn["key"][pl.getPopLog()]
    assert np.array_equal(pop_keys_gpu, op.pop_keys(ro["pops"]))
    # every node of the hash map: stored coord (first discoverer), g, h, flags
    on = _nodes_by_key(op.nodes(ro["n_nodes"]))
    gnk = _nodes_by_key(gn)
    assert set(on) == set(gnk)
    for k, a in gnk.items():
        b = on[k]
        # only the derivatives the control mode uses are part of the node (waypoint.h:46-55); the reference also
        # carries acc = u in the stored coord but nothing on the path reads it
        assert np.array_equal(a["state"][:6], b["state"][:6]), k
        assert a["g"] == b["g"] and a["h"] == b["h"] and a["opened"] == b["opened"] and a["closed"] == b["closed"], k
    # trajectory: actions and the stored parent states (forward_action arguments, env_base.h:228-231)
    assert np.array_equal(pl.getActions(), op.actions(ro["n_seg"]))
    assert np.array_equal(pl.getSegStates()[:, :6], op.seg_states(ro["n_seg"])[:, :6])
    # reference-style getters
    assert len(pl.getCloseSet()) == ro["n_closed"] and len(pl.getOpenSet()) == ro["n_open"]
    traj = pl.getTraj()
    assert traj.getTotalTime() == ro["n_seg"] * params["dt"]
    assert len(traj.getWaypoints()) == ro["n_seg"] + 1
    # debug getters rebuilt from the pop log: finite-cost primitives of all expanded nodes (planner_base.h:30-74,143-145)
    edges = pl.getExpandedEdges()
    assert len(edges) == ro["n_valid"] == len(pl.getValidPrimitives())
    mu = pl._keep[0]
    assert len(mu.getCloud()) == int((mu.getMap() == 100).sum())
    pl.reset()
    assert not pl.initialized()


@pytest.mark.parametrize("name", ["corridor", "simple", "skir"])
def test_expand_trace_parity(name):
    """env_map::get_succ row by row (verdict, sample divisor, samples tested, blocking voxel index, cost, end
    state, lattice key) on every state the oracle's search touched."""
    m, dim, params, U, start, goal = load_config(name)
    pl, op = make_pair(m, dim, params, U)
    sg, so = waypoint_pair(start, mp.ACC)
    gg, go = waypoint_pair(goal, mp.ACC)
    ro = op.plan(so, go)
    nodes = op.nodes(ro["n_nodes"])[:600]
    sts_g, sts_o = waypoint_pair(nodes["state"][:, 0:dim], mp.ACC, vel=nodes["state"][:, 3:3 + dim])
    rows = pl.expand(sts_g)
    for i in range(len(nodes)):
        tr = op.succ_trace(sts_o[i:i + 1])
        for f in ("verdict", "n", "n_tested", "block_idx", "cost", "succ", "key"):
            assert np.array_equal(rows[i][f], tr[f]), (name, i, f, rows[i][f], tr[f])


def _levine_case(which):
    m = maps.levine256() if which == "levine256" else maps.load_fixture("levine")
    U = maps.make_U(1.0, 1, 3)
    params = dict(v_max=2.0, a_max=1.0, dt=1.0, tol_pos=0.5)
    return m, U, params


@pytest.mark.parametrize("which,n", [("levine", 48), ("levine256", 48)])
def test_batch_parity_levine(which, n):
    """BASELINE configs[1] shape (3D, |U| = 27, random free-voxel start/goal pairs, unreachable pairs kept)."""
    m, U, params = _levine_case(which)
    pl, op = make_pair(m, 3, params, U)
    S, G = maps.sample_queries(m, n, seed=0)
    sg, so = waypoint_pair(S, mp.ACC)
    gg, go = waypoint_pair(G, mp.ACC)
    rg, ag, segs = pl.plan_batch(sg, gg, max_seg=64, want_states=True)
    ro, ao = op.plan_batch(so, go, nthreads=8, max_seg=64)
    assert set(np.unique(ro["status"])) <= {0, 3}
    for i in range(n):
        assert_results_equal(rg[i], ro[i], (which, i))
    assert np.array_equal(ag, ao)


def test_edge_cases():
    m, dim, params, U, start, goal = load_config("simple")
    pl, op = make_pair(m, dim, params, U)
    free = m.int_to_float([145, 45, 0])
    # occupied start -> "start is not free" (planner_base.h:283-287)
    occ_idx = int(np.flatnonzero(m.data == 100)[1000])
    d = m.dim.astype(np.int64)
    occ = m.int_to_float([occ_idx % d[0], (occ_idx // d[0]) % d[1], occ_idx // (d[0] * d[1])])
    cases = [(occ, goal, 1), ([-5.0, 0.0, 0.0], goal, 1),          # occupied / outside start
             (free, free + 0.2, 5),                                   # start already in the goal region (graph_search.h:44)
             (start, goal, 0)]
    for s, g, want in cases:
        sg, so = waypoint_pair(s, mp.ACC)
        gg, go = waypoint_pair(g, mp.ACC)
        ok = pl.plan(sg, gg)
        ro = op.plan(so, go)
        assert ro["status"] == want, (s, g, ro["status"])
        assert_results_equal(pl.result(), ro)
        assert ok == (want in (0, 5))
    # MaxExpandStep (graph_search.h:149-154)
    pl.setMaxNum(50)
    op.set_param("max_num", 50)
    sg, so = waypoint_pair(start, mp.ACC)
    gg, go = waypoint_pair(goal, mp.ACC)
    assert not pl.plan(sg, gg)
    ro = op.plan(so, go)
    assert ro["status"] == 2 and ro["pops"] == 50
    assert_results_equal(pl.result(), ro)


def test_nonzero_start_velocity_and_epsilon():
    m, dim, params, U, start, goal = load_config("skir")
    for eps in (1.0, 2.0, 0.0):
        p2 = dict(params, epsilon=eps)
        pl, op = make_pair(m, dim, p2, U)
        sg, so = waypoint_pair(start, mp.ACC, vel=[1.0, 0.0, 0.0])
        gg, go = waypoint_pair(goal, mp.ACC)
        pl.plan(sg, gg)
        ro = op.plan(so, go)
        assert_results_equal(pl.result(), ro, eps)
        # eps = 2 re-opens closed nodes: the predecessor log (MPLB_EXACT_PREDS, automatic for eps > 1) makes recoverTraj
        # resolve every predecessor with its final g, like graph_search.h:391-405
        assert np.array_equal(pl.getActions(), op.actions(ro["n_seg"])), eps
        # the stored coord keeps the derivatives below the control order (ACC: pos, vel); the oracle also carries acc = u
        assert np.array_equal(pl.getSegStates()[:, :6], op.seg_states(ro["n_seg"])[:, :6]), eps


def test_epsilon_gt1_trajectories_batch():
    """Weighted A* (eps = 2 and 3.5, closed nodes re-opened): action sequences and segment states of a whole batch against
    the oracle's predecessor lists, on levine and on the corridor with a start velocity; and the forced log (exact_preds = 1)
    at eps = 1 must reproduce the running best-predecessor results exactly."""
    m = maps.load_fixture("levine")
    U = maps.make_U(1.0, 1, 3)
    S, G = maps.sample_queries(m, 48, seed=11)
    n_reopened = 0
    for eps, force in ((2.0, -1), (3.5, -1), (1.0, 1)):
        pl, op = make_pair(m, 3, dict(v_max=2.0, a_max=1.0, dt=1.0, tol_pos=0.5, epsilon=eps), U)
        pl.setExactPreds(force)
        sg, so = waypoint_pair(S, mp.ACC)
        gg, go = waypoint_pair(G, mp.ACC)
        res, acts, segs = pl.plan_batch(sg, gg, max_seg=64, want_states=True)
        ro, ao = op.plan_batch(so, go, nthreads=8, max_seg=64)
        for f in ("status", "n_seg", "cost", "pops", "n_nodes", "n_open", "n_closed", "pop_hash", "closed_hash"):
            assert np.array_equal(res[f], ro[f]) or (f == "cost" and np.array_equal(res[f][np.isfinite(ro[f])], ro[f][np.isfinite(ro[f])])), (eps, f)
        assert np.array_equal(acts, ao), eps
        n_reopened += int((res["pops"] != res["n_closed"]).sum())
        for i in np.flatnonzero(ro["status"] == 0)[:6]:  # segment states of a few plans against single oracle plans
            r1 = op.plan(so[i:i + 1], go[i:i + 1])
            assert np.array_equal(segs[i, :r1["n_seg"], :6], op.seg_states(r1["n_seg"])[:, :6]), (eps, i)
    assert n_reopened > 0, "no plan re-opened a closed node: the test does not exercise the log"


def test_jrk_control_2d():
    """JRK control on a grid (exercised upstream by MPL/test/test_planner_2d_with_prior_traj.cpp:80-84, u = 0.5)."""
    m, dim, params, U, start, goal = load_config("corridor")
    params = dict(v_max=1.0, a_max=1.0, j_max=1.0, dt=1.0, max_num=4000)
    pl, op = make_pair(m, dim, params, U)
    sg, so = waypoint_pair(start, mp.JRK)
    gg, go = waypoint_pair(goal, mp.JRK)
    pl.plan(sg, gg)
    ro = op.plan(so, go)
    assert_results_equal(pl.result(), ro)
    assert np.array_equal(pl.getActions(), op.actions(ro["n_seg"]))


def test_snp_control_2d():
    """Snap control (Control::SNP, order 4: primitive.h:48-52, validate_primitive with v/a/j bounds): the ORD = 4
    kernel instantiations, with and without a jerk bound (the latter takes the per-control exact sampling path)."""
    m, dim, params, U, start, goal = load_config("corridor")
    for prm, u, vel in ((dict(v_max=1.0, a_max=1.0, j_max=1.0, dt=1.0, tol_pos=0.5, max_num=1500), U, None),
                        (dict(v_max=1.5, a_max=1.0, j_max=2.0, dt=0.5, tol_pos=0.5, max_num=800), maps.make_U(1.0, 1, 2) * 0.5, [0.5, 0.0]),
                        (dict(v_max=1.0, a_max=1.0, dt=1.0, tol_pos=0.5, max_num=600), U, None)):
        pl, op = make_pair(m, dim, prm, u)
        sg, so = waypoint_pair(start, mp.SNP, vel=vel)
        gg, go = waypoint_pair(goal, mp.SNP)
        pl.plan(sg, gg)
        ro = op.plan(so, go)
        assert_results_equal(pl.result(), ro, ("SNP", prm))
        gn = pl.getNodes()
        assert np.array_equal(gn["key"][pl.getPopLog()], op.pop_keys(ro["pops"]))
        on, gk = _nodes_by_key(op.nodes(ro["n_nodes"])), _nodes_by_key(gn)
        assert set(on) == set(gk)
        for k, a in gk.items():
            assert np.array_equal(a["state"][:12], on[k]["state"][:12]) and a["g"] == on[k]["g"], k
        if ro["status"] == 0:
            assert np.array_equal(pl.getActions(), op.actions(ro["n_seg"]))
            assert np.array_equal(pl.getSegStates()[:, :12], op.seg_states(ro["n_seg"])[:, :12])


def test_map_ops():
    m = maps.load_fixture("simple")
    data = m.data.copy()
    data[::7] = -1  # sprinkle unknown cells
    mu = mp.VoxelMapUtil()
    mu.setMap(m.origin, m.dim, data, m.res)
    assert np.array_equal(mu.getMap(), data)
    mu.freeUnknown()
    want = np.where(data == -1, 0, data)
    assert np.array_equal(mu.getMap(), want)
    ns = np.array([[1, 0, 0], [-1, 0, 0], [0, 1, 0], [0, -1, 0]], dtype=np.int32)  # map_planner_node.cpp:75-86 style
    mu.dilate(ns)
    g = want.reshape(tuple(int(x) for x in m.dim[::-1]))
    out = g.copy()
    occ = g == 100
    out[:, :, 1:][occ[:, :, :-1]] = 100
    out[:, :, :-1][occ[:, :, 1:]] = 100
    out[:, 1:, :][occ[:, :-1, :]] = 100
    out[:, :-1, :][occ[:, 1:, :]] = 100
    assert np.array_equal(mu.getMap(), out.reshape(-1))
    assert mu.getRes() == m.res and np.array_equal(mu.getDim(), m.dim) and np.array_equal(mu.getOrigin(), m.origin)


def test_duplicate_sibling_hazard():
    """Controls so small that several successors of one expansion share one lattice key (and one table slot):
    exercises the serial hazard path; the reference keeps the FIRST discoverer's state (graph_search.h:84-88)."""
    m, dim, params, U, start, goal = load_config("corridor")
    U = maps.make_U(0.008, 1, 2)
    params = dict(v_max=1.0, a_max=1.0, dt=1.0, max_num=300)
    pl, op = make_pair(m, dim, params, U)
    sg, so = waypoint_pair(start, mp.ACC, vel=[0.5, 0.1])
    gg, go = waypoint_pair(goal, mp.ACC)
    pl.plan(sg, gg)
    ro = op.plan(so, go)
    assert_results_equal(pl.result(), ro)
    on = _nodes_by_key(op.nodes(ro["n_nodes"]))
    gnk = _nodes_by_key(pl.getNodes())
    assert set(on) == set(gnk)
    for k, a in gnk.items():
        assert np.array_equal(a["state"][:6], on[k]["state"][:6]) and a["g"] == on[k]["g"], k


def test_jrk_125_controls_3d():
    """BASELINE configs[4] shape at test size: 3D, jerk control, |U| = 125 (u in {-2..2}^3), dt = 0.5 — the
    four-batch (|U| > 32) kernel instantiation."""
    m = maps.load_fixture("skir")
    U = maps.make_U(2.0, 2, 3)
    assert U.shape[0] == 125
    params = dict(v_max=3.0, a_max=2.0, dt=0.5, max_num=400, tol_pos=0.5)
    pl, op = make_pair(m, 3, params, U)
    sg, so = waypoint_pair([5.5, 5.5, 0.5], mp.JRK)
    gg, go = waypoint_pair([1.5, 1.5, 5.5], mp.JRK)
    pl.plan(sg, gg)
    ro = op.plan(so, go)
    assert_results_equal(pl.result(), ro)
    assert np.array_equal(pl.getActions(), op.actions(ro["n_seg"]))
    gn = pl.getNodes()
    assert np.array_equal(gn["key"][pl.getPopLog()], op.pop_keys(ro["pops"]))
    # batch of a few more queries through the same instantiation
    S, G = maps.sample_queries(m, 12, seed=5)
    sg, so = waypoint_pair(S, mp.JRK)
    gg, go = waypoint_pair(G, mp.JRK)
    rg, ag, _ = pl.plan_batch(sg, gg, max_seg=48)
    ro2, ao = op.plan_batch(so, go, nthreads=8, max_seg=48)
    for i in range(len(S)):
        assert_results_equal(rg[i], ro2[i], i)
    assert np.array_equal(ag, ao)


@pytest.mark.parametrize("name,dim,ctrl_u", [("skir", 3, 1.0), ("corridor", 2, 0.5)])
def test_large_batch_uses_longest_first_order(name, dim, ctrl_u):
    """Batches larger than half the resident CTAs are pulled longest-first (free-space component labels + distance);
    the order is a scheduling hint only, so every result must still equal the oracle's, in input order."""
    m = maps.load_fixture(name)
    U = maps.make_U(ctrl_u, 1, dim)
    params = dict(v_max=2.0 if dim == 3 else 1.0, a_max=1.0, dt=1.0, max_num=150, tol_pos=0.5)
    pl, op = make_pair(m, dim, params, U)
    n = 700
    S, G = maps.sample_queries(m, n, seed=11, min_dist=1.0)
    sg, so = waypoint_pair(S, mp.ACC)
    gg, go = waypoint_pair(G, mp.ACC)
    rg, ag, _ = pl.plan_batch(sg, gg, max_seg=32)
    ro, ao = op.plan_batch(so, go, nthreads=8, max_seg=32)
    for i in range(n):
        assert_results_equal(rg[i], ro[i], (name, i))
    assert np.array_equal(ag, ao)
    assert pl.last_batch_stats()["launches"] >= 3  # keys + order + search kernel


def test_synthetic_boxes_jrk125_batch():
    """BASELINE configs[4] shape at test size: synthetic box map (seeded generator of SURVEY.md section 8d), jerk control,
    |U| = 125, dt = 0.5, max_num bound.  Every plan here stops at MaxExpandStep with > 32 768 nodes; the MaxExpandStep
    bound (300 * 125 + 2 * 125 + 64 = 37814 nodes) sizes the first and only arena tier, so no plan overflows.  Counters and
    the pop-order hash must still match the oracle."""
    m = maps.synthetic_boxes(n=96, occupied_frac=0.2, seed=1, res=0.1)
    U = maps.make_U(2.0, 2, 3)
    params = dict(v_max=3.0, a_max=2.0, dt=0.5, max_num=300, tol_pos=0.5)
    pl, op = make_pair(m, 3, params, U)
    n = 16
    S, G = maps.sample_queries(m, n, seed=2, min_dist=3.0, max_dist=9.0)
    sg, so = waypoint_pair(S, mp.JRK)
    gg, go = waypoint_pair(G, mp.JRK)
    rg, ag, _ = pl.plan_batch(sg, gg, max_seg=16)
    ro, ao = op.plan_batch(so, go, nthreads=8, max_seg=16)
    assert set(np.unique(ro["status"])) == {2} and ro["n_nodes"].max() > 32768
    for i in range(n):
        assert_results_equal(rg[i], ro[i], i)
    assert pl.last_batch_stats()["tiers"] == 1
    tiers = pl.last_batch_tiers()
    assert len(tiers) == 1 and tiers[0]["cap"] == 37814 and tiers[0]["n_overflow"] == 0, tiers


def test_full_bench_batch_parity():
    """BASELINE configs[1] at FULL size: the 1024-query levine-256 batch (the first 1024 queries of bench.py's list), every
    plan compared with the oracle (status, cost, counters, pop-order hash, closed hash, action rows), plus
    size-independent invariants."""
    import os
    from mpl_ros_b200 import workloads as W
    m = W.c2_map()
    U = W.controls(W.C2)
    pl, op = make_pair(m, 3, dict(W.C2["params"]), U)
    S, G = W.c2_queries(m, 1024)
    s, g = mp.waypoints_array(1024), mp.waypoints_array(1024)
    W.fill(s, g, S, G, W.C2["control"])
    so, go = oracle.make_waypoints(len(s)), oracle.make_waypoints(len(s))
    for f in ("pos", "control"):
        so[f], go[f] = s[f], g[f]
    rg, ag, _ = pl.plan_batch(s, g, max_seg=64)
    ro, ao = op.plan_batch(so, go, nthreads=os.cpu_count() or 8, max_seg=64)
    for f in RESULT_FIELDS:
        a, b = rg[f], ro[f]
        if f == "cost":
            assert np.array_equal(np.isinf(a), np.isinf(b)) and np.array_equal(a[np.isfinite(a)], b[np.isfinite(b)])
        else:
            assert np.array_equal(a, b), f
    assert np.array_equal(ag, ao)
    ok = rg["status"] == 0
    # invariants: cost = w*dt*n_seg + sum of u^2*dt along the action row; exhausted searches closed every node
    J = (U ** 2).sum(axis=1)
    for i in np.flatnonzero(ok)[:200]:
        acts = ag[i][: rg["n_seg"][i]]
        assert rg["cost"][i] == 10.0 * rg["n_seg"][i] + J[acts].sum()
    ex = rg["status"] == 3
    assert np.all(rg["n_open"][ex] == 0) and np.all(rg["n_closed"][ex] == rg["n_nodes"][ex])


def test_batch_in_flight_begin_end():
    """mplb_plan_stripe_begin / _end and mplb_plan_batch_sharded_begin / _end (one batch in flight per planner): two planners
    on one map alternate three batches each way; every batch must equal the synchronous call."""
    import torch
    from mpl_ros_b200 import dist as mdist, _lib
    m = maps.load_fixture("levine")
    U = maps.make_U(1.0, 1, 3)
    dev = torch.device("cuda", 0)
    comm = mdist.Comm(mdist.Comm.unique_id(), 0, 1)

    def mk(o, d, r, mu, first=True):
        if first:
            mu.freeUnknown()
        pl = mp.VoxelMapPlanner(False)
        pl.setMapUtil(mu)
        pl.setVmax(2.0); pl.setAmax(1.0); pl.setDt(1.0); pl.setU(U); pl.setTol(0.5)
        pl._keep = mu
        return pl

    sp = mdist.ShardedBatchPlanner(mk, dev, comm=comm)
    sp.set_map(m.origin, m.dim, m.res, m.data)
    sp2 = mdist.ShardedBatchPlanner(mk, dev, comm=comm)
    sp2.planner = mk(None, None, None, sp.planner.map_util_, first=False)
    n = 700
    batches = []
    for seed in (21, 22, 23):
        S, G = maps.sample_queries(m, n, seed=seed)
        s, g = mp.waypoints_array(n), mp.waypoints_array(n)
        s["pos"], g["pos"], s["control"], g["control"] = S, G, mp.ACC, mp.ACC
        want, want_acts = sp.plan_batch(s, g, max_seg=48)
        batches.append((s, g, want, want_acts))
    fields = [f for f in want.dtype.names if f != "device_ms"]
    # host-buffer halves, alternating planners
    sps = [sp, sp2]
    got = []
    for k, (s, g, _, _) in enumerate(batches):
        sps[k % 2].begin_batch(s, g, 48)
        if k > 0:
            got.append(sps[(k - 1) % 2].end_batch())
    got.append(sps[(len(batches) - 1) % 2].end_batch())
    for (s, g, want, want_acts), (res, acts) in zip(batches, got):
        assert all(np.array_equal(res[f], want[f]) or f == "cost" for f in fields)
        assert np.array_equal(acts, want_acts)
    # device-resident halves
    streams = [torch.cuda.Stream(device=dev), torch.cuda.Stream(device=dev)]
    bufs = [sp.make_device_buffers(n, 48), sp2.make_device_buffers(n, 48)]
    dsg = [(torch.from_numpy(s.view(np.uint8).reshape(n, -1)).to(dev), torch.from_numpy(g.view(np.uint8).reshape(n, -1)).to(dev))
           for s, g, _, _ in batches]
    outs = []
    for k in range(len(batches)):
        sps[k % 2].begin_stripe_device(dsg[k][0], dsg[k][1], n, bufs[k % 2], 48, streams[k % 2])
        if k > 0:
            sps[(k - 1) % 2].end_stripe_device(bufs[(k - 1) % 2])
            outs.append(sp.unstripe(bufs[(k - 1) % 2], n, 48))
    sps[(len(batches) - 1) % 2].end_stripe_device(bufs[(len(batches) - 1) % 2])
    outs.append(sp.unstripe(bufs[(len(batches) - 1) % 2], n, 48))
    for (s, g, want, want_acts), (res, acts) in zip(batches, outs):
        assert all(np.array_equal(res[f], want[f]) or f == "cost" for f in fields)
        assert np.array_equal(acts, want_acts)
