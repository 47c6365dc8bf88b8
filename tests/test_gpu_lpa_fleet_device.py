"""A fleet replan cycle whose output never leaves the device: mplb_lpa_plan_batch_device, mplb_lpa_trajectory_waypoints_device
(the next starts), mplb_lpa_serialize_trajectories_device and mplb_lpa_refine_trajectories_device through MapPlanner's static
members, in lockstep with the same replanners driven by the host calls (plan(), getActions / getSegStates), bitwise after every
step: records, the fixed-row trajectory layout, hm_ / pq_ / best_child_ dumps and the retained trajectories.  The fleet is the one
of test_gpu_lpa_fleet.py (lpa_flow and lpa_shaped_flow flows, 16 seeded random replanners: plain, potential and yaw sessions).
Next starts are held to the stored coords, to the oracle's end-state evaluation and to getWaypoints' running-sum t; messages to
a restatement of the wire format with each robot's own controls and dt, and to an A* planner's serialiser fed the same rows;
refinement to mplb_traj_solve_batch on host-built waypoint lists.  Then: truncation by max_seg, a path longer than one launch's
4096 rows, a failed plan that keeps the previous trajectory, waypoint indices at and past the ends, rejected arguments that leave
every planner as it was, and launch counts that do not grow with the fleet."""
import ctypes as C
import struct

import numpy as np
import pytest

torch = pytest.importorskip("torch")

import mpl_ros_b200 as mp
from mpl_ros_b200 import _lib
import oracle
import lpa_capacity_cases as K
import lpa_flow
from test_gpu_lpa import GpuMap
from test_gpu_lpa_shaped import GpuPlanner
from test_gpu_lpa_fleet import BIG, Member

pytestmark = pytest.mark.gpu

RES = _lib.RESULT_DTYPE
WP = _lib.WAYPOINT_DTYPE
MAX_SEG = 256


def ros_trajectory_bytes(dim, control, actions, seg_states, U, dt, z, frame_id, seq, stamp):
    """std_msgs/Header + Primitive[] + LambdaSeg[] (empty), built from (parent state, U[action], dt) like
    env_base::forward_action (env_base.h:228-231) and Primitive1D's constructors (primitive.h:35-52); as in test_gpu_wire.py."""
    order = {1: 1, 3: 2, 7: 3, 15: 4}[control & 15]
    b = struct.pack("<III", seq, stamp[0], stamp[1]) + struct.pack("<I", len(frame_id)) + frame_id.encode()
    b += struct.pack("<I", len(actions))
    for a, st in zip(actions, seg_states):
        rows = []
        for ax in range(3):
            c = [0.0] * 6
            if ax < dim:
                for d in range(order):
                    c[5 - d] = st[d * 3 + ax]
                c[5 - order] = U[a][ax]
            elif ax == 2:
                c[5] = z
            rows.append(c)
        cyaw = [0.0] * 6
        if control & 16:
            cyaw[4], cyaw[5] = U[a][dim], st[12]
        rows.append(cyaw)
        for c in rows:
            b += struct.pack("<I", 6) + struct.pack("<6d", *c)
        b += struct.pack("<d", dt)
    b += struct.pack("<I", 0)
    return b


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).reshape(-1).copy()).cuda()


def host(t, dtype):
    torch.cuda.synchronize()
    return t.cpu().numpy().view(dtype)


class Out:
    """the plan-batch layout of one device plan"""

    def __init__(self, n, max_seg):
        self.n, self.max_seg = n, max_seg
        self.res = torch.zeros(max(n, 1) * RES.itemsize, dtype=torch.uint8, device="cuda")
        self.act = torch.full((max(n, 1), max(max_seg, 1)), 12345, dtype=torch.int32, device="cuda")
        self.seg = torch.full((max(n, 1), max(max_seg, 1), 13), 7.0, dtype=torch.float64, device="cuda")

    def host(self):
        return host(self.res, RES)[:self.n], self.act.cpu().numpy()[:self.n], self.seg.cpu().numpy()[:self.n]


def plan_device(pls, d_s, d_g, max_seg=MAX_SEG):
    o = Out(len(pls), max_seg)
    mp.MapPlanner.planLPABatchDevice(pls, d_s, d_g, o.res, o.act, o.seg, max_seg)
    return o


def retained(pl):
    try:
        return pl.getActions().tobytes(), pl.getSegStates().tobytes()
    except mp.MplbError:  # no plan has succeeded yet
        return None


def dumps(p):
    pl = p.pl
    return (pl.lpaNodes().tobytes(), pl.lpaHeap().tobytes(), pl.lpaBestChild().tobytes(), retained(pl), pl.lpaCapacity())


def check_plan(members, out, what):
    """device copy (b) == host copy (s): record, rows (truncated as specified), dumps, retained trajectory"""
    res, act, seg = out.host()
    for i, mb in enumerate(members):
        rs = np.array(mb.s.pl.result(), dtype=RES)
        assert res[i].tobytes() == rs.tobytes(), (what, mb.name, res[i], rs)
        assert dumps(mb.b) == dumps(mb.s), (what, mb.name)
        ns = int(rs["n_seg"]) if int(rs["status"]) == 0 else 0
        k = min(ns, out.max_seg)
        if ns:
            acts, segs = mb.s.pl.getActions(), mb.s.pl.getSegStates()
            assert len(acts) == ns
            assert np.array_equal(act[i, :k], acts[:k]), (what, mb.name)
            assert seg[i, :k].tobytes() == segs[:k].tobytes(), (what, mb.name)
        assert (act[i, k:out.max_seg] == -1).all(), (what, mb.name)
        assert (seg[i, k:out.max_seg] == 7.0).all(), (what, mb.name)  # rows past the trajectory are not written


def host_plan(members, starts, goals):
    for i, mb in enumerate(members):
        mb.s.lpa_plan(starts[i:i + 1], goals[i:i + 1])


def oracle_end_state(mb, st, act):
    """the last primitive evaluated at dt: the oracle's get_succ row of the last parent"""
    w = oracle.make_waypoints(1)
    w["pos"][0], w["vel"][0], w["acc"][0], w["jrk"][0], w["yaw"][0] = st[0:3], st[3:6], st[6:9], st[9:12], st[12]
    w["control"] = mb.control
    return mb.o.succ_trace(w)[act]["succ"]


def running_t(j, dt):
    t = 0.0
    for _ in range(j):
        t += dt
    return t


def check_waypoints(members, out, idx):
    n = len(members)
    res, act, seg = out.host()
    d_idx = torch.tensor(idx, dtype=torch.int32, device="cuda")
    sentinel = np.zeros(n, dtype=WP)
    sentinel["t"] = -99.0
    d_w = dev(sentinel)
    d_ok = torch.full((n,), 5, dtype=torch.int32, device="cuda")
    mp.MapPlanner.trajectoryWaypointsBatch([mb.b.pl for mb in members], out.res, out.act, out.seg, out.max_seg, d_idx, d_w, d_ok)
    w, ok = host(d_w, WP), d_ok.cpu().numpy()
    for i, mb in enumerate(members):
        ns, j = int(res[i]["n_seg"]), idx[i]
        good = int(res[i]["status"]) == 0 and 1 <= ns <= out.max_seg and 0 <= j <= ns
        assert ok[i] == int(good), (mb.name, ok[i], good)
        if not good:
            assert w[i]["t"] == -99.0
            continue
        dim, dt = mb.dim, mb.b.pl.dt_
        e = seg[i, j] if j < ns else oracle_end_state(mb, seg[i, ns - 1], act[i, ns - 1])
        got = np.concatenate([w[i]["pos"], w[i]["vel"], w[i]["acc"], w[i]["jrk"]])
        want = np.zeros(12)
        for q in range(4):
            want[3 * q:3 * q + (3 if j < ns else dim)] = e[3 * q:3 * q + (3 if j < ns else dim)]
        assert got.tobytes() == want.tobytes(), (mb.name, j, got, want)
        if j < ns or mb.control & 16:
            assert w[i]["yaw"] == e[12], (mb.name, j)
        assert w[i]["t"] == running_t(j, dt) and int(w[i]["control"]) == mb.control, mb.name
    return d_w, w, ok


def check_messages(members, out):
    n = len(members)
    res, act, seg = out.host()
    stride = int(_lib.lib().mplb_trajectory_msg_size(out.max_seg, b"map"))
    d_out = torch.zeros(n * stride, dtype=torch.uint8, device="cuda")
    d_len = torch.zeros(n, dtype=torch.int32, device="cuda")
    mp.MapPlanner.serializeLPABatch([mb.b.pl for mb in members], out.res, out.act, out.seg, out.max_seg, d_out, stride, d_len,
                                    z=0.25, frame_id="map", seq=3, stamp=(11, 22))
    msgs, lens = d_out.cpu().numpy().reshape(n, stride), d_len.cpu().numpy().view(np.uint32)
    for i, mb in enumerate(members):
        ok = int(res[i]["status"]) == 0
        ns = int(res[i]["n_seg"]) if ok else 0
        if ns > out.max_seg:
            assert lens[i] == 0
            continue
        want = ros_trajectory_bytes(mb.dim, mb.control, act[i, :ns], seg[i, :ns], mb.b.pl.U_, mb.b.pl.dt_, 0.25, "map", 3, (11, 22))
        assert msgs[i, :lens[i]].tobytes() == want, mb.name
    return msgs, lens


def refine_host(members, res, act, seg, max_seg, control, yaw_control):
    """mplb_traj_solve_batch on the waypoint lists built on the host (map_planner_node.cpp:216-227)"""
    n = len(members)
    dim = members[0].dim
    coefs = np.zeros((n, max_seg, dim + 1, 6))
    L = _lib.lib()
    for i, mb in enumerate(members):
        ns = int(res[i]["n_seg"])
        if int(res[i]["status"]) != 0 or not 1 <= ns <= max_seg:
            continue
        ends = np.vstack([seg[i, :ns], oracle_end_state(mb, seg[i, ns - 1], act[i, ns - 1])[None]])
        w = np.zeros(ns + 1, dtype=WP)
        for j, st in enumerate(ends):
            lim = 3 if j < ns else dim
            w["pos"][j, :lim], w["vel"][j, :lim], w["acc"][j, :lim], w["jrk"][j, :lim] = st[0:lim], st[3:3 + lim], st[6:6 + lim], st[9:9 + lim]
            w["yaw"][j] = st[12] if (j < ns or mb.control & 16) else 0.0
            w["t"][j] = j * mb.b.pl.dt_
        w["control"] = mp.VEL
        w["control"][0] = w["control"][ns] = mb.control
        offs = np.array([0, ns + 1], dtype=np.int32)
        dts = np.full(ns, mb.b.pl.dt_)
        c = np.zeros((ns, dim + 1, 6))
        _lib.check(L.mplb_traj_solve_batch(dim, control, yaw_control, 1, _lib.ptr(offs), _lib.ptr(w), _lib.ptr(dts), _lib.ptr(c), None))
        coefs[i, :ns] = c
    return coefs


def check_refine(members, out):
    res, act, seg = out.host()
    for dim in (2, 3):
        ix = [i for i, mb in enumerate(members) if mb.dim == dim]
        if not ix:
            continue
        sub = [members[i] for i in ix]
        o = Out(len(ix), out.max_seg)
        o.res = dev(res[ix])
        o.act = torch.from_numpy(act[ix].copy()).cuda()
        o.seg = torch.from_numpy(seg[ix].copy()).cuda()
        d_c = torch.full((len(ix), out.max_seg, dim + 1, 6), 9.0, dtype=torch.float64, device="cuda")
        nseg = mp.MapPlanner.refineLPABatch([mb.b.pl for mb in sub], o.res, o.act, o.seg, out.max_seg, d_c, mp.JRK, mp.VEL)
        got = d_c.cpu().numpy()
        want = refine_host(sub, res[ix], act[ix], seg[ix], out.max_seg, mp.JRK, mp.VEL)
        for k, i in enumerate(ix):
            ns = int(res[i]["n_seg"])
            good = int(res[i]["status"]) == 0 and 1 <= ns <= out.max_seg
            assert nseg[k] == (ns if good else 0), members[i].name
        assert got.tobytes() == want.tobytes()


def make_fleet():
    members = [Member("flow", n) for n in lpa_flow.FLOWS if n not in BIG]
    members += [Member("shaped", n) for n in __import__("lpa_shaped_flow").FLOWS if n not in BIG]
    members += [Member("fuzz", (seed, dim)) for dim in (2, 3) for seed in range(8)]
    for mb in members:
        mb.control = int(mb.s_wp["control"][0])
    return members


NS3 = np.array([(x, y, 0) for x in range(-1, 2) for y in range(-1, 2)], dtype=np.int32)


def edit(members, rnd):
    """the node's add-cloud edit: on the device copy (b) a ray across the trajectory's middle is traced on the device, its isFree
    stencil cells written with mplb_map_set_cells_device and the whole fleet updated with mplb_lpa_update_nodes_batch_device; the
    host copy (s) and the oracle's map receive the same cells through the host calls"""
    L = _lib.lib()
    vp = lambda t: C.c_void_p(t.data_ptr())  # noqa: E731
    d_lists, lists = [], []
    for i, mb in enumerate(members):
        path = mb.s.lpa_best_child_states()[:, :3]
        d_c = torch.zeros((0, 3), dtype=torch.int32, device="cuda")
        if len(path) >= 4 and (i + rnd) % 4 != 3:
            d1 = torch.tensor(path[len(path) // 3][None], device="cuda")
            d2 = torch.tensor(path[2 * len(path) // 3][None], device="cuda")
            cap = 4096
            d_out = torch.zeros((cap, 3), dtype=torch.int32, device="cuda")
            k = _lib.check(L.mplb_map_trace_cells_device(mb.maps[0].mu._h, vp(d1), vp(d2), 1, _lib.ptr(NS3), len(NS3), mp.TRACE_FREE,
                                                         vp(d_out), cap, None, None))
            d_c = d_out[:min(k, cap)]
            if len(d_c):
                _lib.check(L.mplb_map_set_cells_device(mb.maps[0].mu._h, vp(d_c), len(d_c), 100, None))
        d_lists.append(d_c)
        cells = d_c.cpu().numpy()[:, :mb.dim]  # the test's own view of the edit, for the host copies
        if len(cells):
            mb.grid[mb.lin(cells)] = 100
            for m in mb.maps[1:]:
                m.set_cells(cells, 100)
        lists.append(cells)
    pls = [mb.b.pl for mb in members]
    mp.MapPlanner.getLinkedNodesBatch(pls)
    offs = np.concatenate([[0], np.cumsum([len(c) for c in d_lists])]).astype(np.int64)
    d_all = torch.cat(d_lists).contiguous() if offs[-1] else torch.zeros((1, 3), dtype=torch.int32, device="cuda")
    visited = np.zeros(len(members), dtype=np.int32)
    _lib.check(L.mplb_lpa_update_nodes_batch_device(mp.MapPlanner._handles(pls), len(pls), 1, vp(d_all), _lib.ptr(offs),
                                                    _lib.ptr(visited)))
    for i, mb in enumerate(members):
        mb.s.lpa_get_linked_nodes()
        v = mb.s.lpa_update_blocked_nodes(lists[i]) if len(lists[i]) else 0
        assert visited[i] == v, (mb.name, visited[i], v)
    for mb in members:
        assert dumps(mb.b) == dumps(mb.s), ("edit", mb.name)
    return int(offs[-1])


def host_next_start(mb):
    """getWaypoints()[1] of the host copy's retained trajectory: the parent coord of segment 1, t = 0 + dt"""
    st = mb.s.pl.getSegStates()[1]
    w = np.zeros(1, dtype=WP)
    w["pos"][0], w["vel"][0], w["acc"][0], w["jrk"][0], w["yaw"][0] = st[0:3], st[3:6], st[6:9], st[9:12], st[12]
    w["t"], w["control"] = 0.0 + mb.b.pl.dt_, mb.control
    return w[0]


def test_fleet_device_cycle_equals_host_cycle():
    members = make_fleet()
    n = len(members)
    pls = [mb.b.pl for mb in members]
    s, g = mp.waypoints_array(n), mp.waypoints_array(n)
    for i, mb in enumerate(members):
        s[i], g[i] = mb.s_wp[0], mb.g_wp[0]
    d_s, d_g = dev(s), dev(g)
    out = plan_device(pls, d_s, d_g)
    host_plan(members, s, g)
    check_plan(members, out, "plan 0")
    edited = 0
    for rnd in range(2):
        check_messages(members, out)
        check_refine(members, out)
        res = out.host()[0]
        check_waypoints(members, out, [-1 if i % 7 == 6 else 0 if i % 7 == 5 else int(r["n_seg"]) + (i % 2) if i % 7 == 4 else 1
                                       for i, r in enumerate(res)])
        # the node's next start: ws[1] after getSubStateSpace(1) where the trajectory has two segments or more; others keep theirs
        adv = [int(r["status"]) == 0 and int(r["n_seg"]) >= 2 for r in res]
        d_ok = torch.full((n,), 5, dtype=torch.int32, device="cuda")
        mp.MapPlanner.trajectoryWaypointsBatch(pls, out.res, out.act, out.seg, out.max_seg,
                                               torch.tensor([1 if a else -1 for a in adv], dtype=torch.int32, device="cuda"), d_s, d_ok)
        assert d_ok.cpu().tolist() == [int(a) for a in adv]
        nxt = s.copy()
        for i, mb in enumerate(members):
            if adv[i]:
                nxt[i] = host_next_start(mb)
        assert host(d_s, WP).tobytes() == nxt.tobytes(), rnd
        ts_b = [(1 if adv[i] else 0) if len(mb.s.lpa_best_child()) else 7 for i, mb in enumerate(members)]
        # through the C calls: an entry whose sweep meets a successor that left hm_ reports MPLB_ERR_STATE (where the reference
        # dereferences a null State) and the batch returns that error after the others completed; both copies must agree
        L = _lib.lib()
        sizes = np.zeros(n, dtype=np.int32)
        rc = L.mplb_lpa_sub_state_space_batch(mp.MapPlanner._handles(pls), n, _lib.ptr(np.array(ts_b, dtype=np.int32)), _lib.ptr(sizes))
        assert rc == 0 or rc == -3, rc
        assert (rc == -3) == bool((sizes == -3).any())
        for i, mb in enumerate(members):
            if len(mb.s.lpa_best_child()):
                assert sizes[i] == L.mplb_get_sub_state_space(mb.s.pl._h, ts_b[i]), mb.name
        for mb in members:
            assert dumps(mb.b) == dumps(mb.s), ("subtree", mb.name)
        edited += edit(members, rnd)
        s = nxt
        out = plan_device(pls, d_s, d_g)
        host_plan(members, s, g)
        check_plan(members, out, "plan %d" % (rnd + 1))
    assert edited > 0


def test_messages_equal_astar_serialiser():
    """a flow's LPA* rows through the fleet serialiser == the A* serialiser of a planner configured the same way, fed the same rows"""
    members = [Member("flow", n) for n in ("skir_acc", "corridor_acc")]
    for mb in members:
        mb.control = int(mb.s_wp["control"][0])
    n = len(members)
    s, g = mp.waypoints_array(n), mp.waypoints_array(n)
    for i, mb in enumerate(members):
        s[i], g[i] = mb.s_wp[0], mb.g_wp[0]
    out = plan_device([mb.b.pl for mb in members], dev(s), dev(g))
    msgs, lens = check_messages(members, out)
    res, act, seg = out.host()
    for i, mb in enumerate(members):
        a = mb.b.pl
        twin = mp.MapPlanner(mb.dim, False)  # A*, same map, controls and dt
        twin.setMapUtil(mb.maps[0].mu)
        twin.setVmax(a.v_max_ if hasattr(a, "v_max_") else 2.0)
        twin.setDt(a.dt_)
        twin.setU(a.U_)
        sb, gb = mp.waypoints_array(1), mp.waypoints_array(1)
        sb[0], gb[0] = s[i], g[i]
        twin.plan_batch(sb, gb)  # any batch: the serialiser takes the configuration it was planned with
        want = twin.serialize_trajectories(res[i:i + 1], act[i:i + 1], seg[i:i + 1], z=0.25, frame_id="map", seq=3, stamp=(11, 22))[0]
        assert want is not None and msgs[i, :lens[i]].tobytes() == want, mb.name


def test_truncation_long_paths_and_failed_plans():
    """max_seg below n_seg; a strip longer than one launch's 4096 rows (k_lpa_traj); a failed plan keeps the previous trajectory"""
    case = K.strip_case(K.LONG_SEG)
    sw, gw = K.random_waypoints(case, 2)
    pair = [K.random_planner(GpuMap, GpuPlanner, case, 2)[1] for _ in range(2)]
    flow = Member("flow", "skir_acc")
    flow.control = int(flow.s_wp["control"][0])
    pls = [pair[0].pl, flow.b.pl]
    s, g = mp.waypoints_array(2), mp.waypoints_array(2)
    s[0], g[0], s[1], g[1] = sw[0], gw[0], flow.s_wp[0], flow.g_wp[0]
    out = plan_device(pls, dev(s), dev(g), max_seg=8)
    res, act, seg = out.host()
    r1 = pair[1].lpa_plan(sw, gw)
    flow.s.lpa_plan(flow.s_wp, flow.g_wp)
    assert int(res[0]["n_seg"]) == K.LONG_SEG and res[0].tobytes() == np.array(r1, dtype=RES).tobytes()
    assert 1 <= int(res[1]["n_seg"]) <= 8
    assert dumps(pair[0]) == dumps(pair[1]) and dumps(flow.b) == dumps(flow.s)
    assert len(pair[0].pl.getActions()) == K.LONG_SEG
    assert np.array_equal(act[0], pair[1].pl.getActions()[:8]) and seg[0].tobytes() == pair[1].pl.getSegStates()[:8].tobytes()
    stride = int(_lib.lib().mplb_trajectory_msg_size(8, b"map"))
    d_len = torch.full((2,), 77, dtype=torch.int32, device="cuda")
    mp.MapPlanner.serializeLPABatch(pls, out.res, out.act, out.seg, 8, torch.zeros(2 * stride, dtype=torch.uint8, device="cuda"),
                                    stride, d_len)
    assert d_len.cpu().tolist() == [0, int(_lib.lib().mplb_trajectory_msg_size(int(res[1]["n_seg"]), b"map"))]
    nseg = mp.MapPlanner.refineLPABatch([pair[0].pl], out.res[:RES.itemsize], out.act[:1], out.seg[:1], 8,
                                        torch.zeros((1, 8, 3, 6), dtype=torch.float64, device="cuda"))
    assert nseg == [0]
    # a failed plan (the start's cell occupied: start not free) keeps the previous trajectory
    kept = (flow.b.pl.getActions().copy(), flow.b.pl.getSegStates().copy())
    cell = lpa_flow.cells_on_path(flow.m, 3, flow.s_wp["pos"][:, :3], 1).astype(np.int32)
    flow.set_cells(cell, 100)
    d_res = torch.zeros(RES.itemsize, dtype=torch.uint8, device="cuda")
    d_act = torch.zeros((1, 8), dtype=torch.int32, device="cuda")
    mp.MapPlanner.planLPABatchDevice([flow.b.pl], dev(flow.s_wp), dev(flow.g_wp), d_res, d_act, None, 8)
    flow.s.lpa_plan(flow.s_wp, flow.g_wp)
    r = host(d_res, RES)[0]
    assert int(r["status"]) != 0 and r.tobytes() == np.array(flow.s.pl.result(), dtype=RES).tobytes()
    assert (d_act.cpu().numpy() == -1).all()
    assert np.array_equal(flow.b.pl.getActions(), kept[0]) and flow.b.pl.getSegStates().tobytes() == kept[1].tobytes()
    assert dumps(flow.b) == dumps(flow.s)


def test_rejected_arguments_leave_every_planner_untouched():
    members = [Member("flow", n) for n in ("skir_acc", "corridor_acc")]
    for mb in members:
        mb.control = int(mb.s_wp["control"][0])
    n = 2
    pls = [mb.b.pl for mb in members]
    s, g = mp.waypoints_array(n), mp.waypoints_array(n)
    for i, mb in enumerate(members):
        s[i], g[i] = mb.s_wp[0], mb.g_wp[0]
    d_s, d_g = dev(s), dev(g)
    out = plan_device(pls, d_s, d_g)
    before = [dumps(mb.b) for mb in members]
    off = mp.MapPlanner(3, False)  # LPA* off
    fresh = mp.MapPlanner(3, False)
    fresh.setLPAstar(True)  # on, never planned
    L = _lib.lib()
    H = mp.MapPlanner._handles
    vp = lambda t: C.c_void_p(t.data_ptr())  # noqa: E731
    bad_plan = [
        (H(pls), n, None, vp(d_g), vp(out.res), None, None, 0, None),
        (H([pls[0], pls[0]]), 2, vp(d_s), vp(d_g), vp(out.res), None, None, 0, None),
        (H([pls[0], off]), 2, vp(d_s), vp(d_g), vp(out.res), None, None, 0, None),
        (H(pls), n, vp(d_s), vp(d_g), vp(out.res), vp(out.act), None, -1, None),
    ]
    for args in bad_plan:
        assert L.mplb_lpa_plan_batch_device(*args) < 0
    rows = (vp(out.res), vp(out.act), vp(out.seg), MAX_SEG)
    idx = torch.ones(n, dtype=torch.int32, device="cuda")
    w = torch.zeros(n * WP.itemsize, dtype=torch.uint8, device="cuda")
    ok = torch.zeros(n, dtype=torch.int32, device="cuda")
    for hs in (H([pls[0], pls[0]]), H([pls[0], off]), H([pls[0], fresh])):
        assert L.mplb_lpa_trajectory_waypoints_device(hs, 2, *rows, vp(idx), vp(w), vp(ok), None) < 0
        assert L.mplb_lpa_serialize_trajectories_device(hs, 2, *rows, 0.0, 0, 0, 0, b"map", vp(w), 8, vp(ok), None) < 0
        assert L.mplb_lpa_refine_trajectories_device(hs, 2, *rows, mp.JRK, mp.VEL, vp(w), None, None) < 0
    assert L.mplb_lpa_trajectory_waypoints_device(H(pls), 2, None, vp(out.act), vp(out.seg), MAX_SEG, vp(idx), vp(w), vp(ok), None) < 0
    assert ok.cpu().tolist() == [0, 0]
    assert [dumps(mb.b) for mb in members] == before


def test_launches_per_call_do_not_grow_with_the_fleet():
    counts = {}
    for n in (1, 32):
        ms = [Member("flow", "skir_acc") for _ in range(n)]
        pls = [mb.b.pl for mb in ms]
        s, g = mp.waypoints_array(n), mp.waypoints_array(n)
        for i, mb in enumerate(ms):
            s[i], g[i] = mb.s_wp[0], mb.g_wp[0]
        mp.MapPlanner.planLPABatch(pls, s, g)  # sessions allocated: no growth below
        L = _lib.lib()
        steps = []

        def step(fn):
            c0 = L.mplb_launch_count()
            fn()
            steps.append(int(L.mplb_launch_count() - c0))
        d_s, d_g = dev(s), dev(g)
        o = Out(n, MAX_SEG)
        step(lambda: mp.MapPlanner.planLPABatch(pls, s, g))
        step(lambda: mp.MapPlanner.planLPABatchDevice(pls, d_s, d_g, o.res, o.act, o.seg, MAX_SEG))
        w, ok = torch.zeros(n * WP.itemsize, dtype=torch.uint8, device="cuda"), torch.zeros(n, dtype=torch.int32, device="cuda")
        step(lambda: mp.MapPlanner.trajectoryWaypointsBatch(pls, o.res, o.act, o.seg, MAX_SEG,
                                                            torch.ones(n, dtype=torch.int32, device="cuda"), w, ok))
        stride = int(L.mplb_trajectory_msg_size(MAX_SEG, b"map"))
        step(lambda: mp.MapPlanner.serializeLPABatch(pls, o.res, o.act, o.seg, MAX_SEG,
                                                     torch.zeros(n * stride, dtype=torch.uint8, device="cuda"), stride,
                                                     torch.zeros(n, dtype=torch.int32, device="cuda")))
        step(lambda: mp.MapPlanner.refineLPABatch(pls, o.res, o.act, o.seg, MAX_SEG,
                                                  torch.zeros((n, MAX_SEG, 4, 6), dtype=torch.float64, device="cuda")))
        res = o.host()[0]
        assert ok.cpu().tolist() == [int(int(r["status"]) == 0 and 1 <= int(r["n_seg"]) <= MAX_SEG) for r in res]
        counts[n] = steps
    assert counts[1] == counts[32], counts
