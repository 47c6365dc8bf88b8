"""The batched TrajSolver (mpl_ros_b200/csrc/mplb_trajsolve.cu) at its size and arithmetic edges, exact against the oracle.

Every case of tests/trajsolver_edge_cases.py equals oracle.traj_solve at tolerance 0 (NaN placement for the degenerate
lists) and proves the path it targets through mplb_traj_solve_last_stats: which CTAs kept their work space in shared memory
and which in global scratch, and the largest list.  The device entry points are called directly with torch tensors on a side
stream, sub-range calls and the slots of unsolved trajectories are pinned, the thread-local scratch is grown and shrunk, long
planned trajectories are refined, and a list past the 8 GiB work-space limit is refused."""
import ctypes as C
import functools
import types

import numpy as np
import pytest
import torch

import mpl_ros_b200 as mp
from mpl_ros_b200 import _lib, maps, traj_solver
import oracle
from helpers_gpu import make_pair, waypoint_pair
from trajsolver_cases import ACC, JRK, SNP, VEL
import trajsolver_edge_cases as E
from test_gpu_fuzz import _refine_waypoints

pytestmark = pytest.mark.gpu
CASES = E.cases()
WPB = _lib.WAYPOINT_DTYPE.itemsize


@functools.lru_cache(maxsize=None)
def _want(name, dim, control, yaw_control, W):
    c = next(x for x in CASES + E.mixed_batch() + E.one_global_batch() if x.name == name)
    return oracle.traj_solve(dim, control, c.wps, c.dts, yaw_control)


def want(c):
    return _want(c.name, c.dim, c.control, c.yaw_control, c.W)


def same(got, exp):
    """Bit-identical, except that a NaN matches any NaN (x86 and the GPU make different default NaNs)."""
    if got.shape != exp.shape:
        return False
    ng, ne = np.isnan(got), np.isnan(exp)
    return np.array_equal(ng, ne) and np.array_equal(got[~ng], exp[~ne])


def expected_stats(cs):
    cs = [c for c in cs if c.W >= 2]
    pg = sum(E.pos_global(c.W, c.dim, c.control) for c in cs)
    yg = sum(E.yaw_global(c.W, c.yaw_control) for c in cs)
    return dict(n_traj=len(cs), max_wp=max([c.W for c in cs] + [0]), pos_shared=len(cs) - pg, pos_global=pg,
                yaw_shared=len(cs) - yg, yaw_global=yg)


def check_stats(cs):
    st = traj_solver.last_stats()
    exp = expected_stats(cs)
    assert {k: st[k] for k in exp} == exp, (cs, st)
    assert (st["global_bytes"] > 0) == (exp["pos_global"] + exp["yaw_global"] > 0)
    return st


def test_every_case_exact_and_on_its_path():
    seen = dict(split=0, seg=0, nfree=0, ph4=0, global_=0, shared=0)
    for c in CASES:
        got = traj_solver.solve_batch(c.dim, c.control, [c.wps], [c.dts], c.yaw_control)[0]
        assert same(got, want(c)), (c, np.nanmax(np.abs(got - want(c))))
        if "degenerate" in c.tags:
            assert np.isnan(got).any() and not np.isnan(got).all()
        else:
            assert np.isfinite(got).all(), c
        st = check_stats([c])
        seen["split"] += st["pos_global"] != st["yaw_global"]
        seen["global_"] += st["pos_global"] + st["yaw_global"]
        seen["shared"] += st["pos_shared"] + st["yaw_shared"]
        seen["seg"] += st["max_wp"] >= 258
        seen["nfree"] += E.nfree(c.wps, c.control) > 257
        seen["ph4"] += (c.W - 1) * c.dim > E.THREADS
    assert all(seen.values()), seen
    # the CTA pair that splits: 3-D JRK position in global scratch, its JRK yaw in shared memory, at W = 50
    c = next(x for x in CASES if x.name == "smem_3d_JRK_JRK_50")
    traj_solver.solve_batch(3, JRK, [c.wps], [c.dts], JRK)
    st = traj_solver.last_stats()
    assert (st["pos_global"], st["yaw_shared"], st["pos_shared"], st["yaw_global"]) == (1, 1, 0, 0), st


def test_mixed_batch_one_launch():
    cs = E.mixed_batch()
    got = traj_solver.solve_batch(2, ACC, [c.wps for c in cs], [c.dts for c in cs], VEL)
    st = check_stats(cs)
    assert st["pos_global"] > 0 and st["pos_shared"] > 0 and st["max_wp"] == 300
    for c, g in zip(cs, got):
        if c.W < 2:
            assert len(g) == 0
        else:
            assert np.array_equal(g, want(c)), c


def test_batch_with_one_global_job():
    cs = E.one_global_batch()
    got = traj_solver.solve_batch(3, JRK, [c.wps for c in cs], [c.dts for c in cs], JRK)
    st = check_stats(cs)
    assert (st["pos_global"], st["yaw_global"], st["pos_shared"]) == (1, 0, len(cs) - 1), st
    for c, g in zip(cs, got):
        assert np.array_equal(g, want(c)), c


# ---- the device entry points, called directly

def _pack(cs):
    off = np.zeros(len(cs) + 1, dtype=np.int32)
    for i, c in enumerate(cs):
        off[i + 1] = off[i] + c.W
    segoff = np.concatenate([[0], np.cumsum([max(c.W - 1, 0) for c in cs])]).astype(np.int64)
    wps = np.concatenate([c.wps for c in cs]) if off[-1] else np.zeros(1, dtype=_lib.WAYPOINT_DTYPE)
    dts = np.concatenate([c.dts for c in cs] + [np.zeros(1)])
    return off, segoff, wps, dts


def _dev_solve(dim, control, yaw_control, off, d_wps, d_dts, d_coefs, stream, n_segs=None):
    n = len(off) - 1
    nseg = np.full(max(n, 1), -7, dtype=np.int32) if n_segs is None else n_segs
    rc = _lib.lib().mplb_traj_solve_batch_device(dim, int(control), int(yaw_control), n, _lib.ptr(np.ascontiguousarray(off)),
                                                 C.c_void_p(d_wps), C.c_void_p(d_dts), C.c_void_p(d_coefs), _lib.ptr(nseg),
                                                 C.c_void_p(stream))
    _lib.check(rc)
    return nseg[:n]


def _to_dev(a):
    return torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).copy()).cuda()


def test_device_variant_with_torch_tensors_on_a_side_stream():
    cs = [c for c in CASES if c.dim == 3 and c.control == JRK and c.yaw_control == ACC]  # W = 16 .. 78, both scratch kinds
    off, segoff, wps, dts = _pack(cs)
    d_wps, d_dts = _to_dev(wps), torch.from_numpy(dts).cuda()
    d_coefs = torch.full((int(segoff[-1]), 4, 6), 3.5, dtype=torch.float64, device="cuda")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        nseg = _dev_solve(3, JRK, ACC, off, d_wps.data_ptr(), d_dts.data_ptr(), d_coefs.data_ptr(), s.cuda_stream)
    torch.cuda.current_stream().wait_stream(s)
    got = d_coefs.cpu().numpy()
    assert list(nseg) == [c.W - 1 for c in cs]
    check_stats(cs)
    for i, c in enumerate(cs):
        assert same(got[segoff[i]:segoff[i + 1]], want(c)), c


def test_device_variant_sub_ranges():
    """wp_offsets[0] != 0: the offsets are rebased, d_wps points at the sub-range's first waypoint and d_dts / d_coefs at its
    first segment; slots outside the sub-range are not touched."""
    cs = E.mixed_batch()
    off, segoff, wps, dts = _pack(cs)
    d_wps, d_dts = _to_dev(wps), torch.from_numpy(dts).cuda()
    sentinel = -123.25
    d_coefs = torch.full((int(segoff[-1]) + 1, 3, 6), sentinel, dtype=torch.float64, device="cuda")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    seg_bytes = 3 * 6 * 8
    for lo, hi in ((3, 9), (9, len(cs)), (1, 2)):
        sub = off[lo:hi + 1].copy()
        assert sub[0] != 0
        nseg = _dev_solve(2, ACC, VEL, sub, d_wps.data_ptr() + int(off[lo]) * WPB, d_dts.data_ptr() + int(segoff[lo]) * 8,
                          d_coefs.data_ptr() + int(segoff[lo]) * seg_bytes, s.cuda_stream)
        assert list(nseg) == [max(c.W - 1, 0) for c in cs[lo:hi]]
        check_stats(cs[lo:hi])
    got = d_coefs.cpu().numpy()
    for i, c in enumerate(cs):
        if i == 0 or i == 2:  # not in any sub-range
            assert (got[segoff[i]:segoff[i + 1]] == sentinel).all()
        elif c.W >= 2:
            assert np.array_equal(got[segoff[i]:segoff[i + 1]], want(c)), c
    assert (got[-1] == sentinel).all()


def test_unsolved_trajectories_are_zeroed():
    """An uninitialised solver (SNP, or a yaw order other than VEL / ACC / JRK) returns empty trajectories; both variants
    zero their coefficient slots instead of leaving the caller's data there."""
    cs = [c for c in CASES if c.name.startswith("flags_")][:4]
    off, segoff, wps, dts = _pack(cs)
    d_wps, d_dts = _to_dev(wps), torch.from_numpy(dts).cuda()
    for control, yc in ((SNP, VEL), (JRK, SNP), (JRK, 0)):
        d_coefs = torch.full((int(segoff[-1]), 4, 6), 9.0, dtype=torch.float64, device="cuda")
        nseg = _dev_solve(3, control, yc, off, d_wps.data_ptr(), d_dts.data_ptr(), d_coefs.data_ptr(), 0)
        torch.cuda.synchronize()
        assert not nseg.any() and not d_coefs.cpu().numpy().any(), (control, yc)
        assert traj_solver.last_stats()["n_traj"] == 0
        host = np.full((int(segoff[-1]), 4, 6), 9.0)
        hn = np.full(len(cs), -1, dtype=np.int32)
        _lib.check(_lib.lib().mplb_traj_solve_batch(3, int(control), int(yc), len(cs), _lib.ptr(off), _lib.ptr(wps), _lib.ptr(dts),
                                                    _lib.ptr(host), _lib.ptr(hn)))
        assert not hn.any() and not host.any()


# ---- scratch reuse

def _skir_refine():
    m = maps.load_fixture("skir")
    pl, _ = make_pair(m, 3, dict(v_max=2.0, a_max=1.0, dt=1.0, tol_pos=0.5), maps.make_U(1.0, 1, 3))
    starts, goals = maps.sample_queries(m, 12, seed=9, min_dist=1.5)
    s, g = mp.waypoints_array(12), mp.waypoints_array(12)
    s["pos"], g["pos"] = starts, goals
    s["control"] = g["control"] = mp.ACC
    res, acts, segs = pl.plan_batch(s, g, max_seg=16, want_states=True)
    return lambda: pl.refine_trajectories(res, acts, segs, mp.ACC, mp.JRK)


def test_scratch_grows_and_shrinks():
    """small (shared) -> large (global) -> small -> larger (global), interleaved with refinement: every result equals a fresh
    call on the same input."""
    by = {c.name: c for c in CASES}
    small, large, larger = by["flags_alternating_3d"], by["threads_nfree_258"], by["threads_seg_3d_JRK_258"]
    refine = _skir_refine()
    r0 = refine()
    gb = []
    for c in (small, large, small, larger, small, large):
        got = traj_solver.solve_batch(c.dim, c.control, [c.wps], [c.dts], c.yaw_control)[0]
        assert np.array_equal(got, want(c)), c
        gb.append(traj_solver.last_stats()["global_bytes"])
        r = refine()
        assert np.array_equal(r[0], r0[0]) and np.array_equal(r[1], r0[1])
    assert gb[0] == gb[2] == gb[4] == 0 and 0 < gb[1] == gb[5] < gb[3]


# ---- refinement of long plans

def _corridor(dim, length, origin):
    """A straight corridor one cell wide along x (res 1 m), walls everywhere else: VEL plans move one cell per dt."""
    nd = (length + 2, 5) if dim == 2 else (length + 2, 3, 3)
    data = np.full(nd[::-1], 100, dtype=np.int8)
    if dim == 2:
        data[2, :] = 0
    else:
        data[1, 1, :] = 0
    return maps.GridMap(origin, nd, 1.0, data.reshape(-1))


def _refine_check(m, dim, U, params, plan_control, lengths, control, yaw_control, trig=False, start_yaw=None):
    pl, op = make_pair(m, dim, params, U)
    if trig:
        op.set_param("trig_mode", 1)
    row = 2.5 if dim == 2 else 1.5
    n, max_seg = len(lengths), 320
    P = np.zeros((n, dim))
    P[:, 0] = 0.5
    P[:, 1:] = row
    G = P.copy()
    G[:, 0] += lengths
    P += m.origin
    G += m.origin
    sg, so = waypoint_pair(P, plan_control, yaw=start_yaw)
    gg, go = waypoint_pair(G, plan_control)
    res, acts, segs = pl.plan_batch(sg, gg, max_seg=max_seg, want_states=True)
    coefs, nseg = pl.refine_trajectories(res, acts, segs, plan_control, control, yaw_control)
    st = traj_solver.last_stats()
    c = types.SimpleNamespace(dim=dim, control=plan_control)
    for i in range(n):
        r = op.plan(so[i:i + 1], go[i:i + 1])
        ns = int(r["n_seg"])
        assert r["status"] == 0 and res[i]["status"] == 0 and int(res[i]["n_seg"]) == ns, (i, r, res[i])
        if plan_control == VEL:
            assert ns == lengths[i], (i, ns)  # the length the case intends
        oa = op.actions(ns)
        assert np.array_equal(acts[i, :ns], oa)
        w = _refine_waypoints(c, op, oa, op.seg_states(ns), ns)
        exp = oracle.traj_solve(dim, control, w, np.full(ns, params["dt"]), yaw_control)
        assert nseg[i] == ns and np.array_equal(coefs[i, :ns], exp), i
        assert not coefs[i, ns:].any()
    return res, st


def test_refine_long_plans_2d():
    m = _corridor(2, 270, (0.0, 0.0))
    lengths = [55, 90, 135, 265]
    res, st = _refine_check(m, 2, maps.make_U(1.0, 1, 2), dict(v_max=1.0, dt=1.0, tol_pos=0.5), mp.VEL, lengths, JRK, VEL)
    assert st["max_wp"] == 266 and st["pos_global"] == 4 and st["n_traj"] == 4  # W = 56 .. 266: past 50, 129 and 258


def test_refine_long_plan_3d_far_origin():
    m = _corridor(3, 120, (5.0e6, 4.0e6, 10.0))
    _, st = _refine_check(m, 3, maps.make_U(1.0, 1, 3), dict(v_max=1.0, dt=1.0, tol_pos=0.5), mp.VEL, [40, 100], JRK, ACC)
    assert st["max_wp"] == 101 and st["pos_global"] == 1 and st["pos_shared"] == 1


def test_refine_yaw_and_snp_plans():
    m = _corridor(2, 80, (0.0, 0.0))
    U = np.array([[dx, dy, dyaw] for dx in (-1.0, 0.0, 1.0) for dy in (-1.0, 0.0, 1.0) for dyaw in (-0.4, 0.0, 0.4)])
    _, st = _refine_check(m, 2, U, dict(dt=1.0, tol_pos=0.5, yaw_max=0.9, w=10.0, v_max=1.0), mp.VELxYAW, [30, 60], ACC, JRK,
                          trig=True, start_yaw=0.3)
    assert st["max_wp"] >= 31
    Ux = np.array([[-1.0, 0.0], [0.0, 0.0], [1.0, 0.0]])  # snap along the corridor only
    _, st = _refine_check(m, 2, Ux, dict(v_max=2.0, a_max=1.0, j_max=1.0, dt=1.0, tol_pos=0.5, max_num=20000), mp.SNP, [8, 14],
                          JRK, VEL)
    assert st["n_traj"] == 2


def test_refine_device_on_a_side_stream():
    """plan_batch_device -> mplb_refine_trajectories_device on one side stream equals the host path."""
    m = _corridor(2, 140, (0.0, 0.0))
    pl, _ = make_pair(m, 2, dict(v_max=1.0, dt=1.0, tol_pos=0.5), maps.make_U(1.0, 1, 2))
    lengths = np.array([3, 60, 135, 1])
    P = np.tile([0.5, 2.5], (4, 1))
    G = P + np.stack([lengths, 0 * lengths], axis=1)
    G[3] = (0.5, 0.5)  # inside the wall: a failed plan
    sg, gg = mp.waypoints_array(4), mp.waypoints_array(4)
    sg["pos"][:, :2], gg["pos"][:, :2] = P, G
    sg["control"] = gg["control"] = mp.VEL
    max_seg = 320
    res, acts, segs = pl.plan_batch(sg, gg, max_seg=max_seg, want_states=True)
    want_c, want_n = pl.refine_trajectories(res, acts, segs, mp.VEL, mp.JRK, mp.ACC)
    assert list(want_n) == [3, 60, 135, 0]
    s = torch.cuda.Stream()
    d_s, d_g = _to_dev(sg), _to_dev(gg)
    d_res = torch.zeros(4 * _lib.RESULT_DTYPE.itemsize, dtype=torch.uint8, device="cuda")
    d_act = torch.zeros(4 * max_seg, dtype=torch.int32, device="cuda")
    d_seg = torch.zeros(4 * max_seg * 13, dtype=torch.float64, device="cuda")
    d_coefs = torch.full((4, max_seg, 3, 6), 5.0, dtype=torch.float64, device="cuda")
    s.wait_stream(torch.cuda.current_stream())
    nseg = np.full(4, -1, dtype=np.int32)
    with torch.cuda.stream(s):
        pl.plan_batch_device(d_s.data_ptr(), d_g.data_ptr(), 4, d_res.data_ptr(), d_act.data_ptr(), d_seg.data_ptr(), max_seg,
                             s.cuda_stream)
        _lib.check(_lib.lib().mplb_refine_trajectories_device(pl._h, C.c_void_p(d_res.data_ptr()), C.c_void_p(d_act.data_ptr()),
                                                              C.c_void_p(d_seg.data_ptr()), 4, max_seg, mp.VEL, mp.JRK, mp.ACC,
                                                              C.c_void_p(d_coefs.data_ptr()), _lib.ptr(nseg), C.c_void_p(s.cuda_stream)))
    torch.cuda.current_stream().wait_stream(s)
    assert list(nseg) == list(want_n)
    assert np.array_equal(d_coefs.cpu().numpy(), want_c)
    assert traj_solver.last_stats()["max_wp"] == 136


# ---- refusal

def test_work_space_past_8_gib_is_refused():
    W = 2
    while (E.ws_doubles(W, 6, 3) + E.ws_doubles(W, 6, 1)) * 8 <= 8 << 30:
        W += 64
    while (E.ws_doubles(W - 1, 6, 3) + E.ws_doubles(W - 1, 6, 1)) * 8 > 8 << 30:
        W -= 1
    assert 7000 < W < 8000
    rs = np.random.RandomState(4)
    w, d = E.make_list(rs, 3, W, JRK)
    with pytest.raises(mp.MplbError, match="error -4"):
        traj_solver.solve_batch(3, JRK, [w], [d], JRK)
    assert traj_solver.last_stats()["n_traj"] == 0
    c = next(x for x in CASES if x.name == "flags_alternating_3d")
    got = traj_solver.solve_batch(3, JRK, [c.wps], [c.dts], ACC)[0]
    assert np.array_equal(got, want(c))
    assert traj_solver.last_stats()["n_traj"] == 1
