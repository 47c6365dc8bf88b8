"""The search kernel at its capacity edges, against the oracle with tolerance 0 (problems: capacity_cases.py).

These paths run only once a plan outgrows a fixed size, so each case first asserts -- through
MapPlanner.last_batch_tiers() and the oracle's peaks (largest node count, heap size and predecessor-record count at the
start of an expansion, where the kernel checks its arena) -- that it took the branch it is named for:
  - the shared-memory heap top and its global spill: 512 entries (|U| <= 32, every plain and shaped (DIM, ORD) cell),
    1024 entries (|U| > 32 with more plans resident than SMs) and the large one-plan-per-SM top (|U| > 32, single plans
    or few slots); MaxExpandStep stops with deep heaps and exhausted rooms whose peak heap passed the top;
  - arena tiers: overflow and re-run at 8x the capacity, the straight-to-bound tier of a MaxExpandStep batch, tiers above
    262144 nodes with load factor 1/2, predecessor-log overflow while the nodes still fit, the longest-first work list;
  - MPLB_PLAN_NOMEM: a fully defined record (host and device entry points, stale buffers underneath) and getters that
    refuse a retained NOMEM plan;
  - arena slots that run plan after plan (max_slots 1 and 3).
Every plan is compared with the oracle in every RESULT_FIELDS field and its action row.  Retained single plans also
compare the pop sequence, every node, and the heap array (getOpenSet's ids against orc_get_heap, in array order).  A
|U| > 32 plan can only be retained as a single plan, which always runs with the large heap top: the 1024-entry regime is
compared through batches only.  Arena budgets are capped with setArenaBytes (a few GB at most), so which tier fits does
not depend on how much memory other users of the GPU leave free.  The last test prints one row per (branch, cell)."""
import collections

import numpy as np
import pytest

import mpl_ros_b200 as mp
from mpl_ros_b200 import _lib, maps
import capacity_cases as K
from fuzz_cases import cell_name
from helpers_gpu import RESULT_FIELDS, assert_results_equal
from test_gpu_yaw import _full_compare

pytestmark = pytest.mark.gpu

ARENA = 3 << 30  # arena budget bound of every planner here (bytes)
MAX_SEG = 8
ROWS = collections.OrderedDict()  # (branch, cell) -> Counter(plans, tiers, hcap, heap, overflow, nomem, reached)


def _row(branch, cell):
    return ROWS.setdefault((branch, cell), collections.Counter())


def _note(row, plans, tiers, peaks, hcap=None):
    row["plans"] += plans
    row["tiers"] = max(row["tiers"], len(tiers))
    row["hcap"] = max(row["hcap"], hcap if hcap is not None else max(t["hcap"] for t in tiers))
    row["heap"] = max([row["heap"]] + [p["heap"] for p in peaks])
    row["overflow"] += sum(t["n_overflow"] for t in tiers)
    row["nomem"] += sum(t["n_work"] for t in tiers if t["nomem"])


def _gpu(P, arena=ARENA, max_slots=0):
    pl = P.gpu()
    pl.setArenaBytes(arena)
    pl.setMaxSlots(max_slots)
    return pl


def _open_ids(pl):
    n = _lib.check(_lib.lib().mplb_get_open(pl._h, None, 0))
    ids = np.zeros(max(n, 1), np.int32)
    _lib.check(_lib.lib().mplb_get_open(pl._h, _lib.ptr(ids), ids.size))
    return ids[:n]


def _assert_nomem(r, row, ctx):
    """the MPLB_PLAN_NOMEM record: n_seg 0, cost +inf, every counter, hash and device_ms 0, action row all -1"""
    assert r["status"] == K.NOMEM and r["n_seg"] == 0 and r["cost"] == np.inf, (ctx, r)
    for f in RESULT_FIELDS[3:] + ("device_ms",):
        assert r[f] == 0, (ctx, f, r[f])
    if row is not None:
        assert (np.asarray(row) == -1).all(), (ctx, row)


def _batch(P, S, G, ctx, nomem=(), max_seg=MAX_SEG):
    """S, G as one batch on P's planner: every plan equals the oracle's except the indices in `nomem`, which carry the
    NOMEM record.  Returns (results, tiers, oracle peaks per plan)."""
    pl = P.gpu()
    sg, gg, _, _ = P.waypoints(S, G)
    rg, ag, _ = pl.plan_batch(sg, gg, max_seg=max_seg)
    peaks = []
    for i in range(len(S)):
        ro, row, pk, _ = P.single(S[i], G[i], max_seg)
        peaks.append(pk)
        if i in nomem:
            _assert_nomem(rg[i], ag[i], (ctx, i))
        else:
            assert_results_equal(rg[i], ro, (ctx, i))
            assert np.array_equal(ag[i], row), (ctx, i, ag[i], row)
    return rg, pl.last_batch_tiers(), peaks


def _overflowing(P, peaks, tier):
    return {i for i, pk in enumerate(peaks) if P.overflows(pk, tier["cap"], tier["log_cap"])}


def _single(P, s, g, ctx):
    """a retained single plan: result, pop sequence, every node, actions and segment states (test_gpu_yaw._full_compare),
    then the heap array key for key.  Returns (result, tiers, oracle peaks)."""
    pl, op = P.gpu(), P.oracle()
    sg, gg, so, go = P.waypoints(s, g)
    order = {mp.VEL: 1, mp.ACC: 2, mp.JRK: 3, mp.SNP: 4}[P.control & 15]
    rg = _full_compare(pl, op, sg, gg, so, go, ctx, 3 * order)
    oh = op.heap()
    ids = _open_ids(pl)
    assert len(ids) == len(oh) == rg["n_open"], (ctx, len(ids), len(oh))
    assert np.array_equal(pl.getNodes()["key"][ids], oh["key"]), (ctx, "heap array")
    return rg, pl.last_batch_tiers(), op.peaks()


# ---------------------------------------------------------------------------------------------------- heap regimes
@pytest.mark.parametrize("dim,order,shaped", [(d, o, s) for s in (False, True) for d in (2, 3) for o in (1, 2, 3, 4)])
def test_heap_top_512(dim, order, shaped):
    """(a) |U| <= 32: a fixed 512-entry top.  Single retained plans (heap array, nodes, pop log) with epsilon 0, 1, 2.5
    stopped by MaxExpandStep with heaps above 512; on VEL also exhausted rooms whose peak heap passed 512; then the same
    queries in a batch with near goals."""
    cell = cell_name((dim, order, 1, shaped))
    row = _row("heap top 512", cell)
    deep_final = 0
    for eps in (0.0, 1.0, 2.5):
        for exhaust in ((False, True) if order == 1 else (False,)):
            P, (s, g) = K.heap_cell(dim, order, shaped, eps, exhaust)
            _gpu(P)
            ctx = (cell, eps, exhaust)
            rg, tiers, pk = _single(P, s, g, ctx)
            assert all(t["hcap"] == 512 for t in tiers) and tiers[-1]["n_overflow"] == 0, (ctx, tiers)
            # epsilon > 1 keeps a predecessor log: the exhausted rooms re-expand nodes and outgrow its records
            assert [t["n_overflow"] for t in tiers[:-1]] == [1] * (len(tiers) - 1), (ctx, tiers)
            assert all(P.overflows(pk, t["cap"], t["log_cap"]) for t in tiers[:-1]), (ctx, tiers, pk)
            assert not P.overflows(pk, tiers[-1]["cap"], tiers[-1]["log_cap"]), (ctx, tiers, pk)
            assert pk["heap"] > 512, (ctx, pk)
            assert rg["status"] == (3 if exhaust else 2), (ctx, rg["status"])
            deep_final += int(rg["n_open"] > 512)
            _note(row, 1, tiers, [pk])
            S, G = K.near_queries(P, 5, seed=dim * 10 + order)
            S, G = np.vstack([[s], S, [s]]), np.vstack([[g], G, [g]])
            _, tiers, peaks = _batch(P, S, G, ctx + ("batch",))
            assert all(t["hcap"] == 512 for t in tiers), tiers
            _note(row, len(S), tiers, peaks)
    assert deep_final > 0, cell  # some plan ended with entries at and beyond position 512: the end-of-plan copy ran
    row["reached"] = 1


def _box_125(ctl, eps, max_num, L=30):
    m, rooms = K.box_3d(L)
    params = dict(v_max=1.0, a_max=1.0, j_max=1.0, dt=1.0, tol_pos=0.5, epsilon=eps)
    if max_num:
        params["max_num"] = max_num
    return K.Problem(m, 3, params, maps.make_U(1.0, 2, 3), ctl), rooms


def _box_queries(m, rooms, n, seed):
    """n starts on free cells of the cube, goals in the walled-off column (unreachable)"""
    rs = np.random.RandomState(seed)
    L = rooms[0][3]
    cells = rs.randint(1, 1 + L, size=(n, 3))
    return m.int_to_float(cells), np.repeat([K.centre(m, rooms[1])], n, axis=0)


def test_heap_top_1024_batches():
    """(b) |U| > 32 in batches larger than the SM count: the 1024-entry top.  3D ACC |U| = 125 stopped by MaxExpandStep
    (epsilon 0, 1, 2.5), and 2D VEL |U| = 49 exhausting rooms with peak heaps above 1024 among near goals."""
    for eps in (0.0, 1.0, 2.5):
        P, rooms = _box_125(mp.ACC, eps, 60)
        _gpu(P)
        S, G = _box_queries(P.m, rooms, 140, seed=int(eps * 10))
        _, tiers, peaks = _batch(P, S, G, ("1024", eps))
        assert tiers[0]["slots"] > 132 and all(t["hcap"] == 1024 for t in tiers), tiers
        assert max(p["heap"] for p in peaks) > 1024, max(p["heap"] for p in peaks)
        _note(_row("heap top 1024", "3D-ACC-Ugt32"), len(S), tiers, peaks)
    P, rooms = K.vel_rooms([150, 40, 12], nu_class=4)
    _gpu(P)
    S, G = K.room_queries(P.m, rooms, [(0, "exhaust")] * 4 + [(i % 3, "near") for i in range(136)])
    _, tiers, peaks = _batch(P, S, G, ("1024", "exhausted"))
    assert tiers[0]["slots"] > 132 and all(t["hcap"] == 1024 for t in tiers), tiers
    assert peaks[0]["heap"] > 1024, peaks[0]
    _note(_row("heap top 1024", "2D-VEL-Ugt32 exhausted"), len(S), tiers, peaks)
    for k in ("3D-ACC-Ugt32", "2D-VEL-Ugt32 exhausted"):
        _row("heap top 1024", k)["reached"] = 1


def test_heap_top_large():
    """(c) |U| > 32 with one plan per SM: single retained plans (heap array, nodes, pop log) of 3D |U| = 125 whose heaps
    pass the large top -- MaxExpandStep stops and an exhausted cube -- and a batch with max_slots below the SM count."""
    row = _row("heap top large", "3D-Ugt32")
    hcaps = {}
    for ctl, eps, mx in ((mp.ACC, 0.0, 1000), (mp.JRK, 1.0, 1500), (mp.ACC, 2.5, 20000), (mp.VEL, 0.0, 0)):
        P, rooms = _box_125(ctl, eps, mx)
        _gpu(P)
        ctx = ("large", ctl, eps)
        s, g = K.centre(P.m, rooms[0]), K.centre(P.m, rooms[1])
        rg, tiers, pk = _single(P, s, g, ctx)
        hcap = hcaps[ctl] = tiers[0]["hcap"]  # the instantiation's shared-memory room decides it
        assert len(tiers) == 1 and hcap > 1024, (ctx, tiers)
        assert pk["heap"] > hcap and rg["status"] == (2 if mx else 3), (ctx, pk, rg["status"])
        if mx and eps < 2:  # past twice the top: pushes whose parents live in the spill go through the ancestor cache
            assert pk["heap"] > 2 * hcap, (ctx, pk)
        _note(row, 1, tiers, [pk])
    P, rooms = _box_125(mp.JRK, 1.0, 500)
    _gpu(P, max_slots=16)
    S, G = _box_queries(P.m, rooms, 24, seed=4)
    _, tiers, peaks = _batch(P, S, G, ("large", "max_slots 16"))
    assert tiers[0]["slots"] == 16 and tiers[0]["hcap"] == hcaps[mp.JRK], (tiers, hcaps)
    assert max(p["heap"] for p in peaks) > hcaps[mp.JRK]
    _note(row, len(S), tiers, peaks)
    row["reached"] = 1


# ---------------------------------------------------------------------------------------------------- arena tiers
TIER_ROOMS = [181, 180, 150, 190, 20, 8]  # 181 and 190 outgrow the first tier, 180 just fits


def _tier_problem():
    P, rooms = K.vel_rooms(TIER_ROOMS)
    picks = [(r, "exhaust") for r in range(len(rooms))] + [(r, "near") for r in range(len(rooms))]
    return P, rooms, picks


def test_tiers_without_max_num():
    """No MaxExpandStep: the first tier holds 32768 nodes; exactly the plans the oracle's peaks say outgrow it run again in
    a 262144-node tier.  A small batch takes plans in query order, one larger than half the resident CTAs longest-first."""
    P, rooms, picks = _tier_problem()
    _gpu(P)
    S, G = K.room_queries(P.m, rooms, picks)
    _, tiers, peaks = _batch(P, S, G, "tiers identity")
    over = _overflowing(P, peaks, tiers[0])
    assert tiers[0]["cap"] == K.TIER0 and tiers[0]["ordered"] == 0 and len(over) == 2, (tiers, over)
    assert tiers[0]["n_overflow"] == len(over) and len(tiers) == 2, tiers
    assert tiers[1]["cap"] == 262144 and tiers[1]["n_work"] == len(over) and tiers[1]["n_overflow"] == 0, tiers
    assert tiers[1]["load_inv"] == 4 and tiers[1]["ordered"] == 1, tiers
    _note(_row("tier 32768 -> 262144", "query order"), len(S), tiers, peaks)
    n = tiers[0]["resident"] // 2 + 1
    S, G = np.resize(S, (n, 2)), np.resize(G, (n, 2))
    _, tiers, peaks = _batch(P, S, G, "tiers longest-first")
    over = _overflowing(P, peaks, tiers[0])
    assert tiers[0]["ordered"] == 1 and tiers[0]["n_overflow"] == len(over) > 2 and len(tiers) == 2, (tiers, len(over))
    assert tiers[1]["cap"] == 262144 and tiers[1]["n_work"] == len(over) and tiers[1]["n_overflow"] == 0, tiers
    _note(_row("tier 32768 -> 262144", "longest-first"), len(S), tiers, peaks)
    _row("tier 32768 -> 262144", "query order")["reached"] = _row("tier 32768 -> 262144", "longest-first")["reached"] = 1


def test_tiers_above_262144_with_max_num():
    """MaxExpandStep bound above 262144 nodes (2D VEL |U| = 9, max_num 300000: bound 2700082): the first tier holds
    262144 nodes, the second has load factor 1/2 and holds 8x as many when at most half the plans overflowed, the whole
    bound when more did."""
    m, rooms = K.rooms_2d([530, 520, 10])
    P = K.Problem(m, 2, dict(v_max=0.5, dt=1.0, tol_pos=0.5, max_num=300000), maps.make_U(0.5, 1, 2), mp.VEL)
    _gpu(P)
    bound = 300000 * 9 + 2 * 9 + 64
    for picks, cap2, name in (([(0, "exhaust"), (2, "near")], 8 * 262144, "8x"),
                              ([(0, "exhaust"), (1, "exhaust"), (2, "near")], bound, "straight to bound")):
        S, G = K.room_queries(m, rooms, picks)
        _, tiers, peaks = _batch(P, S, G, ("bound", name))
        over = _overflowing(P, peaks, tiers[0])
        assert tiers[0]["cap"] == 262144 and tiers[0]["n_overflow"] == len(over) == len(picks) - 1, (tiers, over)
        assert len(tiers) == 2 and tiers[1]["cap"] == cap2 and tiers[1]["load_inv"] == 2 and tiers[1]["n_overflow"] == 0, tiers
        _note(_row("tier 262144 -> " + name, "2D-VEL-Ule32"), len(S), tiers, peaks)
        _row("tier 262144 -> " + name, "2D-VEL-Ule32")["reached"] = 1


def test_tiers_predecessor_log_overflow():
    """Predecessor-log mode (setExactPreds(1)): rooms of 10000 and 14400 nodes fit the 32768-node tier but not its
    6 * 32768 + |U| predecessor records; exactly those plans run again."""
    P, rooms = K.vel_rooms([120, 100, 60, 10])
    P.exact_preds = 1
    _gpu(P)
    S, G = K.room_queries(P.m, rooms, [(r, "exhaust") for r in range(4)] + [(r, "near") for r in range(4)])
    _, tiers, peaks = _batch(P, S, G, "log")
    t0 = tiers[0]
    assert t0["cap"] == K.TIER0 and t0["log_cap"] == 6 * K.TIER0 + P.nU, t0
    over = _overflowing(P, peaks, t0)
    assert over == {0, 1} and all(peaks[i]["nodes"] + P.nU <= K.TIER0 for i in over), (over, peaks[:2])
    assert t0["n_overflow"] == 2 and len(tiers) == 2 and tiers[1]["n_overflow"] == 0, tiers
    _note(_row("predecessor log overflow", "2D-VEL-Ule32"), len(S), tiers, peaks)
    _row("predecessor log overflow", "2D-VEL-Ule32")["reached"] = 1


def test_retained_plan_through_second_tier():
    """A retained single plan that outgrows the first tier (epsilon 0 across a 190-cell room to a reachable far corner):
    nodes, pop sequence and heap array read from the 262144-node tier's arena."""
    P, rooms = K.vel_rooms([190, 10], epsilon=0.0)
    _gpu(P)
    x, y, s = rooms[0]
    rg, tiers, pk = _single(P, P.m.int_to_float([x + 2, y + 2]), P.m.int_to_float([x + s - 3, y + s - 3]), "retained tier 2")
    assert rg["status"] == 0 and rg["n_open"] > 0, rg
    assert len(tiers) == 2 and tiers[0]["n_overflow"] == 1 and tiers[1]["cap"] == 262144, tiers
    assert P.overflows(pk, K.TIER0, 0), pk
    _note(_row("retained through tier 2", "2D-VEL-Ule32"), 1, tiers, [pk])
    _row("retained through tier 2", "2D-VEL-Ule32")["reached"] = 1


# ---------------------------------------------------------------------------------------------------- NOMEM
def test_nomem_below_first_tier():
    """A budget below one slot of the first tier: every plan gets the NOMEM record, through plan_batch after a successful
    batch on the same planner (its buffers hold that batch's records) and through plan_batch_device over buffers filled
    with a sentinel.  The planner plans normally again once the budget allows."""
    import torch
    P, rooms, picks = _tier_problem()
    pl = _gpu(P)
    S, G = K.room_queries(P.m, rooms, picks)
    _, tiers, _ = _batch(P, S, G, "before nomem")
    stride = tiers[0]["stride_bytes"]
    pl.setArenaBytes(stride - 1)
    sg, gg, _, _ = P.waypoints(S, G)
    rg, ag, _ = pl.plan_batch(sg, gg, max_seg=MAX_SEG)
    for i in range(len(S)):
        _assert_nomem(rg[i], ag[i], ("host", i))
    tiers = pl.last_batch_tiers()
    assert len(tiers) == 1 and tiers[0]["nomem"] == 1 and tiers[0]["n_work"] == len(S) and tiers[0]["slots"] == 0, tiers
    n = len(S)
    d_s, d_g = (torch.from_numpy(w.view(np.uint8)).cuda() for w in (sg, gg))
    d_r = torch.full((n * _lib.RESULT_DTYPE.itemsize,), 0x5A, dtype=torch.uint8, device="cuda")
    d_a = torch.full((n, MAX_SEG), 7, dtype=torch.int32, device="cuda")
    pl.plan_batch_device(d_s.data_ptr(), d_g.data_ptr(), n, d_r.data_ptr(), d_a.data_ptr(), 0, MAX_SEG)
    rd, ad = d_r.cpu().numpy().view(_lib.RESULT_DTYPE), d_a.cpu().numpy()
    for i in range(n):
        _assert_nomem(rd[i], ad[i], ("device", i))
    _note(_row("nomem below tier 1", "2D-VEL-Ule32"), 2 * n, pl.last_batch_tiers(), [])
    pl.setArenaBytes(ARENA)
    _batch(P, S, G, "after nomem")
    _row("nomem below tier 1", "2D-VEL-Ule32")["reached"] = 1


def test_nomem_between_tiers():
    """A budget that holds two slots of the first tier and no slot of the second: exactly the plans the oracle says
    outgrow the first tier report NOMEM, every other plan equals the oracle."""
    P, rooms, picks = _tier_problem()
    pl = _gpu(P)
    S, G = K.room_queries(P.m, rooms, picks)
    _, tiers, peaks = _batch(P, S, G, "strides")
    s1, s2 = tiers[0]["stride_bytes"], tiers[1]["stride_bytes"]
    assert 2 * s1 < s2, (s1, s2)
    over = _overflowing(P, peaks, tiers[0])
    pl.setArenaBytes(2 * s1)
    _, tiers, _ = _batch(P, S, G, "between", nomem=over)
    assert tiers[0]["slots"] == 2 and tiers[0]["n_overflow"] == len(over) == 2, tiers
    assert len(tiers) == 2 and tiers[1]["nomem"] == 1 and tiers[1]["n_work"] == len(over), tiers
    _note(_row("nomem in tier 2", "2D-VEL-Ule32"), len(S), tiers, peaks)
    _row("nomem in tier 2", "2D-VEL-Ule32")["reached"] = 1


def test_retained_nomem_plan():
    """A retained plan that ends in NOMEM -- as a planner's first plan (budget below one slot) and after overflowing the
    first tier (budget between the tiers) -- has the NOMEM record and no search state: the node, pop-log and open-set
    getters fail with MPLB_ERR_STATE.  The next plan on the same planner and its getters are correct."""
    P, rooms, _ = _tier_problem()
    pl = _gpu(P, arena=1 << 16)
    big = (K.centre(P.m, rooms[0]), K.centre(P.m, rooms[1]))  # 181: overflows the first tier
    fits = (K.centre(P.m, rooms[2]), K.centre(P.m, rooms[3]))  # 150
    sg, gg, _, _ = P.waypoints(*big)
    for arena in (1 << 16, "between tiers"):
        if arena != 1 << 16:
            arena = 2 * pl.last_batch_tiers()[0]["stride_bytes"]  # of the fitting plan just before
        pl.setArenaBytes(arena)
        assert not pl.plan(sg, gg)
        _assert_nomem(pl.result(), pl.getActions(), ("retained", arena))
        assert len(pl.getActions()) == 0 and len(pl.getSegStates()) == 0
        tiers = pl.last_batch_tiers()
        assert tiers[-1]["nomem"] == 1 and len(tiers) == (1 if arena == 1 << 16 else 2), tiers
        for get in (pl.getNodes, pl.getPopLog, pl.getOpenSet):
            with pytest.raises(mp.MplbError, match="mplb error -3: .*NOMEM"):
                get()
        pl.setArenaBytes(ARENA)
        _single(P, *fits, ("after nomem", arena))
    _row("retained nomem", "2D-VEL-Ule32").update(plans=4, nomem=2, reached=1)


# ---------------------------------------------------------------------------------------------------- slot reuse
@pytest.mark.parametrize("max_slots", [1, 3])
@pytest.mark.parametrize("nu_class", [1, 4])
def test_slot_reuse(max_slots, nu_class):
    """Few CTAs run plan after plan in one arena slot: big tables followed by small ones, exhausted searches by early
    goals, overflowing plans by fitting ones (no MaxExpandStep; 2D VEL with |U| = 25 or 49)."""
    P, rooms = K.vel_rooms([181, 150, 60, 20, 8], nu_class=nu_class)
    _gpu(P, max_slots=max_slots)
    picks = [(1, "exhaust"), (4, "near"), (2, "exhaust"), (1, "near"), (0, "exhaust"), (3, "exhaust"), (2, "near"),
             (1, "exhaust"), (3, "near"), (4, "exhaust"), (0, "near"), (0, "exhaust"), (4, "exhaust")]
    S, G = K.room_queries(P.m, rooms, picks)
    _, tiers, peaks = _batch(P, S, G, ("slots", max_slots, nu_class))
    assert tiers[0]["slots"] == max_slots and tiers[0]["n_overflow"] == len(_overflowing(P, peaks, tiers[0])) > 0, tiers
    cell = "2D-VEL-U%s" % ("le32" if nu_class == 1 else "gt32")
    row = _row("slot reuse, max_slots %d" % max_slots, cell)
    _note(row, len(S), tiers, peaks)
    row["reached"] = 1


# ---------------------------------------------------------------------------------------------------- coverage
EXPECTED = ([("heap top 512", cell_name((d, o, 1, s))) for s in (False, True) for d in (2, 3) for o in (1, 2, 3, 4)] +
            [("heap top 1024", "3D-ACC-Ugt32"), ("heap top 1024", "2D-VEL-Ugt32 exhausted"), ("heap top large", "3D-Ugt32"),
             ("tier 32768 -> 262144", "query order"), ("tier 32768 -> 262144", "longest-first"),
             ("tier 262144 -> 8x", "2D-VEL-Ule32"), ("tier 262144 -> straight to bound", "2D-VEL-Ule32"),
             ("predecessor log overflow", "2D-VEL-Ule32"), ("retained through tier 2", "2D-VEL-Ule32"),
             ("nomem below tier 1", "2D-VEL-Ule32"), ("nomem in tier 2", "2D-VEL-Ule32"), ("retained nomem", "2D-VEL-Ule32")] +
            [("slot reuse, max_slots %d" % k, "2D-VEL-U%s" % c) for k in (1, 3) for c in ("le32", "gt32")])


def test_every_branch_ran(capsys):
    lines = ["%-34s %-24s %6s %5s %5s %7s %8s %6s" % ("branch", "cell", "plans", "tiers", "hcap", "heap", "overflow", "nomem")]
    for (b, c), r in ROWS.items():
        lines.append("%-34s %-24s %6d %5d %5d %7d %8d %6d" % (b, c, r["plans"], r["tiers"], r["hcap"], r["heap"], r["overflow"],
                                                              r["nomem"]))
    with capsys.disabled():
        print("\n" + "\n".join(lines))
    missing = [k for k in EXPECTED if not ROWS.get(k, {}).get("reached")]
    assert not missing, missing
