"""Search region, potential map and yaw controls on control sets of more than 32 rows: the |U| > 32 cost-shaping kernels
(astar_batch_kernel<DIM, ORD, 4, true>) against the oracle with tolerance 0.

tests/fuzz_cases.py's module docstring predates these kernels: shaped plans with more than 32 rows now launch the shaped
MAXU = 4 instantiation, which fuzz_cases.instantiation() already reports as (dim, ord, 4, True).

Yaw comparisons run the oracle in the correctly rounded cos/sin definition (trig_mode 1, test_gpu_yaw.py); the oracle
in the libm definition equals the reference's own sources on the same configurations (tests/test_oracle_shaped_wide.py).
Single plans compare the result record, the pop order, every node with its yaw, actions and segment states
(test_gpu_yaw._full_compare); batches compare the result records and action rows.  Capacity cases assert the branch they
are named for through MapPlanner.last_batch_tiers() and the oracle's peaks, as tests/test_gpu_capacity.py does."""
import math

import numpy as np
import pytest

import mpl_ros_b200 as mp
from mpl_ros_b200 import maps
import capacity_cases as K
import fuzz_cases as F
from helpers import load_config
from helpers_gpu import assert_results_equal, make_pair, waypoint_pair
from test_gpu_capacity import _assert_nomem, _batch, _gpu, _single
from test_gpu_yaw import _full_compare
from test_oracle_shaped_wide import node_U_yaw

pytestmark = pytest.mark.gpu

SM_COUNT = 132  # H100 SXM


def _ncell(m):
    return int(np.prod(np.asarray(m.dim, dtype=np.int64)))


def _wide_tier(pl):
    tiers = pl.last_batch_tiers()
    assert len(tiers) >= 1 and all(256 <= t["hcap"] <= 8192 and t["hcap"] % 256 == 0 for t in tiers), tiers
    return tiers


# ---------------------------------------------------------------------------------------------------- node configurations
@pytest.mark.parametrize("name,yaw_max,wyaw", [("skir", 0.7, 1.0), ("skir", -1.0, 1.0), ("skir", 1.2, 0.0), ("levine", -1.0, 0.0)])
def test_node_3d_yaw_81_rows(name, yaw_max, wyaw):
    """map_planner_node with use_3d and use_yaw (81 rows, ACCxYAW): single retained plans."""
    U = node_U_yaw(1.0, 1, 0.3, 3)
    assert F.instantiation(3, mp.ACCxYAW, len(U), True) == (3, 2, 4, True)
    if name == "skir":
        m, dim, params, _, start, goal = load_config("skir")
    else:
        m, dim = maps.load_fixture("levine"), 3
        params = dict(v_max=2.0, a_max=1.0, dt=1.0, tol_pos=0.5)
        S, G = maps.sample_queries(m, 4, seed=21)
        start, goal = S[1], G[1]
    pl, op = make_pair(m, dim, dict(params, yaw_max=yaw_max, wyaw=wyaw), U)
    op.set_param("trig_mode", 1)
    sg, so = waypoint_pair(start, mp.ACCxYAW, yaw=0.4)
    gg, go = waypoint_pair(goal, mp.ACCxYAW)
    rg = _full_compare(pl, op, sg, gg, so, go, (name, yaw_max, wyaw), 6)
    assert rg["status"] == 0 or name == "levine"
    _wide_tier(pl)


def test_node_3d_yaw_81_rows_batch():
    """the same set as one batch of 64 levine queries with random start yaws"""
    m = maps.load_fixture("levine")
    U = node_U_yaw(1.0, 1, 0.3, 3)
    pl, op = make_pair(m, 3, dict(v_max=2.0, a_max=1.0, dt=1.0, tol_pos=0.5, yaw_max=1.0, wyaw=1.0), U)
    op.set_param("trig_mode", 1)
    n = 64
    S, G = maps.sample_queries(m, n, seed=17)
    yaws = np.random.default_rng(17).uniform(-3, 3, n)
    sg, so = waypoint_pair(S, mp.ACCxYAW, yaw=yaws)
    gg, go = waypoint_pair(G, mp.ACCxYAW)
    rg, ag, _ = pl.plan_batch(sg, gg, max_seg=64, want_states=True)
    ro, ao = op.plan_batch(so, go, nthreads=8, max_seg=64)
    for i in range(n):
        assert_results_equal(rg[i], ro[i], ("81-row yaw batch", i))
    assert np.array_equal(ag, ao)
    assert (ro["status"] == 0).sum() >= 8
    _wide_tier(pl)


@pytest.mark.parametrize("yaw_max,wyaw", [(0.7, 1.0), (-1.0, 1.0), (0.7, 0.0), (1.2, 2.5)])
def test_planner_2d_with_yaw_75_rows(yaw_max, wyaw):
    """test_planner_2d_with_yaw's flow on corridor.yaml with the node's num = 2 set (75 rows)"""
    m, dim, params, _, start, goal = load_config("corridor")
    U = node_U_yaw(0.5, 2, 0.5, 2)
    assert U.shape == (75, 3)
    pl, op = make_pair(m, dim, dict(params, yaw_max=yaw_max, wyaw=wyaw), U)
    op.set_param("trig_mode", 1)
    sg, so = waypoint_pair(start, mp.ACCxYAW, yaw=math.pi / 2)
    gg, go = waypoint_pair(goal, mp.ACCxYAW)
    rg = _full_compare(pl, op, sg, gg, so, go, ("75-row yaw", yaw_max, wyaw), 6)
    assert rg["status"] == 0


@pytest.mark.parametrize("num", [3, 4])
@pytest.mark.parametrize("grad_w", [0.0, 0.3])
def test_distance_map_flow_wide(num, grad_w):
    """distance_map_planner_node's flow with num = 3 / 4 (49 / 81 rows) on corridor.yaml: plain plan, search region
    around it, potential map, shaped plan; then iterativePlan"""
    m, dim, params, _, start, goal = load_config("corridor")
    U = maps.make_U(0.5, num, 2)
    pl, op = make_pair(m, dim, params, U)
    sg, so = waypoint_pair(start, mp.ACC)
    gg, go = waypoint_pair(goal, mp.ACC)
    rg = _full_compare(pl, op, sg, gg, so, go, ("plain", num), 6)
    assert rg["status"] == 0
    path = [np.array(w.pos, dtype=np.float64) for w in pl.getTraj().getWaypoints()]
    opath = np.zeros((len(path), 3))
    opath[:, :2] = np.array(path)
    mu, om = pl._keep

    pl2, op2 = make_pair(m, dim, dict(params, epsilon=1.0), U)
    pl2.setMapUtil(mu)
    op2.set_map(om)
    pl2.setSearchRadius([0.5, 0.5])
    op2.set_vec("search_radius", [0.5, 0.5, 0.0])
    pl2.setSearchRegion(path)
    op2.set_search_region(opath, dense=False)
    region = pl2.getSearchRegionMask()
    assert np.array_equal(region, op2.get_search_region(_ncell(m))) and 0 < region.sum() < region.size
    pl2.setPotentialRadius([1.0, 1.0])
    op2.set_vec("potential_radius", [1.0, 1.0, 0.0])
    pl2.setPotentialWeight(0.5)
    op2.set_param("potential_weight", 0.5)
    pl2.setGradientWeight(grad_w)
    op2.set_param("gradient_weight", grad_w)
    pl2.updatePotentialMap(start)
    op2.update_potential_map(np.array([start[0], start[1], 0.0]))
    assert np.array_equal(mu.getMap(), om.get_data(_ncell(m)))
    rg2 = _full_compare(pl2, op2, sg, gg, so, go, ("shaped", num, grad_w), 6)
    assert rg2["status"] == 0 and rg2["cost"] > rg["cost"]
    _wide_tier(pl2)

    raw = pl2.getTraj()
    assert pl2.iterativePlan(sg, gg, raw, 3)
    from mpl_ros_b200.planner import Primitive, Trajectory
    traj, prev = raw, 0.0
    for _ in range(3):
        op2.set_search_region(np.array([list(w.pos) + [0.0] for w in traj.getWaypoints()]), dense=False)
        ro = op2.plan(so, go)
        assert ro["status"] == 0
        acts, st = op2.actions(ro["n_seg"]), op2.seg_states(ro["n_seg"])
        traj = Trajectory([Primitive(dim, mp.ACC, st[i], U[acts[i]], params["dt"]) for i in range(len(acts))])
        if prev == ro["cost"]:
            break
        prev = ro["cost"]
    assert pl2.getTrajCost() == ro["cost"]
    assert_results_equal(pl2.result(), ro, ("iterative", num, grad_w))
    assert np.array_equal(pl2.getActions(), acts)


def test_jrk_125_rows_region_and_potential():
    """3D JRK with 125 rows on skir, stopped by MaxExpandStep: search regions (dense and not) around the straight line from
    start to goal, then a local-range potential map"""
    m, dim, params, _, start, goal = load_config("skir")
    U = maps.make_U(1.0, 2, 3)
    pl, op = make_pair(m, dim, dict(params, j_max=2.0, max_num=3000), U)
    mu, om = pl._keep
    sg, so = waypoint_pair(start, mp.JRK)
    gg, go = waypoint_pair(goal, mp.JRK)
    _full_compare(pl, op, sg, gg, so, go, "JRK 125 plain", 9)
    path = [start + (goal - start) * k / 8.0 for k in range(9)]
    for radius, dense in (([0.5, 0.5, 0.5], False), ([1.0, 1.0, 0.3], True)):
        pl.setSearchRadius(radius)
        op.set_vec("search_radius", radius)
        pl.setSearchRegion(path, dense)
        op.set_search_region(np.array(path), dense=dense)
        assert np.array_equal(pl.getSearchRegionMask(), op.get_search_region(_ncell(m)))
        _full_compare(pl, op, sg, gg, so, go, ("JRK 125 region", dense), 9)
        _wide_tier(pl)
    pl.setPotentialRadius([0.4, 0.4, 0.2])
    op.set_vec("potential_radius", [0.4, 0.4, 0.2])
    pl.setPotentialMapRange([3.0, 2.5, 1.0])
    op.set_vec("potential_map_range", [3.0, 2.5, 1.0])
    pl.setPotentialWeight(0.2)
    op.set_param("potential_weight", 0.2)
    pl.setGradientWeight(0.1)
    op.set_param("gradient_weight", 0.1)
    pl.updatePotentialMap(start)
    op.update_potential_map(np.asarray(start, dtype=np.float64))
    assert np.array_equal(mu.getMap(), om.get_data(_ncell(m)))
    _full_compare(pl, op, sg, gg, so, go, "JRK 125 region + potential", 9)


# ---------------------------------------------------------------------------------------------------- fuzz
WIDE_CELLS = [(dim, order, 4, True) for dim in (2, 3) for order in (1, 2, 3, 4)]
FUZZ_STATS = {}


def _widen(c, seed):
    """fuzz_cases.make_case for the matching |U| <= 32 shaped cell with a control set of 33..128 rows substituted"""
    rng = np.random.default_rng([seed, c.dim, 977])
    u = float(np.abs(c.U[:, :c.dim]).max())
    base = maps.make_U(u, 2, c.dim) if c.dim == 3 else maps.make_U(u, int(rng.choice([3, 4, 5])), 2)  # 125 / 49, 81, 121
    n = int(rng.integers(33, min(len(base), 128) + 1))
    U = base[np.sort(rng.choice(len(base), n, replace=False))]
    if c.control & 16:
        U = np.hstack([U, rng.choice([-0.5, 0.0, 0.5], size=(n, 1))])
    c.U = U
    if (c.control & 15) == mp.VEL and "v_max" in c.params and c.params["v_max"] < u:
        c.params["v_max"] = 0.75 * u  # keep the predecessor-log case where make_case drew it
    return c


@pytest.mark.parametrize("cell", WIDE_CELLS, ids=F.cell_name)
def test_fuzz_wide(cell):
    dim, order, _, _ = cell
    st = FUZZ_STATS.setdefault(cell, dict(plans=0, ok=0, met_obstacle=0))
    for seed in range(4):
        c = _widen(F.make_case((dim, order, 1, True), seed), seed)
        assert 33 <= len(c.U) <= 128 and c.cell == cell, (c.cell, len(c.U))
        ctx = (F.cell_name(cell), seed)
        pl, op = c.build()
        sg, so = c.waypoints(c.start, vel=c.vel, yaw=c.yaw)
        gg, go = c.waypoints(c.goal)
        rg = _full_compare(pl, op, sg, gg, so, go, ctx, 3 * order)
        st["plans"] += 1
        st["ok"] += int(rg["status"] == 0)
        st["met_obstacle"] += int(rg["n_valid"] < rg["n_prims"])
        sg, gg, so, go = c.batch_waypoints(seed)
        rb, ab, _ = pl.plan_batch(sg, gg, max_seg=c.max_seg, want_states=True)
        ro, ao = op.plan_batch(so, go, nthreads=8, max_seg=c.max_seg)
        for i in range(len(sg)):
            assert_results_equal(rb[i], ro[i], ctx + ("batch", i))
        assert np.array_equal(ab, ao), ctx
        st["plans"] += len(sg)
        st["ok"] += int((rb["status"] == 0).sum())
        st["met_obstacle"] += int((rb["n_valid"] < rb["n_prims"]).sum())
    assert st["ok"] > 0 and st["met_obstacle"] > 0, (cell, st)


# ---------------------------------------------------------------------------------------------------- capacity
def _vel49_shaped(sizes, **kw):
    P, rooms = K.vel_rooms(sizes, nu_class=4, **kw)
    P.shaped = True
    return P, rooms


def test_heap_regimes_and_spill():
    """Both heap-top regimes, each spilled past its top.  2D VEL, 49 rows, whole-map region and potential map: the term
    area is small enough for two plans per SM, so a batch larger than the SM count runs with the 1024-entry top.  3D ACC,
    125 rows, shaped: a single plan runs alone on its SM with the large top (test_gpu_capacity.test_heap_top_large's
    problem)."""
    P, rooms = _vel49_shaped([150, 40, 12])
    _gpu(P)
    S, G = K.room_queries(P.m, rooms, [(0, "exhaust")] * 4 + [(i % 3, "near") for i in range(136)])
    _, tiers, peaks = _batch(P, S, G, "wide shaped 1024")
    assert tiers[0]["resident"] >= 2 * SM_COUNT and tiers[0]["slots"] > SM_COUNT, tiers
    assert all(t["hcap"] == 1024 for t in tiers), tiers
    assert peaks[0]["heap"] > 1024, peaks[0]
    m, rooms = K.box_3d(30)
    P = K.Problem(m, 3, dict(v_max=1.0, a_max=1.0, dt=1.0, tol_pos=0.5, epsilon=0.0, max_num=1000), maps.make_U(1.0, 2, 3),
                  mp.ACC, shaped=True)
    _gpu(P)
    rg, tiers, pk = _single(P, K.centre(m, rooms[0]), K.centre(m, rooms[1]), "wide shaped large")
    assert len(tiers) == 1 and tiers[0]["hcap"] > 1024 and pk["heap"] > tiers[0]["hcap"], (tiers, pk)
    assert rg["status"] == 2, rg["status"]


def test_arena_overflow_rerun_and_log_mode():
    """an exhausted 181-cell room outgrows the first 32768-node tier and runs again; VEL with v_max below the control
    bound keeps predecessor records"""
    for kw in ({}, dict(v_max=1.0)):
        P, rooms = _vel49_shaped([181, 20], **kw)
        _gpu(P)
        S, G = K.room_queries(P.m, rooms, [(0, "exhaust"), (1, "near"), (1, "exhaust")])
        _, tiers, peaks = _batch(P, S, G, ("overflow", kw))
        assert len(tiers) >= 2 and tiers[0]["n_overflow"] >= 1, tiers
        assert P.overflows(peaks[0], tiers[0]["cap"], tiers[0]["log_cap"])
        assert (tiers[0]["log_cap"] > 0) == bool(kw), tiers


def test_nomem_record():
    """an arena budget below one slot of the first tier: every plan of the batch carries the NOMEM record"""
    P, rooms = _vel49_shaped([40, 12])
    pl = _gpu(P, arena=1 << 20)
    S, G = K.room_queries(P.m, rooms, [(0, "near"), (1, "near")])
    sg, gg, _, _ = P.waypoints(S, G)
    rg, ag, _ = pl.plan_batch(sg, gg, max_seg=8)
    for i in range(len(S)):
        _assert_nomem(rg[i], ag[i], ("nomem", i))
    assert pl.last_batch_tiers()[-1]["nomem"] == 1


def test_largest_term_area():
    """128 rows, 3D SNP with yaw, at the largest sample divisor the shaped kernels accept: 44 at res 0.1 (the fast
    sample-time table holds 1000 of its 1024 entries; divisor 45 would need 1045).  45 samples, 6 granules per control:
    128 * 48 (term, yaw term) pairs = 96 KB behind the heap.  The plan runs alone on its SM and its heap top is what the
    227 KB opt-in limit leaves: (232448 - 85152 (plan record) - 98304 - 1024) / 20, rounded down to 2304 entries."""
    m, rooms = K.box_3d(12, res=0.1)
    U = np.hstack([maps.make_U(1.0, 2, 3), np.zeros((125, 1))])
    U = np.vstack([U, [[1.0, 1.0, 1.0, 0.5], [-1.0, -1.0, -1.0, -0.5], [0.0, 0.0, 0.0, 0.5]]])
    assert len(U) == 128
    params = dict(v_max=4.25, a_max=2.0, j_max=2.0, dt=1.0, tol_pos=0.5, yaw_max=1.3, wyaw=1.0, max_num=300)
    pl, op = make_pair(m, 3, params, U)
    op.set_param("trig_mode", 1)
    s, g = K.centre(m, rooms[0]), K.centre(m, rooms[1])
    sg, so = waypoint_pair(s, mp.SNPxYAW, yaw=0.2)
    gg, go = waypoint_pair(g, mp.SNPxYAW)
    rg = _full_compare(pl, op, sg, gg, so, go, "largest term area", 12)
    assert rg["status"] in (2, 3) and rg["n_valid"] > 0, rg
    tiers = _wide_tier(pl)
    assert tiers[0]["hcap"] == 2304, tiers
