"""GPU results against the REFERENCE'S OWN planner sources directly (oracle/_ref/libmplref.so, see oracle/ref_harness.cpp),
without the oracle in between.  The library is built only where the reference tree exists; elsewhere the reference's side
is the value it returned when it was recorded (tests/ref_record.py).  Each test takes the reference's side first."""
import numpy as np
import pytest

import oracle
from oracle import ref
import mpl_ros_b200 as mp
from mpl_ros_b200 import maps
from helpers import load_config
import ref_record as R

pytestmark = pytest.mark.gpu

FIELDS = ("n_seg", "cost", "pops", "n_nodes", "n_open", "n_closed", "n_prims", "n_valid", "pop_hash", "closed_hash")


def _ref_planner(m, dim, params, U):
    if not R.LIVE:
        return R.Absent()
    rm = ref.RefMap(m.origin, m.dim, m.data, m.res)
    rm.free_unknown()
    rp = ref.RefPlanner(dim)
    rp.set_map(rm)
    for k, v in params.items():
        rp.set_param(k, v)
    rp.set_controls(U)
    rp._keep = rm
    return rp


def _gpu_planner(m, dim, params, U):
    mu = mp.MapUtil(dim)
    mu.setMap(m.origin, m.dim, m.data, m.res)
    mu.freeUnknown()
    pl = mp.MapPlanner(dim, False)
    pl.setMapUtil(mu)
    setters = dict(v_max="setVmax", a_max="setAmax", j_max="setJmax", dt="setDt", w="setW", epsilon="setEpsilon",
                   max_num="setMaxNum")
    for k, v in params.items():
        if k in setters:
            getattr(pl, setters[k])(v)
    pl.setTol(params.get("tol_pos", 0.5), params.get("tol_vel", -1), params.get("tol_acc", -1))
    pl.setU(U)
    pl._keep = mu
    return pl


def _wps(pos, control):
    a, b = mp.waypoints_array(len(np.atleast_2d(pos))), oracle.make_waypoints(len(np.atleast_2d(pos)))
    for w in (a, b):
        p = np.atleast_2d(np.asarray(pos, dtype=np.float64))
        w["pos"][:, :p.shape[1]] = p
        w["control"] = control
    return a, b


def _same(rg, rr, ctx):
    sg, sr = int(rg["status"]), int(rr["status"])
    assert sg == sr or (sr == -1 and sg in (2, 3, 4)), (ctx, sg, sr)
    for f in FIELDS:
        if f == "n_seg" and sg != 0:
            continue
        a, b = rg[f], rr[f]
        assert a == b or (f == "cost" and np.isinf(a) and np.isinf(b)), (ctx, f, a, b)


@pytest.mark.parametrize("name", ["corridor", "simple", "skir"])
def test_single_plans(name):
    m, dim, params, U, start, goal = load_config(name)
    rp = _ref_planner(m, dim, params, U)
    sg, sr = _wps(start, mp.ACC)
    gg, gr = _wps(goal, mp.ACC)
    rr = R.value("plan", lambda: rp.plan(sr, gr))
    pop_keys = R.value("pop_keys", lambda: R.digest(rp.pop_keys(rr["pops"])))
    # trajectory: coefficient rows of every primitive (what toTrajectoryROSMsg would publish)
    coeffs = R.value("coeffs", lambda: rp.traj_coeffs(rr["n_seg"]))
    if name == "corridor":
        assert rr["n_closed"] == 615 and rr["cost"] == 351.5  # MPL/README.md:200-202 out of the reference's own code
    pl = _gpu_planner(m, dim, params, U)
    pl.plan(sg, gg)
    rg = pl.result()
    _same(rg, rr, name)
    gn = pl.getNodes()
    assert str(R.digest(gn["key"][pl.getPopLog()])) == str(pop_keys)
    prs = pl.getTraj().getPrimitives()
    assert len(prs) == rr["n_seg"]
    for i, pr in enumerate(prs):
        assert np.array_equal(pr.coeffs, coeffs[i, :dim]), i


def test_bench_workload_sample():
    """96 queries of bench.py's workload (levine-256, |U| = 27): the GPU batch against the reference's sources."""
    m = maps.levine256()
    U = maps.make_U(1.0, 1, 3)
    params = dict(v_max=2.0, a_max=1.0, dt=1.0, tol_pos=0.5)
    rp = _ref_planner(m, 3, params, U)
    S, G = maps.sample_queries(m, 96, seed=0)
    sg, sr = _wps(S, mp.ACC)
    gg, gr = _wps(G, mp.ACC)
    rr = R.value("plan_batch", lambda: rp.plan_batch(sr, gr, nthreads=16))
    pl = _gpu_planner(m, 3, params, U)
    rg, _, _ = pl.plan_batch(sg, gg, max_seg=64)
    for i in range(96):
        _same(rg[i], rr[i], i)


def test_cost_shaping_flow():
    """test_distance_map_planner_2d.cpp flow: GPU vs the reference's setSearchRegion / updatePotentialMap / plan."""
    m, dim, params, U, start, goal = load_config("corridor")
    params = dict(params, potential_weight=0.5, gradient_weight=0.3)
    ncell = int(np.prod(m.dim))
    sg, sr = _wps(start, mp.ACC)
    gg, gr = _wps(goal, mp.ACC)
    # the reference's side: first plan, then the tunnel along its waypoints, the potential map and the shaped plan
    rp = _ref_planner(m, dim, params, U)
    r0 = R.value("plain", lambda: rp.plan(sr, gr))
    co = R.value("plain/coeffs", lambda: rp.traj_coeffs(r0["n_seg"]))
    path = np.zeros((len(co) + 1, 3))
    path[:-1, :2] = co[:, :2, 5]
    t = params["dt"]
    path[-1, :2] = co[-1, :2, 5] + co[-1, :2, 4] * t + 0.5 * co[-1, :2, 3] * t * t  # exact here: dyadic values
    rp.set_vec("search_radius", [0.5, 0.5, 0.0])
    rp.set_search_region(path, dense=False)
    region = R.value("region", lambda: R.digest(rp.get_search_region(ncell)))
    rp.set_vec("potential_radius", [1.0, 1.0, 0.0])
    rp.update_potential_map(np.array([start[0], start[1], 0.0]))
    potmap = R.value("potential_map", lambda: R.digest(rp._keep.get_data()))
    rr = R.value("shaped", lambda: rp.plan(sr, gr))
    pop_keys = R.value("shaped/pop_keys", lambda: R.digest(rp.pop_keys(rr["pops"])))

    pl = _gpu_planner(m, dim, params, U)
    pl.setPotentialWeight(0.5)
    pl.setGradientWeight(0.3)
    assert pl.plan(sg, gg)
    _same(pl.result(), r0, "plain")
    assert np.array_equal(np.array([w.pos for w in pl.getTraj().getWaypoints()]), path[:, :2])
    pl.setSearchRadius([0.5, 0.5])
    pl.setSearchRegion(list(path[:, :2]))
    assert str(R.digest(pl.getSearchRegionMask())) == str(region)
    pl.setPotentialRadius([1.0, 1.0])
    pl.updatePotentialMap(start)
    assert str(R.digest(pl._keep.getMap())) == str(potmap)
    pl.plan(sg, gg)
    _same(pl.result(), rr, "shaped")
    gn = pl.getNodes()
    assert str(R.digest(gn["key"][pl.getPopLog()])) == str(pop_keys)
