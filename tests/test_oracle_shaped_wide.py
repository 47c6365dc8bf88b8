"""The oracle against the reference's own planner sources (oracle/_ref/libmplref.so, see test_oracle_vs_reference.py) on
the cost-shaping and yaw configurations with more than 32 control rows, which the |U| > 32 cost-shaping kernels
(astar_batch_kernel<DIM, ORD, 4, true>) plan on the GPU:
  - map_planner_node's 3D + yaw set (81 rows, ACCxYAW), and test_planner_2d_with_yaw's flow with num = 2 (75 rows);
    the oracle in trig_mode 0 calls the same libm as the reference code does;
  - distance_map_planner_node's flow with num = 3 (49 rows): plain plan, search region around it, potential map, shaped
    plan, then iterativePlan.
Everything is compared exactly: counters, the pop sequence, every node, the region mask and the rewritten map.  These
comparisons need the library, so the module is skipped where it was not built."""
import math

import numpy as np
import pytest

import oracle
from oracle import ref
from mpl_ros_b200 import maps
from helpers import load_config
from test_oracle_vs_reference import EXACT_FIELDS, _node_table, _same_status, _wp

pytestmark = pytest.mark.skipif(not ref.available(), reason="oracle/_ref/libmplref.so is built only where the reference tree exists")


def node_U_yaw(u, num, u_yaw, dim):
    """map_planner_node.cpp:120-139: the node's (dx, dy[, dz]) loop, then dyaw in {-u_yaw, 0, u_yaw} innermost"""
    yaws, d = [], -u_yaw
    while d <= u_yaw:
        yaws.append(d)
        d += u_yaw
    return np.array([list(r) + [y] for r in maps.make_U(u, num, dim) for y in yaws])


def _pair(m, dim, params, U, trig_mode=None):
    om, rm = oracle.OracleMap(m.origin, m.dim, m.data, m.res), ref.RefMap(m.origin, m.dim, m.data, m.res)
    om.free_unknown()
    rm.free_unknown()
    op, rp = oracle.OraclePlanner(dim), ref.RefPlanner(dim)
    op.set_map(om)
    rp.set_map(rm)
    for k, v in params.items():
        op.set_param(k, v)
        rp.set_param(k, v)
    if trig_mode is not None:
        op.set_param("trig_mode", trig_mode)
    op.set_controls(U)
    rp.set_controls(U)
    op._keep, rp._keep = om, rm
    return op, rp


def _compare(op, rp, s, g, ctx):
    ro, rr = op.plan(s, g), rp.plan(s, g)
    assert _same_status(int(ro["status"]), int(rr["status"])), (ctx, ro["status"], rr["status"])
    for f in EXACT_FIELDS:
        if f == "n_seg" and ro["status"] != 0:
            continue
        assert ro[f] == rr[f] or (f == "cost" and np.isinf(ro[f]) and np.isinf(rr[f])), (ctx, f, ro[f], rr[f])
    assert np.array_equal(op.pop_keys(ro["pops"]), rp.pop_keys(rr["pops"])), ctx
    assert np.array_equal(_node_table(op.nodes(ro["n_nodes"])), _node_table(rp.nodes(rr["n_nodes"]))), ctx
    return ro


@pytest.mark.parametrize("yaw_max,wyaw", [(0.7, 1.0), (-1.0, 1.0), (1.2, 0.0)])
def test_node_3d_yaw_81_rows(yaw_max, wyaw):
    m, dim, params, _, start, goal = load_config("skir")
    U = node_U_yaw(1.0, 1, 0.3, 3)
    assert U.shape == (81, 4)
    op, rp = _pair(m, dim, dict(params, yaw_max=yaw_max, wyaw=wyaw), U, trig_mode=0)
    ro = _compare(op, rp, _wp(start, 19, yaw=0.4), _wp(goal, 19), ("3D yaw", yaw_max, wyaw))
    assert ro["status"] == 0


@pytest.mark.parametrize("yaw_max,wyaw", [(0.7, 1.0), (-1.0, 1.0), (0.7, 0.0), (1.2, 2.5)])
def test_planner_2d_with_yaw_75_rows(yaw_max, wyaw):
    m, dim, params, _, start, goal = load_config("corridor")
    U = node_U_yaw(0.5, 2, 0.5, 2)
    assert U.shape == (75, 3)
    op, rp = _pair(m, dim, dict(params, yaw_max=yaw_max, wyaw=wyaw), U, trig_mode=0)
    ro = _compare(op, rp, _wp(start, 19, yaw=math.pi / 2), _wp(goal, 19), ("2D yaw", yaw_max, wyaw))
    assert ro["status"] == 0


def _path(op, ro, U, dt):
    st, acts = op.seg_states(ro["n_seg"]), op.actions(ro["n_seg"])
    path = np.zeros((ro["n_seg"] + 1, 3))
    path[:-1, :2] = st[:, :2]
    last = st[-1]
    path[-1, :2] = last[:2] + last[3:5] * dt + 0.5 * U[acts[-1]] * dt * dt
    return path


@pytest.mark.parametrize("grad_w", [0.0, 0.3])
def test_distance_map_flow_wide(grad_w, num=3):
    m, dim, params, _, start, goal = load_config("corridor")
    U = maps.make_U(0.5, num, 2)
    assert len(U) == (2 * num + 1) ** 2
    ncell = int(np.prod(m.dim))
    op, rp = _pair(m, dim, params, U)
    s, g = _wp(start, 3), _wp(goal, 3)
    ro = _compare(op, rp, s, g, "plain")
    assert ro["status"] == 0
    path = _path(op, ro, U, params["dt"])
    op2, rp2 = _pair(m, dim, dict(params, epsilon=1.0, potential_weight=0.5, gradient_weight=grad_w), U)
    op2.set_map(op._keep)
    rp2.set_map(rp._keep)
    for p in (op2, rp2):
        p.set_vec("search_radius", [0.5, 0.5, 0.0])
        p.set_search_region(path, dense=False)
        p.set_vec("potential_radius", [1.0, 1.0, 0.0])
        p.update_potential_map(np.array([start[0], start[1], 0.0]))
    assert np.array_equal(op2.get_search_region(ncell), rp2.get_search_region(ncell))
    assert np.array_equal(op._keep.get_data(ncell), rp._keep.get_data())
    ro2 = _compare(op2, rp2, s, g, "shaped")
    assert ro2["status"] == 0 and ro2["cost"] > ro["cost"]
    rit = rp2.iterative_plan(s, g, rp2, 3)
    prev, pth = 0.0, _path(op2, ro2, U, params["dt"])
    for _ in range(3):
        op2.set_search_region(pth, dense=False)
        roi = op2.plan(s, g)
        assert roi["status"] == 0
        pth = _path(op2, roi, U, params["dt"])
        if prev == roi["cost"]:
            break
        prev = roi["cost"]
    for f in ("status", "cost", "n_seg", "pops", "pop_hash"):
        assert rit[f] == roi[f], (f, rit[f], roi[f])
