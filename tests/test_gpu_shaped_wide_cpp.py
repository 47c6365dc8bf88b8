"""tests/cpp/test_map_planner_node_3d_yaw.cpp: map_planner_node's planning block with use_3d and use_yaw (81 control rows)
through include/mpl_b200/map_planner.hpp, on skir, against the oracle (correctly rounded cos/sin, trig_mode 1)."""
import struct
import subprocess

import numpy as np
import pytest

import oracle
from helpers import load_config
from test_cpp_shim import _build
from test_oracle_shaped_wide import node_U_yaw


def _write_skir(tmp_path):
    m, _, _, _, start, goal = load_config("skir")
    p = str(tmp_path / "skir.bin")
    with open(p, "wb") as f:
        f.write(struct.pack("<3i", *m.dim.tolist()))
        f.write(struct.pack("<3d", *m.origin.tolist()))
        f.write(struct.pack("<d", m.res))
        f.write(struct.pack("<3d", *start.tolist()))
        f.write(struct.pack("<3d", *goal.tolist()))
        f.write(m.data.tobytes())
    return p, m, start, goal


def test_cpp_node_3d_yaw_program_compiles_and_links(tmp_path):
    _build(tmp_path, "test_map_planner_node_3d_yaw")


@pytest.mark.gpu
@pytest.mark.parametrize("yaw_max,wyaw", [(0.7, 1.0), (-1.0, 0.0)])
def test_cpp_node_3d_yaw(tmp_path, yaw_max, wyaw):
    exe = _build(tmp_path, "test_map_planner_node_3d_yaw")
    path, m, start, goal = _write_skir(tmp_path)
    r = subprocess.run([exe, path, repr(yaw_max), repr(wyaw)], stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
    out = r.stdout.decode()
    assert r.returncode == 0, out
    lines = out.split("\n")
    head = [ln.split() for ln in lines if ln.startswith("plan ")]
    assert len(head) == 1, out
    ok, cost, n_seg = int(head[0][1]), float.fromhex(head[0][2]), int(head[0][3])
    wps = np.array([[float.fromhex(x) for x in ln.split()[1:]] for ln in lines if ln.startswith("wp ")])

    om = oracle.OracleMap(m.origin, m.dim, m.data, m.res)
    om.free_unknown()
    op = oracle.OraclePlanner(3)
    op.set_map(om)
    for k, v in dict(v_max=2.0, a_max=1.0, dt=1.0, tol_pos=0.5, yaw_max=yaw_max, wyaw=wyaw).items():
        op.set_param(k, v)
    op.set_param("trig_mode", 1)
    U = node_U_yaw(1.0, 1, 0.3, 3)
    assert len(U) == 81
    op.set_controls(U)
    s, g = oracle.make_waypoints(1), oracle.make_waypoints(1)
    s["pos"][0], g["pos"][0] = start, goal
    s["control"] = g["control"] = 19  # ACCxYAW
    ro = op.plan(s, g)
    assert ok == 1 and ro["status"] == 0, (out, ro["status"])
    assert cost == ro["cost"] and n_seg == ro["n_seg"], (cost, ro["cost"], n_seg, ro["n_seg"])
    st = op.seg_states(n_seg)
    assert len(wps) == n_seg + 1
    assert np.array_equal(wps[:-1, :3], st[:, :3]) and np.array_equal(wps[:-1, 3], st[:, 12])
    assert np.max(np.abs(wps[-1, :3] - goal)) <= 0.5
