"""tests/cpp/test_replanner_fleet_device.cpp: two replanners (dt 1.0 and 0.5) through the device members of
include/mpl_b200/map_planner.hpp (planLPABatchDevice, serializeLPABatch, trajectoryWaypointsBatch, refineLPABatch) print the same
records, retained trajectories, messages, next starts and refined coefficients as two driven by planLPABatch and the host members."""
import os
import re
import subprocess

import pytest

from test_cpp_shim import _write_corridor

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAME = "test_replanner_fleet_device"


def _build(tmp_path):
    """the driver allocates its device buffers itself: compiled against the CUDA runtime next to nvcc"""
    from mpl_ros_b200.build import build_lib
    so = build_lib()
    cuda = os.path.dirname(os.path.dirname(os.path.realpath(os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc"))))
    exe = str(tmp_path / NAME)
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-Wall", "-I", os.path.join(ROOT, "include"), "-I", os.path.join(cuda, "include"),
                           os.path.join(ROOT, "tests", "cpp", NAME + ".cpp"), "-o", exe, so, "-L", os.path.join(cuda, "lib64"), "-lcudart",
                           "-Wl,-rpath," + os.path.dirname(so), "-Wl,-rpath," + os.path.join(cuda, "lib64")])
    return exe


def test_cpp_fleet_device_program_compiles_and_links(tmp_path):
    assert os.path.exists(_build(tmp_path))


@pytest.mark.gpu
def test_cpp_device_members_equal_host_members(tmp_path):
    exe = _build(tmp_path)
    r = subprocess.run([exe, _write_corridor(tmp_path)], stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
    out = r.stdout.decode()
    assert r.returncode == 0, out
    for tag in ("first", "subtree"):
        assert "%s: device call 1 rows 1" % tag in out, out
        rows = re.findall(r"^%s mode (\d) planner (\d): n_seg (\d+) len (\d+) digest (\w+)$" % tag, out, re.M)
        assert len(rows) == 4, out
        for i in "01":
            a = [x[2:] for x in rows if x[0] == "0" and x[1] == i]
            b = [x[2:] for x in rows if x[0] == "1" and x[1] == i]
            assert a == b and int(a[0][0]) > 0 and int(a[0][1]) > 0, (tag, i, out)
    assert len(re.findall(r"^next \d: call 1 ok 1 same 1$", out, re.M)) == 2, out
    ref = re.findall(r"^refine mode (\d): call 1 n_segs (\d+) (\d+) digest (\w+)$", out, re.M)
    assert len(ref) == 2 and ref[0][1:] == ref[1][1:] and int(ref[0][1]) > 0, out
