"""tests/cpp/test_replanner_fleet.cpp: two replanners through the fleet members of include/mpl_b200/map_planner.hpp
(planLPABatch, getLinkedNodesBatch, updateBlockedNodesBatch / updateClearedNodesBatch, getSubStateSpaceBatch, MapUtil::traceCells)
and two through the single members print the same digests after every step."""
import re
import subprocess

import pytest

from test_cpp_shim import _build, _write_corridor


def test_cpp_fleet_program_compiles_and_links(tmp_path):
    _build(tmp_path, "test_replanner_fleet")


@pytest.mark.gpu
def test_cpp_fleet_members_equal_single_members(tmp_path):
    exe = _build(tmp_path, "test_replanner_fleet")
    r = subprocess.run([exe, _write_corridor(tmp_path)], stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
    out = r.stdout.decode()
    assert r.returncode == 0, out
    rows = re.findall(r"^(\w+) mode (\d): (.*)$", out, re.M)
    assert [t for t, m, _ in rows if m == "0"] == ["first", "blocked", "cleared", "subtree"], out
    for tag in ("first", "blocked", "cleared", "subtree"):
        a = [d for t, m, d in rows if t == tag and m == "0"]
        b = [d for t, m, d in rows if t == tag and m == "1"]
        assert a == b, (tag, out)
    assert "first: ok batched 1 1" in out and "waypoints 0 " not in out.split("blocked")[0], out
    linked = re.findall(r"^linked \d: (\d+) (\d+)$", out, re.M)
    assert len(linked) == 2 and all(x == y and int(x) > 0 for x, y in linked), out
    assert all(int(x) > 0 for x in re.search(r"^blocked (\d+) (\d+)$", out, re.M).groups()), out
