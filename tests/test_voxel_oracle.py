"""The VoxelGrid oracle (oracle/voxel_oracle.cpp) against the reference's own voxel_grid.cpp (skipped where that harness
is not built) and against the fixture recorded from it (always).  No GPU."""
import os

import numpy as np
import pytest

import voxel_cases as vc
from oracle import voxel as ov

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "voxel_grid.npz")
MAPS = ("simple", "levine", "skir")


@pytest.fixture(scope="module")
def gold():
    return np.load(GOLD)


@pytest.mark.parametrize("name", MAPS)
def test_oracle_equals_fixture_clouds(gold, name):
    out = vc.fixture_members(ov.OracleVoxelGrid, gold, name)
    vc.check_fixture_members(out, gold, name)
    assert len(out["obs"]) > 0 and len(out["obs2"]) > 0 and len(out["local"]) > 0


@pytest.mark.parametrize("seed", range(4))
def test_oracle_equals_fixture_sequences(gold, seed):
    o = vc.replay(ov.OracleVoxelGrid(vc.ORIGIN, vc.DIM, vc.RES), vc.sequence(seed), seed)
    assert [vc.digest(np.asarray(x)) for x in o] == list(gold["seq_%d" % seed])


needs_ref = pytest.mark.skipif(not ov.ref_available(), reason="the reference's voxel_grid.cpp harness is not built here")


@needs_ref
@pytest.mark.parametrize("seed", range(12))
def test_oracle_equals_reference_sequences(seed):
    ops = vc.sequence(seed)
    a = vc.replay(ov.OracleVoxelGrid(vc.ORIGIN, vc.DIM, vc.RES), ops, seed)
    b = vc.replay(ov.RefVoxelGrid(vc.ORIGIN, vc.DIM, vc.RES), ops, seed)
    assert len(a) == len(b)
    for i, (x, y) in enumerate(zip(a, b)):
        assert np.array_equal(np.asarray(x), np.asarray(y)), i


@needs_ref
@pytest.mark.parametrize("name", MAPS)
def test_oracle_equals_reference_clouds(gold, name):
    a, b = vc.fixture_members(ov.OracleVoxelGrid, gold, name), vc.fixture_members(ov.RefVoxelGrid, gold, name)
    for k in a:
        assert np.array_equal(a[k], b[k]), k


def test_sequences_hit_the_delicate_cases():
    """What the sequences are meant to cover actually happens (checked on the oracle, which equals the reference)."""
    g = ov.OracleVoxelGrid(vc.ORIGIN, vc.DIM, vc.RES)
    dim, ori, ori_d, res = g.info()
    assert list(ori) == [-19, -10, 0] and list(dim) == [31, 24, 8] and res == np.float32(0.1)
    r = float(res)
    # truncation band: a point up to one cell below the origin lands in cell 0
    g.add_cloud([(ori_d[0] - 0.9 * r, ori_d[1] + 0.5 * r, ori_d[2] + 0.5 * r)])
    m = g.get_map().reshape(8, 24, 31)
    assert m[0, 0, 0] == 100 and m.sum() == 100
    # the z = 0 rule and an unchanged allocate
    h = ov.OracleVoxelGrid((0.0, 0.0, 0.0), (1.0, 1.0, 0.0), 0.1)
    assert h.info()[0][2] == 1 and h.allocate((1.0, 1.0, 0.0), (0.0, 0.0, 0.0)) == 0
    # inflated insertion after decay: a decayed cell dilates again, a cell still at 100 does not
    g.clear()
    p = np.array([(ori_d[0] + 5.5 * r, ori_d[1] + 5.5 * r, ori_d[2] + 3.5 * r)])
    assert len(g.add_cloud_inflated(p, vc.NS_CUBE)) == 27
    assert len(g.add_cloud_inflated(p, vc.NS_CUBE)) == 0
    g.decay()
    assert len(g.add_cloud_inflated(p, vc.NS_CUBE)) == 27
    # duplicates within one call and offsets outside
    g.clear()
    edge = np.array([(ori_d[0] + 0.5 * r, ori_d[1] + 0.5 * r, ori_d[2] + 0.5 * r)] * 3)
    assert len(g.add_cloud_inflated(edge, vc.NS_CUBE)) == 8
    seqs = [vc.sequence(s) for s in range(4)]
    assert all(any(n == "allocate" for n, _ in s) for s in seqs)


def test_replanner_flow_oracle_equals_fixture(gold):
    """the replanner node's flow (tests/voxel_flow.py) with the oracle's grid, rayTrace, map and LPA*, step by step against
    the run recorded from the reference's own sources"""
    import oracle
    import voxel_flow
    snaps, edits = voxel_flow.host_flow(gold, ov.OracleVoxelGrid, oracle.OracleMap, oracle.OraclePlanner)
    voxel_flow.check(snaps, edits, gold)
    assert edits[0]["updated"] > 0 and len(edits[1]["cells"]) > 0
    assert snaps[2]["res"]["pops"] != snaps[0]["res"]["pops"]  # the replan after add_cloud is incremental


@needs_ref
def test_replanner_flow_reference_equals_oracle(gold):
    import lpa_flow
    import oracle
    import voxel_flow
    from oracle import ref
    a, ea = voxel_flow.host_flow(gold, ov.RefVoxelGrid, ref.RefMap, ref.RefPlanner, ov.RefMapUtil)
    b, eb = voxel_flow.host_flow(gold, ov.OracleVoxelGrid, oracle.OracleMap, oracle.OraclePlanner)
    lpa_flow.assert_same(b, a, "replanner")
    for x, y in zip(ea, eb):
        assert np.array_equal(x["cells"], y["cells"]) and np.array_equal(x["map"], y["map"])


@needs_ref
def test_ray_trace_equals_reference(gold):
    """the oracle's MapUtil::rayTrace against the reference's, on the script rays and on random rays, a third of them with
    end points on a 0.05 lattice (ties of std::round)"""
    g = ov.RefVoxelGrid(gold["simple_origin"], gold["simple_dim"], float(gold["simple_res"]))
    dim, _, o, r = g.info()
    mu = ov.RefMapUtil(o, dim, float(r), g.get_map())
    rs = np.random.RandomState(0)
    rays = [(gold["replanner_" + k][0], gold["replanner_" + k][-1]) for k in ("add_cloud", "add_cloud2", "add_cloud3", "add_cloud4",
                                                                             "clear_cloud", "clear_cloud2")]
    for i in range(300):
        p1, p2 = o + rs.rand(3) * dim * float(r), o + rs.rand(3) * dim * float(r)
        rays.append((np.round(p1 * 20) / 20, np.round(p2 * 20) / 20) if i % 3 == 0 else (p1, p2))
    for p1, p2 in rays:
        p1, p2 = np.asarray(p1, dtype=np.float64), np.asarray(p2, dtype=np.float64)
        assert np.array_equal(ov.ray_trace(o, dim, float(r), p1, p2), mu.ray_trace(p1, p2))
