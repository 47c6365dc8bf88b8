"""VoxelGrid on the GPU (mplb_voxel.cu) through mpl_ros_b200.VoxelGrid and the C ABI, against the oracle
(oracle/voxel_oracle.cpp) with tolerance 0 — grids, ordered new_obs lists, ordered clouds, allocate's changed flag — and
against the fixture recorded from the reference's own voxel_grid.cpp (tests/golden/voxel_grid.npz).  Then the map it hands
over: write_map on the device against a map built from getMap's host bytes, for single and batch plans, and the
replanner node's flow (map_replanner_node.cpp:175-241,326-331) run through the new calls plus LPA*."""
import os

import numpy as np
import pytest

import mpl_ros_b200 as mp
import oracle
import voxel_cases as vc
from oracle import voxel as ov

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "voxel_grid.npz")
MAPS = ("simple", "levine", "skir")


class Dev:
    """mpl_ros_b200.VoxelGrid under the oracle's method names (tests/voxel_cases.py)"""

    def __init__(self, origin, dim, res, chunk=0):
        self.g = mp.VoxelGrid(origin, dim, res)
        self.g.setChunkPoints(chunk)

    def info(self):
        return self.g.info()

    def allocate(self, dim, origin):
        return int(self.g.allocate(dim, origin))

    def clear(self):
        self.g.clear()

    def add_cloud(self, pts):
        self.g.addCloud(pts)

    def add_cloud_inflated(self, pts, ns):
        return self.g.addCloud(pts, ns)

    def decay(self):
        self.g.decay()

    def fill(self, cells, column):
        (self.g.fillColumns if column else self.g.fillCells)(cells)

    def clear_columns(self, cells):
        self.g.clearColumns(cells)

    def get_cloud(self):
        return self.g.getCloud()

    def get_local_cloud(self, pos, ori, dim):
        return self.g.getLocalCloud(pos, ori, dim)

    def get_map(self, inflated=False):
        return self.g.getMapData(inflated)


def chunked(n):
    return lambda *a: Dev(*a, chunk=n)


def assert_obs_equal(a, b):
    assert len(a) == len(b)
    for i, (x, y) in enumerate(zip(a, b)):
        assert np.array_equal(np.asarray(x), np.asarray(y)), i


@pytest.mark.parametrize("seed", range(6))
@pytest.mark.parametrize("chunk", [0, 7])
def test_sequences_equal_oracle(seed, chunk):
    """every member, including the cases the reference leaves undefined (as include/mplb.h defines them); chunk = 7 runs the
    inflated insertion in many passes, with duplicate cells straddling pass boundaries"""
    ops = vc.sequence(seed, defined_only=False)
    if chunk:
        assert vc.straddles(ops, chunk)
    a = vc.replay(ov.OracleVoxelGrid(vc.ORIGIN, vc.DIM, vc.RES), ops, seed)
    b = vc.replay(Dev(vc.ORIGIN, vc.DIM, vc.RES, chunk), ops, seed)
    assert_obs_equal(a, b)
    assert any(len(x) for x in a if getattr(x, "ndim", 0) == 2 and x.dtype == np.int32)


@pytest.mark.parametrize("seed", range(4))
def test_sequences_equal_fixture(seed):
    o = vc.replay(Dev(vc.ORIGIN, vc.DIM, vc.RES), vc.sequence(seed), seed)
    assert [vc.digest(np.asarray(x)) for x in o] == list(np.load(GOLD)["seq_%d" % seed])


@pytest.mark.parametrize("name", MAPS)
@pytest.mark.parametrize("chunk", [0, 4093])
def test_fixture_clouds(name, chunk):
    z = np.load(GOLD)
    out = vc.fixture_members(chunked(chunk), z, name)
    vc.check_fixture_members(out, z, name)


def test_device_inputs_fp32_fp64_and_determinism():
    import torch
    z = np.load(GOLD)
    name = "levine"
    args = (z[name + "_origin"], z[name + "_dim"], float(z[name + "_res"]))
    pts32 = z[name + "_pts"]
    ref = ov.OracleVoxelGrid(*args)
    want_obs = ref.add_cloud_inflated(pts32.astype(np.float64), vc.NS_NODE)
    ref.add_cloud(pts32.astype(np.float64)[::3] + 0.05)
    want = (ref.get_map(False), ref.get_map(True), ref.get_cloud())
    runs = []
    for dtype in (torch.float32, torch.float64, torch.float64):
        g = mp.VoxelGrid(*args)
        t = torch.from_numpy(pts32).to(device="cuda", dtype=dtype)
        obs = g.addCloudDevice(t, ns=vc.NS_NODE)
        assert obs.is_cuda and obs.dtype == torch.int32
        g.addCloudDevice(torch.from_numpy(pts32.astype(np.float64)[::3] + 0.05).cuda())
        got = (obs.cpu().numpy(), g.getMapData(False), g.getMapData(True), g.getCloud())
        assert np.array_equal(got[0], want_obs)
        for x, y in zip(got[1:], want):
            assert np.array_equal(x, y)
        runs.append(got)
    for x, y in zip(runs[1], runs[2]):  # two runs of the same inputs: bitwise identical
        assert x.tobytes() == y.tobytes()
    # raw pointer and a caller-provided output buffer, in several passes
    g = mp.VoxelGrid(*args)
    g.setChunkPoints(1000)
    t = torch.from_numpy(pts32).cuda()
    out = torch.full((len(want_obs) + 5, 3), -7, dtype=torch.int32, device="cuda")
    k = g.addCloudDevice((t.data_ptr(), 1), n=len(pts32), ns=vc.NS_NODE, out=out)
    assert k == len(want_obs) and np.array_equal(out[:k].cpu().numpy(), want_obs)
    assert (out[k:] == -7).all()
    small = torch.zeros((10, 3), dtype=torch.int32, device="cuda")  # cap below the count: the count, first rows only
    g2 = mp.VoxelGrid(*args)
    assert g2.addCloudDevice(t, ns=vc.NS_NODE, out=small) == len(want_obs)
    assert np.array_equal(small.cpu().numpy(), want_obs[:10])


def test_large_cloud_many_passes():
    """a tiled, jittered 400 k point cloud in the default pass size and in passes of 1000 points"""
    z = np.load(GOLD)
    args = (z["skir_origin"], z["skir_dim"], float(z["skir_res"]))
    rs = np.random.RandomState(3)
    base = z["skir_pts"].astype(np.float64)
    pts = np.concatenate([base + rs.normal(0, 0.05, base.shape) for _ in range(22)])
    a = ov.OracleVoxelGrid(*args)
    want = a.add_cloud_inflated(pts, vc.NS_CUBE)
    for chunk in (0, 1000):
        d = Dev(*args, chunk=chunk)
        assert np.array_equal(d.add_cloud_inflated(pts, vc.NS_CUBE), want)
        assert np.array_equal(d.get_map(True), a.get_map(True)) and np.array_equal(d.get_map(False), a.get_map(False))


def _planner(mu, U, lpa=False):
    pl = mp.VoxelMapPlanner(False)
    pl.setMapUtil(mu)
    pl.setVmax(2.0); pl.setAmax(1.0); pl.setJmax(1.0); pl.setDt(1.0); pl.setU(U); pl.setTol(0.5, 1)  # tol_acc unset: the library takes it only above ACC control
    if lpa:
        pl.setLPAstar(True)
    return pl


def _waypoints(z, module):
    s = mp.waypoints_array(1) if module is mp else oracle.make_waypoints(1)
    g = mp.waypoints_array(1) if module is mp else oracle.make_waypoints(1)
    st = z["replanner_start"]
    s["pos"][0], s["vel"][0], s["acc"][0] = st[0:3], st[3:6], st[6:9]
    g["pos"][0] = z["replanner_goal"]
    s["control"] = g["control"] = mp.ACC
    return s, g


FIELDS = ("status", "n_seg", "cost", "pops", "n_nodes", "n_open", "n_closed", "n_prims", "n_samples", "n_valid", "pop_hash",
          "closed_hash")


def test_write_map_then_plan():
    z = np.load(GOLD)
    args = (z["simple_origin"], z["simple_dim"], float(z["simple_res"]))
    g = mp.VoxelGrid(*args)
    g.addCloud(z["simple_pts"].astype(np.float64))
    dim, _, ori_d, res = g.info()
    host = g.getMapData()
    mu_dev = mp.VoxelMapUtil()
    mu_dev.setMap(ori_d, dim, np.zeros(host.size, dtype=np.int8), float(res))
    g.writeMap(mu_dev)
    assert np.array_equal(mu_dev.getMap(), host)
    mu_host = mp.VoxelMapUtil()
    mu_host.setMap(ori_d, dim, host, float(res))
    mu_new = g.toMapUtil()
    assert np.array_equal(mu_new.getMap(), host) and np.array_equal(mu_new.getOrigin(), ori_d) and mu_new.getRes() == float(res)
    U = mp.maps.make_U(1.0, 1, 3, use_3d=False)
    s, gl = _waypoints(z, mp)
    recs = []
    for mu in (mu_dev, mu_host, mu_new):
        pl = _planner(mu, U)
        pl.plan(s, gl)
        r = pl.result()
        recs.append((tuple(r[f] for f in FIELDS), pl.getActions().copy()))
        # a batch on the same map
        n = 6
        rs = np.random.RandomState(5)
        S, G = mp.waypoints_array(n), mp.waypoints_array(n)
        S["pos"][:] = s["pos"][0] + rs.uniform(-1, 1, (n, 3)) * (1, 1, 0)
        G["pos"][:] = gl["pos"][0]
        S["control"] = G["control"] = mp.ACC
        res_b, act, _ = pl.plan_batch(S, G, max_seg=64)
        recs.append((tuple(tuple(r[f] for f in FIELDS) for r in res_b), act.copy()))
    assert recs[0][0] == recs[2][0] == recs[4][0] and np.array_equal(recs[0][1], recs[2][1])
    assert recs[1][0] == recs[3][0] == recs[5][0] and np.array_equal(recs[1][1], recs[3][1])
    # and the oracle on getMap's bytes
    om = oracle.OracleMap(ori_d, dim, host, float(res))
    op = oracle.OraclePlanner(3)
    op.set_map(om)
    for k, v in dict(v_max=2.0, a_max=1.0, j_max=1.0, dt=1.0, tol_pos=0.5, tol_vel=1.0, tol_acc=-1).items():
        op.set_param(k, v)
    op.set_controls(U)
    so, go = _waypoints(z, oracle)
    ro = op.plan(so, go)
    assert recs[0][0] == tuple(ro[f] for f in FIELDS)


def test_write_map_rejects_other_geometry():
    g = mp.VoxelGrid((0.0, 0.0, 0.0), (2.0, 2.0, 1.0), 0.1)
    dim, _, ori_d, res = g.info()
    for d, o, r in ((dim + (1, 0, 0), ori_d, float(res)), (dim, ori_d + 0.01, float(res)), (dim, ori_d, 0.1)):
        mu = mp.VoxelMapUtil()
        mu.setMap(o, d, np.zeros(int(np.prod(d)), dtype=np.int8), r)
        with pytest.raises(mp.MplbError, match="error -1"):
            g.writeMap(mu)
    mu2 = mp.OccMapUtil()
    mu2.setMap(ori_d[:2], dim[:2], np.zeros(int(dim[0] * dim[1]), dtype=np.int8), float(res))
    with pytest.raises(mp.MplbError, match="error -1"):
        g.writeMap(mu2)


def test_map_get_cells():
    z = np.load(GOLD)
    g = mp.VoxelGrid(z["skir_origin"], z["skir_dim"], float(z["skir_res"]))
    g.addCloud(z["skir_pts"].astype(np.float64))
    mu = g.toMapUtil()
    dim = mu.getDim()
    rs = np.random.RandomState(1)
    cells = np.stack([rs.randint(-3, d + 3, 500) for d in dim], axis=1)
    got = mu.getCells(cells)
    data = mu.getMap()
    inside = np.all((cells >= 0) & (cells < dim), axis=1)
    lin = cells[:, 0] + dim[0] * cells[:, 1] + dim[0] * dim[1] * cells[:, 2]
    assert np.array_equal(got[inside], data[lin[inside]].astype(np.int32))
    assert np.all(got[~inside] == np.iinfo(np.int32).min) and (~inside).any() and (got[inside] == 100).any()


def test_replanner_node_flow():
    """map_replanner_node.cpp's start-up, add_cloud.sh, clear_cloud.sh and subtree steps through the VoxelGrid calls (addCloud,
    create_map, fill / clear columns, write_map), MapUtil.getCells for isFree / isOccupied and LPA*; step by step equal to the
    oracle and to the run recorded from the reference's own VoxelGrid, MapUtil and LPA* sources"""
    import lpa_flow
    import voxel_flow
    from test_gpu_lpa import GpuPlanner
    z = np.load(GOLD)
    d = Dev(*voxel_flow.geometry(z))
    d.add_cloud(z["simple_pts"].astype(np.float64))
    dim, _, ori_d, res = d.info()

    class Map:
        mu = d.g.toMapUtil()

    Map.mu.freeUnknown()
    pl = GpuPlanner(3)
    pl.set_map(Map)
    voxel_flow.configure(pl)
    edit = voxel_flow.oracle_cells_edit(d, Map.mu.getCells, lambda: d.g.writeMap(Map.mu), ori_d, dim, float(res))
    snaps, edits = voxel_flow.run(z, d, pl, edit)
    voxel_flow.check(snaps, edits, z)
    a, ea = voxel_flow.host_flow(z, ov.OracleVoxelGrid, oracle.OracleMap, oracle.OraclePlanner)
    lpa_flow.assert_same(a, snaps, "replanner")
    assert edits[0]["updated"] > 0 and len(edits[1]["cells"]) > 0
    assert snaps[2]["res"]["pops"] != snaps[0]["res"]["pops"]


def test_cpp_cloud_to_map_and_replanner_edits(tmp_path):
    """tests/cpp/test_voxel_grid.cpp (cloud_to_map's processCloud and the replanner node's edits through the C++ header)
    against the fixture recorded from the reference"""
    import subprocess
    import struct
    from test_voxel_cpp import build

    def fnv(b):
        h = 1469598103934665603
        for x in bytes(b):
            h = ((h ^ x) * 1099511628211) & 0xFFFFFFFFFFFFFFFF
        return h

    def grid_bytes(bits, n):
        return np.where(np.unpackbits(bits)[:n].astype(bool), 100, 0).astype(np.int8).tobytes()

    z = np.load(GOLD)
    pts = z["simple_pts"]
    p = str(tmp_path / "simple.bin")
    with open(p, "wb") as f:
        f.write(struct.pack("<3d", *z["simple_origin"].tolist()) + struct.pack("<3d", *z["simple_dim"].tolist()))
        f.write(struct.pack("<f", float(z["simple_res"])) + struct.pack("<q", len(pts)))
        f.write(np.ascontiguousarray(pts, dtype=np.float32).tobytes())
        f.write(np.concatenate([z["replanner_add_cloud"][[0, -1]], z["replanner_clear_cloud"][[0, -1]]]).astype(np.float32).tobytes())
    out = subprocess.check_output([build(tmp_path), p]).decode()
    og = ov.OracleVoxelGrid(z["simple_origin"], z["simple_dim"], float(z["simple_res"]))
    dim = og.info()[0]
    n = int(np.prod(dim))
    obs = og.add_cloud_inflated(pts.astype(np.float64), vc.NS_NODE)
    assert len(obs) == int(z["simple_obs_n"]) and vc.digest(obs) == str(z["simple_obs_sha"])
    occ = int(np.unpackbits(z["simple_map"])[:n].sum())
    lines = ["cloud_to_map: dim %d %d %d occupied %d hash %d cloud %d" % (*dim, occ, fnv(grid_bytes(z["simple_map"], n)),
                                                                          int(z["simple_cloud_n"])),
             "inflated: new_obs %d hash %d" % (len(obs), fnv(obs.tobytes())),
             "add_cloud: new_obs %d hash %d map %d" % (len(z["flow_cells_0"]), fnv(z["flow_cells_0"].astype(np.int32).tobytes()),
                                                       fnv(grid_bytes(z["flow_map_0"], n))),
             "clear_cloud: new_clear %d hash %d map %d" % (len(z["flow_cells_1"]), fnv(z["flow_cells_1"].astype(np.int32).tobytes()),
                                                          fnv(grid_bytes(z["flow_map_1"], n)))]
    for line in lines:
        assert line in out, (line, out)
