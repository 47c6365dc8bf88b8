"""Records tests/golden/voxel_grid.npz from the reference's own VoxelGrid (oracle/_ref/libvoxelref.so, built from
planning_ros_utils/src/mapping_utils/voxel_grid.cpp) — run once where the reference tree exists.

Contents:
  <map>_pts (float32 bits of every 16th /cloud point of mpl_test_node/maps/<map>/<map>.bag), <map>_origin / _dim / _res (the
  bag's /voxel_map geometry, as map_replanner_node.cpp:326-331 turns it into VoxelGrid(origin, dim * res, res)), and the
  reference's outputs on them:
    <map>_map             packed bits of getMap() after addCloud(pts)
    <map>_cloud_n / _sha  getCloud() count and SHA-256 of its float64 bytes
    <map>_obs_n / _sha    addCloud(pts, 5x5x1 ns) on a fresh grid: new_obs count and SHA-256 (int32 rows)
    <map>_inf             packed bits of getInflatedMap() after that
    <map>_obs2_n / _sha   decay(), then addCloud(every 2nd point, 3x3x3 ns)
    <map>_local_n / _sha  getLocalCloud over a box around the map's centre
  seq_<seed>             SHA-256 of every observation of tests/voxel_cases.py's sequence(seed), in order
  replanner_*            the map_replanner_node scripts (launch/map_replanner_node/*.sh, float32 points) and test.launch
                         parameters, as data
  flow_*                 the node's flow (tests/voxel_flow.py) on the reference's own VoxelGrid, MapUtil (rayTrace, isFree,
                         isOccupied, setMap) and LPA* sources: a digest row per step (lpa_flow.digest), the new_obs / new_clear
                         cells of each edit and the map bits after it; the update counts are the oracle's (the reference's
                         updateBlockedNodes result is not exported by the harness)
"""
import os
import struct
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))
from extract_fixtures import REF, _parse_header, _records, read_bag_voxelmap  # noqa: E402

import lpa_flow  # noqa: E402
import oracle  # noqa: E402
import voxel_cases as vc  # noqa: E402
import voxel_flow  # noqa: E402
from oracle import ref  # noqa: E402
from oracle import voxel as ov  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "voxel_grid.npz")
SCRIPTS = {  # launch/map_replanner_node/<name>.sh: the two geometry_msgs/Point32 of each message
    "add_cloud": [(12.55, 9.55, 0.025), (12.55, 11.05, 0.025)],
    "add_cloud2": [(4, 5, 0.025), (12, 5, 0.025)],
    "add_cloud3": [(13, 14, 0.025), (13, 18, 0.025)],
    "add_cloud4": [(12.75, 9.55, 0.025), (12.75, 12.0, 0.025)],
    "clear_cloud": [(12.75, 9.55, 0.025), (12.65, 11.95, 0.025)],
    "clear_cloud2": [(4, 5, 0.025), (12, 5, 0.025)],
}


def read_bag_cloud(path, topic="/cloud"):
    """the last sensor_msgs/PointCloud on `topic` (points as float32 rows; the bags carry no channels)"""
    raw = open(path, "rb").read()
    conns, last = {}, None

    def handle(hdr, data):
        nonlocal last
        op = hdr["op"][0]
        if op == 0x07:
            conns[struct.unpack("<I", hdr["conn"])[0]] = (hdr["topic"].decode(), _parse_header(data))
        elif op == 0x02:
            c = struct.unpack("<I", hdr["conn"])[0]
            if conns.get(c, ("",))[0] == topic:
                last = data

    for hdr, data in _records(raw, 13):
        if hdr["op"][0] == 0x05:
            for h2, d2 in _records(data):
                handle(h2, d2)
        else:
            handle(hdr, data)
    assert last is not None, (path, topic)
    _, _, _, flen = struct.unpack_from("<IIII", last, 0)
    off = 16 + flen
    (n,) = struct.unpack_from("<I", last, off)
    pts = np.frombuffer(last, dtype="<f4", count=3 * n, offset=off + 4).reshape(n, 3).copy()
    (nch,) = struct.unpack_from("<I", last, off + 4 + 12 * n)
    assert nch == 0
    return pts


def main():
    assert ov.ref_available(), "the reference harness is not built"
    out = {}
    for name in ("simple", "levine", "skir"):
        base = os.path.join(REF, "mpl_test_node/maps/%s/%s.bag" % (name, name))
        pts32 = read_bag_cloud(base)[::16].copy()
        vm = read_bag_voxelmap(base)
        res = float(vm["res"])
        origin, dim_m = vm["origin"], vm["dim"].astype(np.float64) * res
        z = {name + "_pts": pts32, name + "_origin": origin, name + "_dim": dim_m, name + "_res": np.float32(res)}
        r = vc.fixture_members(ov.RefVoxelGrid, z, name)
        out.update(z)
        out.update({name + "_map": np.packbits(r["map"] == 100), name + "_inf": np.packbits(r["inf"] == 100)})
        for key in ("cloud", "obs", "obs2", "local"):
            out[name + "_%s_n" % key] = len(r[key])
            out[name + "_%s_sha" % key] = vc.digest(r[key])
        print(name, len(pts32), {k: len(r[k]) for k in ("cloud", "obs", "obs2", "local")})
    for seed in range(4):
        o = vc.replay(ov.RefVoxelGrid(vc.ORIGIN, vc.DIM, vc.RES), vc.sequence(seed), seed)
        out["seq_%d" % seed] = np.array([vc.digest(np.asarray(x)) for x in o])
    for k, v in SCRIPTS.items():
        out["replanner_" + k] = np.array(v, dtype=np.float32)
    out["replanner_start"] = np.array([14.5, 2.4, 0.025, 0.0, 1.0, 0.0, 0.0, 0.0, 0.0])  # test.launch: pos, vel, acc
    out["replanner_goal"] = np.array([4.0, 16.0, 0.025])
    out["replanner_limits"] = np.array([2.0, 1.0, 1.0])  # v_max, a_max, dt
    # the replanner node's flow on the reference's own VoxelGrid, MapUtil and LPA* sources (tests/voxel_flow.py); the oracle's
    # restatement is asserted identical while recording
    snaps, edits = voxel_flow.host_flow(out, ov.RefVoxelGrid, ref.RefMap, ref.RefPlanner, ov.RefMapUtil)
    snaps_o, edits_o = voxel_flow.host_flow(out, ov.OracleVoxelGrid, oracle.OracleMap, oracle.OraclePlanner)
    lpa_flow.assert_same(snaps_o, snaps, "replanner")
    out["flow_digest"] = lpa_flow.digest(snaps)
    # the reference harness's update hooks return nothing; the counts are the oracle's, whose state after every update
    # equals the reference's (assert_same above)
    out["flow_updated"] = np.array([e["updated"] for e in edits_o])
    for k, (e, eo) in enumerate(zip(edits, edits_o)):
        assert np.array_equal(e["cells"], eo["cells"]) and np.array_equal(e["map"], eo["map"])
        out["flow_cells_%d" % k], out["flow_map_%d" % k] = e["cells"], e["map"]
    print("flow", [(int(r["status"]), float(r["cost"]), int(r["pops"])) for r in out["flow_digest"]], "edits",
          [(len(e["cells"]), e["updated"]) for e in edits_o])
    np.savez_compressed(OUT, **out)
    print(OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
