"""Seeded VoxelGrid operation sequences and their replay (shared by the oracle, reference-harness and GPU tests and by
tools/make_golden_voxel.py).

A grid here is anything with the oracle's method names (oracle.voxel.OracleVoxelGrid); the GPU tests wrap
mpl_ros_b200.VoxelGrid to the same names.  Every sequence hits the cases the reference's arithmetic makes delicate:
points in the (-1, 0) truncation band below the origin, points exactly on cell boundaries, duplicate points within a call
and across calls, ns offsets reaching outside, inflated insertion after decay (cells at 1..99 dilate again), allocate
with positive, negative, partial-overlap and unchanged shifts (origin -2.0 -> -19 at res float(0.1), the z = 0 rule), and
getLocalCloud boxes that clip each face.  `defined_only=False` adds what the reference leaves undefined (NaN and huge
points, columns outside the grid) for the oracle-vs-GPU comparison only.
"""
import hashlib

import numpy as np

RES = 0.1
ORIGIN = (-2.0, -1.05, 0.1)  # -2.0 / float(0.1) truncates to -19; z origin 0.1 to 0 (levine's case)
DIM = (3.2, 2.5, 0.9)
NS_CUBE = np.array([(x, y, z) for x in (-1, 0, 1) for y in (-1, 0, 1) for z in (-1, 0, 1)], dtype=np.int32)
NS_NODE = np.array([(x, y, 0) for x in range(-2, 3) for y in range(-2, 3)], dtype=np.int32)  # map_replanner_node.cpp:204-206
NS_FAR = np.array([(0, 0, 0), (40, 0, 0), (0, -40, 0), (0, 0, 9), (-1, 2, -1)], dtype=np.int32)
# getLocalCloud (pos, ori, dim) of the fixture maps, around each map's centre
LOCAL_BOX = dict(simple=((10.0, 10.0, 0.0), (-3.0, -3.0, -1.0), (6.0, 6.0, 3.0)),
                 levine=((7.0, 14.0, 1.0), (-4.0, -4.0, -1.0), (8.0, 8.0, 2.0)),
                 skir=((5.0, 5.0, 3.0), (-2.5, -2.5, -2.5), (5.0, 5.0, 5.0)))


def digest(a):
    a = np.ascontiguousarray(a)
    return hashlib.sha256(a.tobytes()).hexdigest()


def points(rs, origin_d, dims, res, n, dup=True):
    """n points over the grid and a margin of two cells around it, a third of them on cell boundaries or in the truncation
    band just below the origin, with duplicates"""
    res = float(np.float32(res))
    o = np.asarray(origin_d, dtype=np.float64)
    ext = np.asarray(dims, dtype=np.float64) * res
    p = o - 2 * res + rs.rand(n, 3) * (ext + 4 * res)
    k = n // 3
    cells = np.stack([rs.randint(-1, int(d) + 2, size=k) for d in dims], axis=1)
    p[:k] = o + cells * res                                        # exactly on boundaries (as computed in double)
    band = rs.rand(k, 3) < 0.5
    p[k:2 * k] = np.where(band, o - rs.rand(k, 3) * res, p[k:2 * k])  # (-1, 0) band below the origin, some axes
    if dup and n >= 8:
        idx = rs.randint(0, n, size=n // 8)
        p[rs.randint(0, n, size=n // 8)] = p[idx]
    return p


def sequence(seed, defined_only=True):
    """list of (op, args) for one seeded run on a grid created as (ORIGIN, DIM, RES)"""
    rs = np.random.RandomState(seed)
    ops = []
    geo = dict(origin=np.array(ORIGIN), dims=(32, 25, 9))
    ops.append(("add_cloud", (points(rs, geo["origin"], geo["dims"], RES, 300),)))
    ops.append(("add_cloud_inflated", (points(rs, geo["origin"], geo["dims"], RES, 200), NS_CUBE)))
    ops.append(("add_cloud_inflated", (points(rs, geo["origin"], geo["dims"], RES, 150), NS_FAR)))
    ops.append(("decay", ()))
    ops.append(("add_cloud_inflated", (points(rs, geo["origin"], geo["dims"], RES, 200), NS_NODE)))
    for _ in range(3):
        ops.append(("decay", ()))
    pts = points(rs, geo["origin"], geo["dims"], RES, 120)
    ops.append(("add_cloud_inflated", (np.concatenate([pts, pts[::-1]]), NS_CUBE)))  # duplicates within and across calls
    ops.append(("add_cloud_inflated", (pts, NS_CUBE)))
    cells = np.stack([rs.randint(-2, 35, 12), rs.randint(-2, 28, 12), rs.randint(-2, 11, 12)], axis=1)
    ops.append(("fill", (cells, True)))
    ops.append(("fill", (cells[::-1] + 1, False)))
    cols = np.stack([rs.randint(0, 31, 6), rs.randint(0, 24, 6), np.zeros(6, dtype=np.int64)], axis=1)  # dim_ is (31, 24, 8)
    if not defined_only:
        cols = np.concatenate([cols, [(-1, 3, 0), (31, 0, 0), (5, 24, 0), (2, -7, 0)]])
    ops.append(("clear_columns", (cols,)))
    if not defined_only:
        bad = np.array([(np.nan, 0.0, 0.5), (0.0, np.inf, 0.5), (1e12, 0.0, 0.5), (-1e12, 0.0, 0.5), (0.1, 0.2, -np.inf)])
        ops.append(("add_cloud_inflated", (bad, NS_CUBE)))
        ops.append(("add_cloud", (bad,)))
    # allocate: unchanged, positive / negative / partial-overlap shifts, the z = 0 rule, a grown grid
    ops.append(("allocate", (np.array(DIM), np.array(ORIGIN))))
    ops.append(("allocate", (np.array(DIM), np.array(ORIGIN) + (0.35, -0.2, 0.1))))
    ops.append(("add_cloud_inflated", (points(rs, np.array(ORIGIN) + (0.35, -0.2, 0.1), (32, 25, 9), RES, 150), NS_CUBE)))
    ops.append(("allocate", (np.array((2.0, 3.3, 0.6)), np.array(ORIGIN) - (0.5, 0.15, 0.0))))
    ops.append(("allocate", (np.array((2.5, 2.0, 0.0)), np.array((-1.2, -0.6, 0.0)))))  # z = 0: one layer
    ops.append(("add_cloud", (points(rs, (-1.2, -0.6, 0.0), (25, 20, 1), RES, 200),)))
    ops.append(("allocate", (np.array((4.0, 3.0, 1.2)), np.array((-2.0, -1.0, -0.3)))))
    ops.append(("add_cloud_inflated", (points(rs, (-2.0, -1.0, -0.3), (40, 30, 12), RES, 250), NS_NODE)))
    return ops


def local_boxes(rs, origin_d, dims, res):
    """(pos, ori, dim) boxes: one clipping each face, one inside, one beyond everything"""
    o = np.asarray(origin_d, dtype=np.float64)
    ext = np.asarray(dims, dtype=np.float64) * float(np.float32(res))
    boxes = []
    for a in range(3):
        lo = o + rs.rand(3) * ext * 0.5
        lo[a] = o[a] - 0.3 * ext[a]                                    # clips the low face of axis a
        boxes.append((lo, np.zeros(3), ext * 0.6))
        hi = o + rs.rand(3) * ext * 0.3
        boxes.append((hi, np.array([0.05, -0.05, 0.0]), ext * 1.2))   # clips the high faces
    boxes.append((o + ext * 0.25, np.array([0.1, 0.1, 0.0]), ext * 0.4))
    boxes.append((o - 10 * ext, np.zeros(3), ext))                    # entirely outside: empty
    return boxes


def replay(g, ops, seed=0):
    """Apply ops to grid g; returns the list of observations in order (numpy arrays / ints)."""
    rs = np.random.RandomState(10_000 + seed)
    obs = []

    def snapshot():
        dim, _, ori_d, res = g.info()
        obs.extend([dim.copy(), ori_d.copy(), np.float32(res), g.get_map(False), g.get_map(True), g.get_cloud()])
        for pos, ori, box in local_boxes(rs, ori_d, dim, res):
            obs.append(g.get_local_cloud(pos, ori, box))

    for name, args in ops:
        r = getattr(g, name)(*args)
        if name in ("allocate", "add_cloud_inflated"):
            obs.append(r)
        snapshot()
    return obs


def fixture_members(G, z, name):
    """The members tests/golden/voxel_grid.npz records for map `name`, computed by grid class G(origin, dim, res):
    getMap after addCloud(pts), getCloud, addCloud(pts, 5x5x1) on a fresh grid, getInflatedMap, decay then
    addCloud(every 2nd point, 3x3x3), getLocalCloud."""
    pts = z[name + "_pts"].astype(np.float64)
    args = (z[name + "_origin"], z[name + "_dim"], float(z[name + "_res"]))
    g = G(*args)
    g.add_cloud(pts)
    h = G(*args)
    obs = h.add_cloud_inflated(pts, NS_NODE)
    inf = h.get_map(True)
    h.decay()
    obs2 = h.add_cloud_inflated(pts[::2], NS_CUBE)
    local = h.get_local_cloud(*[np.array(v) for v in LOCAL_BOX[name]])
    return dict(map=g.get_map(), cloud=g.get_cloud(), obs=obs, inf=inf, obs2=obs2, local=local)


def check_fixture_members(out, z, name):
    assert np.array_equal(np.packbits(out["map"] == 100), z[name + "_map"])
    assert np.array_equal(np.packbits(out["inf"] == 100), z[name + "_inf"])
    for key in ("cloud", "obs", "obs2", "local"):
        a = out[key]
        assert len(a) == int(z[name + "_%s_n" % key]) and digest(a) == str(z[name + "_%s_sha" % key]), key


def straddles(ops, chunk):
    """True when an inflated insertion of ops, on the starting geometry (the ops before the first allocate), has one cell
    hit by points in two different passes of `chunk` points"""
    r = float(np.float32(RES))
    g = np.array(ORIGIN)
    dims = np.array([31, 24, 8])  # dim_ of (ORIGIN, DIM, RES)
    for name, args in ops:
        if name == "allocate":
            return False
        if name != "add_cloud_inflated":
            continue
        with np.errstate(invalid="ignore", over="ignore"):
            q = (np.asarray(args[0], dtype=np.float64) - g) / r
        ok = np.all(np.isfinite(q) & (q > -1) & (q < dims), axis=1)
        cells = {}
        for i in np.flatnonzero(ok):
            cells.setdefault(tuple(q[i].astype(int)), set()).add(i // chunk)
        if any(len(p) > 1 for p in cells.values()):
            return True
    return False
