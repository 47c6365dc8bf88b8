"""MapUtil::rayTrace and the replanner node's cell selection on the GPU (mplb_map_trace_cells / _device, MapUtil.traceCells),
exactly (tolerance 0) against the oracle's restatement of map_util.h:117-134, the reference's own MapUtil where oracle/_ref holds
it, and the cells the node's callbacks recorded from the reference (tests/golden/voxel_grid.npz); then the node's flow with the
whole edit on the device: trace -> VoxelGrid fill / clear -> write_map -> the device-list LPA* update."""
import ctypes as C
import os

import numpy as np
import pytest

import mpl_ros_b200 as mp
from mpl_ros_b200 import _lib
from oracle import voxel as ov

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "voxel_grid.npz")
NS5 = np.array([(x, y, 0) for x in range(-2, 3) for y in range(-2, 3)], dtype=np.int32)  # the node's 5 x 5 stencil


def oracle_trace(origin, dim, res, p1, p2):
    """the oracle's rayTrace; a 2D map is traced as a one-cell-high 3D map at the cell's centre height (no z step, no z cut)"""
    if len(dim) == 2:
        o3, d3 = np.r_[origin, 0.0], np.r_[dim, 1]
        c = ov.ray_trace(o3, d3, res, np.r_[p1[:2], 0.5 * res], np.r_[p2[:2], 0.5 * res])
        return c[:, :2]
    return ov.ray_trace(origin, dim, res, p1[:3], p2[:3])


def rays(rs, origin, dim, res, n):
    """inside, crossing, outside starts, zero-length, shorter than 0.8 res (max_diff 0 and 1), axis-aligned and corner rays"""
    d = len(dim)
    lo, hi = np.asarray(origin, dtype=np.float64), np.asarray(origin) + np.asarray(dim) * res
    span = hi - lo
    out = []

    def pt(margin=0.0):
        return lo - margin * span + rs.rand(d) * span * (1 + 2 * margin)
    for i in range(n):
        kind = i % 8
        if kind == 0:
            a, b = pt(), pt()
        elif kind == 1:
            a, b = pt(), pt(0.6)
        elif kind == 2:
            a, b = pt(0.6), pt()
            k = rs.randint(d)
            a[k] = lo[k] - span.max() * (1 + rs.rand())  # certainly outside
        elif kind == 3:
            a = pt()
            b = a.copy()
        elif kind == 4:
            a = pt()
            b = a + (rs.rand(d) - 0.5) * res * rs.choice([0.5, 1.0, 1.5, 1.9])  # max_diff 0, 1 or 2
        elif kind == 5:
            a = pt()
            b = a.copy()
            b[rs.randint(d)] += (rs.rand() - 0.5) * 2 * span.max()
        elif kind == 6:  # endpoints on cell corners
            a = lo + rs.randint(0, dim) * res
            b = lo + rs.randint(0, dim) * res
        else:  # corners and diagonals: equal steps on every axis
            a = lo + rs.randint(0, dim) * res
            b = a + rs.randint(-20, 21) * res
        out.append((a, b))
    p1 = np.array([a for a, _ in out])
    p2 = np.array([b for _, b in out])
    return p1, p2


def maps():
    z = np.load(GOLD)
    g = mp.VoxelGrid(z["skir_origin"], z["skir_dim"], float(z["skir_res"]))
    g.addCloud(z["skir_pts"].astype(np.float64))
    yield "skir3d", g.toMapUtil()
    rs = np.random.RandomState(5)
    for name, dim, origin, res in (("2d", (61, 47), (-3.1, 2.05), 0.25), ("2d_far", (40, 33), (5.0e6 + 0.3, -4.0e6), 0.1),
                                   ("3d_far", (24, 19, 11), (-5.0e6, 5.0e6 + 0.05, 1.0e5), 0.2)):
        data = np.where(rs.rand(int(np.prod(dim))) < 0.3, 100, 0).astype(np.int8)
        mu = mp.MapUtil(len(dim))
        mu.setMap(np.asarray(origin), np.asarray(dim), data, res)
        yield name, mu


@pytest.mark.parametrize("which", range(4))
def test_ray_trace_equals_oracle(which):
    name, mu = list(maps())[which]
    dim, origin, res = mu.getDim(), mu.getOrigin(), mu.getRes()
    rs = np.random.RandomState(100 + which)
    p1, p2 = rays(rs, origin, dim, res, 2000)
    want = [oracle_trace(origin, dim, res, a, b) for a, b in zip(p1, p2)]
    # one ray per call
    for i in range(0, len(p1), 7):
        assert np.array_equal(mu.rayTrace(p1[i], p2[i]), want[i]), (name, i)
    # all in one call
    cells, offs = mu.traceCells(p1, p2)
    assert offs[0] == 0 and offs[-1] == len(cells)
    for i in range(len(p1)):
        assert np.array_equal(cells[offs[i]:offs[i + 1]], want[i]), (name, i)
    lens = np.diff(offs)
    assert (lens == 0).sum() > 100 and lens.max() > 20  # empty rays (outside starts, short rays) and long ones
    if len(dim) == 3 and ov.ref_available():  # the reference's own MapUtil::rayTrace
        ref = ov.RefMapUtil(origin, dim, res, mu.getMap())
        for i in range(0, len(p1), 3):
            assert np.array_equal(ref.ray_trace(p1[i], p2[i]), want[i]), (name, i)


def test_device_variant_equals_host_and_cap_prefix():
    import torch
    name, mu = next(maps())
    dim, origin, res = mu.getDim(), mu.getOrigin(), mu.getRes()
    p1, p2 = rays(np.random.RandomState(7), origin, dim, res, 500)
    for ns, sel in ((None, mp.TRACE_ALL), (NS5, mp.TRACE_FREE), (None, mp.TRACE_OCCUPIED), (NS5, mp.TRACE_ALL)):
        cells, offs = mu.traceCells(p1, p2, ns, sel)
        total = len(cells)
        d1, d2 = torch.tensor(p1, device="cuda"), torch.tensor(p2, device="cuda")
        d_cells = torch.full((total + 5, 3), -7, dtype=torch.int32, device="cuda")
        d_offs = torch.zeros(len(p1) + 1, dtype=torch.int64, device="cuda")
        ns3 = None if ns is None else np.ascontiguousarray(ns)
        vp = lambda t: C.c_void_p(t.data_ptr())  # noqa: E731
        stream = torch.cuda.Stream()
        with torch.cuda.stream(stream):
            k = _lib.check(_lib.lib().mplb_map_trace_cells_device(mu._h, vp(d1), vp(d2), len(p1), _lib.ptr(ns3), 0 if ns is None else len(ns),
                                                                  sel, vp(d_cells), total + 5, vp(d_offs), C.c_void_p(stream.cuda_stream)))
        stream.synchronize()
        assert k == total
        got = d_cells.cpu().numpy()
        assert np.array_equal(got[:total], cells) and np.all(got[total:] == -7)
        assert np.array_equal(d_offs.cpu().numpy(), offs)
        # a cap below the total: the total is returned and only the prefix written
        cap = total // 3
        out = np.full((total, 3), -9, dtype=np.int32)
        o2 = np.zeros(len(p1) + 1, dtype=np.int64)
        k = _lib.check(_lib.lib().mplb_map_trace_cells(mu._h, _lib.ptr(p1), _lib.ptr(p2), len(p1), _lib.ptr(ns3),
                                                       0 if ns is None else len(ns), sel, _lib.ptr(out), cap, _lib.ptr(o2)))
        assert k == total and np.array_equal(out[:cap], cells[:cap]) and np.all(out[cap:] == -9) and np.array_equal(o2, offs)


def test_rejected_endpoints():
    name, mu = next(maps())
    origin = mu.getOrigin()
    good = np.array([origin + 1.0])
    for bad in (np.array([[np.nan, 1.0, 1.0]]), np.array([[1.0, np.inf, 1.0]]), np.array([[1e300, 0.0, 0.0]]),
                np.array([[origin[0] + 1.0 + mu.getRes() * 0.8 * (2.0 ** 31 + 1000), origin[1], origin[2]]])):
        for a, b in ((good, bad), (bad, good)):
            with pytest.raises(mp.MplbError):
                mu.traceCells(a, b)
    # just below the limit the ray is accepted and traced until it leaves the map
    ok = np.array([[origin[0] + 1.0 + mu.getRes() * 0.8 * (2.0 ** 31 - 1000), origin[1] + 1.0, origin[2] + 1.0]])
    cells, _ = mu.traceCells(good, ok)
    assert len(cells) > 0


def node_map():
    import voxel_flow
    z = np.load(GOLD)
    g = mp.VoxelGrid(*voxel_flow.geometry(z))
    g.addCloud(z["simple_pts"].astype(np.float64))
    mu = g.toMapUtil()
    mu.freeUnknown()
    return z, g, mu


def oracle_select(mu, p1, p2, add):
    """the node's selection with the oracle's rayTrace and the map's values (voxel_flow.oracle_cells_edit)"""
    pns = ov.ray_trace(mu.getOrigin(), mu.getDim(), mu.getRes(), p1, p2)
    if add:
        cand = (pns[:, None, :] + NS5[None, :, :]).reshape(-1, 3)
        v = mu.getCells(cand)
        return cand[(v >= 0) & (v < 100)]
    return pns[mu.getCells(pns) == 100]


def test_node_selection_equals_fixture_and_oracle():
    z, g, mu = node_map()
    pa, pc = (z["replanner_" + k].astype(np.float64) for k in ("add_cloud", "clear_cloud"))
    free, offs = mu.traceCells([pa[0]], [pa[-1]], NS5, mp.TRACE_FREE)
    assert np.array_equal(free, z["flow_cells_0"]) and np.array_equal(free, oracle_select(mu, pa[0], pa[-1], True))
    assert offs.tolist() == [0, len(free)]
    assert len(np.unique(free, axis=0)) < len(free)  # overlapping stencils: duplicates are kept, as in new_obs
    g.fillColumns(free)
    g.writeMap(mu)
    occ, _ = mu.traceCells([pc[0]], [pc[-1]], None, mp.TRACE_OCCUPIED)
    assert np.array_equal(occ, z["flow_cells_1"]) and np.array_equal(occ, oracle_select(mu, pc[0], pc[-1], False))
    # stencil cells outside the map: FREE drops them, ALL keeps them
    dim, origin, res = mu.getDim(), mu.getOrigin(), mu.getRes()
    a = origin + (np.array([0.5, 0.5, 0.5]) + [0, 0, 0]) * res
    b = origin + (np.array([0.5, dim[1] - 0.5, 0.5])) * res
    allc, _ = mu.traceCells([a], [b], NS5, mp.TRACE_ALL)
    freec, _ = mu.traceCells([a], [b], NS5, mp.TRACE_FREE)
    outside = np.any((allc < 0) | (allc >= dim), axis=1)
    assert outside.any() and not np.any(np.any((freec < 0) | (freec >= dim), axis=1))
    ray = mu.rayTrace(a, b)
    assert len(allc) == len(ray) * len(NS5)


def test_replanner_flow_with_the_edit_on_the_device():
    """voxel_flow.run with trace -> *_device fill / clear -> write_map -> mplb_lpa_update_nodes_batch_device: equal to the
    fixture recorded from the reference and to the oracle's flow"""
    import torch
    import lpa_flow
    import oracle
    import voxel_flow
    from test_gpu_lpa import GpuPlanner
    from test_gpu_voxel_grid import Dev
    z = np.load(GOLD)
    d = Dev(*voxel_flow.geometry(z))
    d.add_cloud(z["simple_pts"].astype(np.float64))

    class Map:
        mu = d.g.toMapUtil()
    Map.mu.freeUnknown()
    L = _lib.lib()
    vp = lambda t: C.c_void_p(t.data_ptr())  # noqa: E731
    pending = {}

    class DevicePlanner(GpuPlanner):
        def _update(self, cells, blocked):
            dc, n = pending.pop("cells")
            assert n == len(cells)
            h = (C.c_void_p * 1)(self.pl._h)
            offs = np.array([0, n], dtype=np.int64)
            v = np.zeros(1, dtype=np.int32)
            _lib.check(L.mplb_lpa_update_nodes_batch_device(h, 1, int(blocked), vp(dc), _lib.ptr(offs), _lib.ptr(v)))
            return int(v[0])

        def lpa_update_blocked_nodes(self, pns):
            return self._update(pns, True)

        def lpa_update_cleared_nodes(self, pns):
            return self._update(pns, False)

    pl = DevicePlanner(3)
    pl.set_map(Map)
    voxel_flow.configure(pl)

    def edit(add, p1, p2):
        d1 = torch.tensor(np.asarray(p1, dtype=np.float64)[None], device="cuda")
        d2 = torch.tensor(np.asarray(p2, dtype=np.float64)[None], device="cuda")
        cap = 1 << 14
        dc = torch.zeros((cap, 3), dtype=torch.int32, device="cuda")
        do = torch.zeros(2, dtype=torch.int64, device="cuda")
        ns = NS5 if add else None
        n = _lib.check(L.mplb_map_trace_cells_device(Map.mu._h, vp(d1), vp(d2), 1, _lib.ptr(ns), 0 if ns is None else len(ns),
                                                     mp.TRACE_FREE if add else mp.TRACE_OCCUPIED, vp(dc), cap, vp(do), None))
        assert n <= cap
        if add:
            _lib.check(L.mplb_voxel_grid_fill_device(d.g._h, vp(dc), n, 1, None))
        else:
            _lib.check(L.mplb_voxel_grid_clear_columns_device(d.g._h, vp(dc), n, None))
        d.g.writeMap(Map.mu)
        pending["cells"] = (dc, n)
        return dc[:n].cpu().numpy()

    snaps, edits = voxel_flow.run(z, d, pl, edit)
    voxel_flow.check(snaps, edits, z)
    a, ea = voxel_flow.host_flow(z, ov.OracleVoxelGrid, oracle.OracleMap, oracle.OraclePlanner)
    lpa_flow.assert_same(a, snaps, "replanner on the device")
    assert edits[0]["updated"] > 0 and len(edits[1]["cells"]) > 0 and not pending


def test_map_set_cells_device_equals_host():
    import torch
    rs = np.random.RandomState(3)
    dim = np.array([30, 20, 7])
    data = np.where(rs.rand(int(np.prod(dim))) < 0.2, 100, 0).astype(np.int8)
    a, b = mp.MapUtil(3), mp.MapUtil(3)
    for m in (a, b):
        m.setMap(np.array([-1.0, 2.0, 0.5]), dim, data, 0.3)
    cells = np.stack([rs.randint(-2, d + 2, 400) for d in dim], axis=1).astype(np.int32)
    for v in (100, 0):
        a.setCells(cells[:250] if v else cells[150:], v)
        c = torch.tensor(cells[:250] if v else cells[150:], device="cuda")
        _lib.check(_lib.lib().mplb_map_set_cells_device(b._h, C.c_void_p(c.data_ptr()), len(c), v, None))
        assert np.array_equal(a.getMap(), b.getMap())
