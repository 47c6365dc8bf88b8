"""A fleet of LPA* replanners on ONE shared map, and the same fleet sharded over the ranks of a libmplb communicator
(mplb_fleet_map_edit, mplb_fleet_plan, mpl_ros_b200.dist.ShardedFleet; DESIGN.md section 6.1).

The reference run steps the fleet on one device with the single-device calls: every robot traces its edit on the map
(mplb_map_trace_cells: a ray across the middle of its trajectory, the isFree cells of a 3 x 3 stencil), the map takes the
concatenation of all edits, then getLinkedNodes, updateBlockedNodes (every robot receives the whole concatenation), plan and
getSubStateSpace(1) run as batches.  It is held to the oracle (one oracle planner per robot on one shared oracle map) after
every call.  The sharded run (robot i on rank i mod N, one map replica per rank) must leave every planner bit-identical to the
reference run after every call: hm_ dump, heap, best_child_, linked points, capacity, results, trajectories and the replicas.

Potential-map sessions stay out of the shared map (updatePotentialMap rewrites the map it is given): they run in the fleet of
per-robot maps of the two-GPU test, where only the plan is collective."""
import os
import sys
import time

import numpy as np
import pytest

import mpl_ros_b200 as mp
import oracle
import lpa_flow
import lpa_shaped_flow as F
from helpers import load_config
from mpl_ros_b200 import _lib, dist as mdist, maps
from test_gpu_lpa import GpuMap
from test_gpu_lpa_shaped import GpuPlanner

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NS3 = np.array([(x, y, 0) for x in range(-1, 2) for y in range(-1, 2)], dtype=np.int32)


def robot_specs(kind):
    """(map config, [(control, U, params, start waypoint, goal waypoint, oracle class)]) of a shared-map fleet: several start /
    goal pairs on one map, drawn with a fixed seed"""
    if kind in ("skir", "corridor"):
        m, dim, params, U, start, goal = load_config(kind)
        S, G = maps.sample_queries(m, 5, seed=11, min_dist=1.5, max_dist=4.0)
        pairs = [(start, goal)] + list(zip(S, G))
        out = []
        for s, g in pairs:
            sw, gw = F.waypoints(s, lpa_flow.ACC, 0.0), F.waypoints(g, lpa_flow.ACC, 0.0)
            out.append((lpa_flow.ACC, U, dict(params), sw, gw, oracle.OraclePlanner))
        if kind == "corridor":  # the yaw session of tests/lpa_shaped_flow.py and one more yaw robot on the same map
            f = F.FLOWS["corridor_yaw"]
            Uy = F.controls(U, f["u_yaw"])
            for s, g, y in ((start, goal, f["start_yaw"]), (pairs[1][0], pairs[1][1], 0.0)):
                out.append((f["control"], Uy, dict(params, **f["params"]), F.waypoints(s, f["control"], y),
                            F.waypoints(g, f["control"], 0.0), F.OraclePlanner))
        return m, dim, out
    raise KeyError(kind)


def random_specs(n=16):
    """16 seeded random replanners on one random 3-D map (ACC, |U| = 27)"""
    rng = np.random.default_rng(5)
    nd = np.array([24, 20, 6])
    data = np.where(rng.random(int(np.prod(nd))) < 0.12, 100, 0).astype(np.int8)

    class M:
        pass
    m = M()
    m.origin, m.dim, m.res, m.data, m.ndim = np.array([-1.0, -2.0, 0.0]), nd, 0.25, data, 3
    U = maps.make_U(1.0, 1, 3)
    free = np.flatnonzero(data == 0)
    cells = np.stack([free % nd[0], (free // nd[0]) % nd[1], free // (nd[0] * nd[1])], axis=1)
    pick = rng.choice(len(free), size=(n, 2), replace=False)
    S, G = ((cells[pick[:, k]] + 0.5) * m.res + m.origin for k in range(2))  # free cell centres
    params = dict(v_max=2.0, a_max=1.0, dt=1.0, tol_pos=0.5, max_num=4000)
    return m, 3, [(lpa_flow.ACC, U, params, F.waypoints(s, lpa_flow.ACC, 0.0), F.waypoints(g, lpa_flow.ACC, 0.0), oracle.OraclePlanner)
                  for s, g in zip(S, G)]


def make_planner(cls, dim, m_obj, spec):
    control, U, params, sw, gw, _ = spec
    p = cls(dim)
    p.set_map(m_obj)
    for k, v in params.items():
        p.set_param(k, v)
    p.set_controls(U)
    p._lpa_control = control
    return p


class Reference:
    """the reference run: every robot on one GpuMap, the single-device batch calls, and the oracle beside it"""

    def __init__(self, m, dim, specs, with_oracle=True):
        self.m, self.dim, self.specs = m, dim, specs
        self.gm = GpuMap(m.origin, m.dim, m.data, m.res)
        self.gm.free_unknown()
        self.rob = [make_planner(GpuPlanner, dim, self.gm, s) for s in specs]
        self.s = [s[3] for s in specs]
        self.g = [s[4] for s in specs]
        self.om = None
        if with_oracle:
            self.om = oracle.OracleMap(m.origin, m.dim, m.data, m.res)
            self.om.free_unknown()
            self.orc = [make_planner(s[5], dim, self.om, s) for s in specs]
            self.oracle_ok = [True] * len(specs)

    def pls(self):
        return [r.pl for r in self.rob]

    def traced(self):
        """each robot's edit c_i, traced on the map as it is now"""
        out = []
        for r in self.rob:
            best = r.lpa_best_child_states()[:, :self.dim]
            if len(best) < 4:
                out.append(np.zeros((0, 3), dtype=np.int32))
                continue
            c, _ = self.gm.mu.traceCells(best[len(best) // 3][None], best[2 * len(best) // 3][None], NS3[:, :self.dim], mp.TRACE_FREE)
            out.append(mdist._rows3(c))
        return out

    def edit(self, lists, value=100):
        cells = np.concatenate(lists) if lists else np.zeros((0, 3), dtype=np.int32)
        if len(cells):
            self.gm.set_cells(cells[:, :self.dim], value)
            if self.om is not None:
                self.om.set_cells(cells[:, :self.dim], value)
        return cells

    def plan(self):
        n = len(self.rob)
        s, g = mp.waypoints_array(n), mp.waypoints_array(n)
        for i in range(n):
            s[i], g[i] = self.s[i][0], self.g[i][0]
        mp.MapPlanner.planLPABatch(self.pls(), s, g)
        res = [self._rec(r) for r in self.rob]
        if self.om is not None:
            for i, o in enumerate(self.orc):
                if not self.oracle_ok[i]:
                    continue
                ro = o.lpa_plan(self.s[i], self.g[i])
                if int(ro["status"]) == 3 and int(ro["pops"]) == 0 or o.lpa_last_fault() & 2:
                    self.oracle_ok[i] = False  # the reference reads an empty heap / walks a cycle here: no verdict
                    continue
                lpa_flow.assert_same([lpa_flow.snapshot(o, ro)], [lpa_flow.snapshot(self.rob[i], res[i])], "plan %d oracle" % i)
        return res

    @staticmethod
    def _rec(r):
        rec = np.zeros(1, dtype=oracle.RESULT_DTYPE)[0]
        for f in oracle.RESULT_DTYPE.names:
            rec[f] = r.pl.result()[f]
        return rec

    def links(self):
        got = mp.MapPlanner.getLinkedNodesBatch(self.pls())
        if self.om is not None:
            for i, o in enumerate(self.orc):
                if self.oracle_ok[i]:
                    lo = o.lpa_get_linked_nodes()
                    assert np.array_equal(lo[:, :self.dim], got[i]), ("linked oracle", i)
        return got

    def update(self, cells):
        v = mp.MapPlanner.updateBlockedNodesBatch(self.pls(), [cells[:, :self.dim]] * len(self.rob))
        self.check_oracle("blocked", lambda o: o.lpa_update_blocked_nodes(cells[:, :self.dim]) if len(cells) else None)
        return v

    def subtree(self):
        n_best = [len(r.lpa_best_child()) for r in self.rob]
        ts = [1 if n > 2 else 0 for n in n_best]
        nxt = [r.lpa_waypoint(1) if t else None for r, t in zip(self.rob, ts)]
        sizes = mp.MapPlanner.getSubStateSpaceBatch(self.pls(), ts)
        if self.om is not None:
            for i, o in enumerate(self.orc):
                if self.oracle_ok[i] and n_best[i] and o.lpa_get_sub_state_space(ts[i]) < 0:
                    self.oracle_ok[i] = False
            self.check_oracle("subtree", lambda o: None)
        for i, w in enumerate(nxt):
            if w is not None:
                self.s[i] = w
        return ts, sizes

    def check_oracle(self, what, fn):
        for i, o in enumerate(self.orc if self.om is not None else []):
            if self.oracle_ok[i]:
                fn(o)
                lpa_flow.assert_same([lpa_flow.snapshot(o, None)], [lpa_flow.snapshot(self.rob[i], None)], "%s %d oracle" % (what, i))


def state(r):
    return (r.pl.lpaNodes().tobytes(), r.pl.lpaHeap().tobytes(), r.pl.lpaBestChild().tobytes(), r.pl.lpaCapacity())


def same_result(a, b):
    return all(a[f] == b[f] or (f == "cost" and np.isnan(a[f]) and np.isnan(b[f])) for f in a.dtype.names if f != "device_ms")


class Sharded:
    """the sharded run on this process's rank: its robots (rank, rank + N, ...) on its replica of the map"""

    def __init__(self, comm, m, dim, specs, device):
        self.dim, self.comm = dim, comm
        self.mu = comm.broadcast_map(dim, m.origin, m.dim, m.res, m.data, 0) if comm.rank == 0 else comm.broadcast_map(0)
        self.mu.freeUnknown()

        class Replica:
            pass
        rep = Replica()
        rep.mu = self.mu
        self.idx = mdist.shard_indices(len(specs), comm.rank, comm.size)
        self.rob = [make_planner(GpuPlanner, dim, rep, specs[i]) for i in self.idx]
        self.s = [specs[i][3] for i in self.idx]
        self.g = [specs[i][4] for i in self.idx]
        self.fleet = mdist.ShardedFleet([r.pl for r in self.rob], len(specs), self.mu, comm=comm, device=device)

    def plan(self, max_seg=256):
        return self.fleet.plan([w[0] for w in self.s], [w[0] for w in self.g], max_seg=max_seg)

    def subtree(self):
        ts = [1 if len(r.lpa_best_child()) > 2 else 0 for r in self.rob]
        nxt = [r.lpa_waypoint(1) if t else None for r, t in zip(self.rob, ts)]
        sizes = self.fleet.sub_state_space(ts)
        for k, w in enumerate(nxt):
            if w is not None:
                self.s[k] = w
        return sizes


def actions_of(r, max_seg):
    a = np.full(max_seg, -1, dtype=np.int32)
    if int(r.pl.result()["status"]) == 0:
        x = r.pl.getActions()[:max_seg]
        a[:len(x)] = x
    return a


@pytest.mark.parametrize("kind", ["skir", "corridor", "random"])
def test_shared_map_fleet_oracle_and_comm_of_one(kind):
    """two cycles of the reference run, held to the oracle after every call, and a communicator of size 1 running the sharded
    calls in lockstep with it: bit-identical after every call"""
    import torch
    m, dim, specs = random_specs() if kind == "random" else robot_specs(kind)
    ref = Reference(m, dim, specs)
    comm = mdist.Comm(mdist.Comm.unique_id(), 0, 1)
    sh = Sharded(comm, m, dim, specs, torch.device("cuda", 0))

    def compare(what, linked=None, got_linked=None):
        for i, (a, b) in enumerate(zip(ref.rob, sh.rob)):
            assert state(a) == state(b), (kind, what, i)
        assert np.array_equal(ref.gm.mu.getMap(), sh.mu.getMap()), (kind, what, "replica")
        if linked is not None:
            for i in range(len(linked)):
                assert np.array_equal(linked[i], got_linked[i]), (kind, what, "linked", i)

    max_seg = 256
    ref.plan()
    res, acts = sh.plan(max_seg)
    for i, r in enumerate(ref.rob):
        assert same_result(res[i], Reference._rec(r)) and np.array_equal(acts[i], actions_of(r, max_seg)), (kind, "plan", i)
    compare("first plan")
    edited = 0
    for cyc in range(2):
        lists = ref.traced()
        cells = ref.edit(lists)
        assert sh.fleet.map_edit(lists, 100) == len(cells)
        got_cells, got_offs = sh.fleet.edit_cells(), sh.fleet.edit_offsets()
        assert np.array_equal(got_cells, cells) and list(got_offs) == [0] + list(np.cumsum([len(c) for c in lists])), (kind, cyc)
        edited += len(cells)
        compare("edit %d" % cyc)
        lk = ref.links()
        compare("links %d" % cyc, lk, sh.fleet.links())
        v_ref = ref.update(cells)
        assert sh.fleet.update(True) == v_ref, (kind, cyc)
        compare("update %d" % cyc)
        ref_res = ref.plan()
        res, acts = sh.plan(max_seg)
        for i, r in enumerate(ref.rob):
            assert same_result(res[i], ref_res[i]) and np.array_equal(acts[i], actions_of(r, max_seg)), (kind, "plan", cyc, i)
            pa, pb = r.pl.getTraj().getPrimitives(), sh.rob[i].pl.getTraj().getPrimitives()
            assert len(pa) == len(pb) and all(np.array_equal(x.coeffs, y.coeffs) for x, y in zip(pa, pb)), (kind, cyc, i)
        compare("plan %d" % cyc)
        _, sizes = ref.subtree()
        assert sh.subtree() == sizes, (kind, cyc)
        compare("subtree %d" % cyc)
    assert edited > 0
    assert sum(ref.oracle_ok) >= len(specs) - 2


def test_sharded_calls_launch_the_same_for_any_fleet_size():
    """the launches of mplb_fleet_map_edit and mplb_fleet_plan do not grow with the number of robots, and argument errors
    change no planner"""
    import torch
    L = _lib.lib()
    counts = {}
    for n in (2, 12):
        m, dim, specs = robot_specs("skir")
        specs = (specs * 3)[:n]
        comm = mdist.Comm(mdist.Comm.unique_id(), 0, 1)
        sh = Sharded(comm, m, dim, specs, torch.device("cuda", 0))
        sh.plan()
        sh.fleet.links()
        lists = [np.array([[3 + k % 4, 4, 1]], dtype=np.int32) for k in range(n)]
        sh.fleet.map_edit(lists, 100)  # buffers grow on the first call
        steps = []
        for fn in (lambda: sh.fleet.map_edit(lists, 0), lambda: sh.plan()):
            c0 = L.mplb_launch_count()
            fn()
            steps.append(int(L.mplb_launch_count() - c0))
        counts[n] = steps
        before = [state(r) for r in sh.rob]
        h = mp.MapPlanner._handles([r.pl for r in sh.rob] + [sh.rob[0].pl])
        s, g = mp.waypoints_array(n + 1), mp.waypoints_array(n + 1)
        res = np.zeros(n + 1, dtype=_lib.RESULT_DTYPE)
        for bad in ((h, n + 1, n + 1), (h, n, n + 1)):  # a planner listed twice; n_local not what the striping gives
            assert L.mplb_fleet_plan(comm._h, bad[0], bad[1], bad[2], _lib.ptr(s), _lib.ptr(g), _lib.ptr(res), None, 0, 0) < 0
        off = mp.MapPlanner(3)  # LPA* off
        off.setMapUtil(sh.mu)
        h2 = mp.MapPlanner._handles([off])
        assert L.mplb_fleet_plan(comm._h, h2, 1, 1, _lib.ptr(s), _lib.ptr(g), _lib.ptr(res), None, 0, 0) < 0
        assert L.mplb_fleet_plan(comm._h, None, 1, 1, _lib.ptr(s), _lib.ptr(g), _lib.ptr(res), None, 0, 0) < 0
        assert [state(r) for r in sh.rob] == before
    assert counts[2] == counts[12], counts


def test_device_merge_of_several_ranks_payloads():
    """the scan and merge kernels of mplb_fleet_map_edit on the payloads of N = 1 .. 4 ranks (built on the host as each rank
    packs them): robot i = the (i / N)-th robot of rank i mod N lands at the prefix of robots 0 .. i-1, empty lists and ranks
    without robots included; counts that do not add up to a payload's rows are refused"""
    import ctypes as C
    import torch
    L = _lib.lib()
    rng = np.random.default_rng(3)
    for R, N in ((1, 1), (5, 2), (2, 3), (7, 3), (33, 4), (300, 3)):
        lists = [rng.integers(-5, 50, (int(rng.integers(0, 6)) if i % 4 else 0, 3)).astype(np.int32) for i in range(R)]
        parts = [mdist.pack_edits([lists[i] for i in mdist.shard_indices(R, r, N)]) for r in range(N)]
        words = [np.concatenate([c.astype(np.int32), w.reshape(-1)]).astype(np.int32) for c, w in parts]
        d_pay = torch.as_tensor(np.concatenate(words)).cuda()
        nw = np.array([len(w) for w in words], dtype=np.int64)
        want_cells, want_offs = mdist.merge_edits(parts, R)
        cap = max(len(want_cells), 1)
        d_all = torch.full((cap, 3), -7, dtype=torch.int32, device="cuda")
        d_off = torch.zeros(R + 1, dtype=torch.int64, device="cuda")
        vp = lambda t: C.c_void_p(t.data_ptr())  # noqa: E731
        T = _lib.check(L.mplb_fleet_merge_device(vp(d_pay), _lib.ptr(nw), N, R, vp(d_all), vp(d_off), cap, None))
        assert T == len(want_cells), (R, N)
        assert np.array_equal(d_all[:T].cpu().numpy(), want_cells) and np.array_equal(d_off.cpu().numpy(), want_offs), (R, N)
        if len(want_cells):
            assert L.mplb_fleet_merge_device(vp(d_pay), _lib.ptr(nw), N, R, vp(d_all), vp(d_off), T - 1, None) == T  # too small
            bad = np.concatenate(words).astype(np.int32)
            k = next(r for r in range(N) if len(parts[r][0]))
            bad[int(nw[:k].sum())] += 1  # the first count of rank k no longer adds up to its rows
            assert L.mplb_fleet_merge_device(vp(torch.as_tensor(bad).cuda()), _lib.ptr(nw), N, R, vp(d_all), vp(d_off), cap,
                                             None) == -1


def test_map_edit_size_query_small_cap_and_errors():
    """with one rank: a size query and a cap below the total apply nothing; an argument error is an error"""
    import ctypes as C
    import torch
    m, dim, specs = robot_specs("skir")
    comm = mdist.Comm(mdist.Comm.unique_id(), 0, 1)
    mu = comm.broadcast_map(dim, m.origin, m.dim, m.res, m.data, 0)
    mu.freeUnknown()
    L = _lib.lib()
    before = mu.getMap().copy()
    rows = np.array([[3, 4, 1], [5, 6, 1], [7, 8, 2]], dtype=np.int32)
    d_rows = torch.as_tensor(rows).cuda()
    offs = np.array([0, 1, 1, 3], dtype=np.int64)
    d_all = torch.zeros((2, 3), dtype=torch.int32, device="cuda")
    d_off = torch.zeros(4, dtype=torch.int64, device="cuda")
    vp = lambda t: C.c_void_p(t.data_ptr())  # noqa: E731
    assert L.mplb_fleet_map_edit(comm._h, mu._h, vp(d_rows), _lib.ptr(offs), 3, 100, None, None, 0, None) == 3  # size query
    assert L.mplb_fleet_map_edit(comm._h, mu._h, vp(d_rows), _lib.ptr(offs), 3, 100, vp(d_all), vp(d_off), 2, None) == 3
    assert np.array_equal(mu.getMap(), before)
    assert L.mplb_fleet_map_edit(comm._h, mu._h, None, _lib.ptr(offs), 3, 100, vp(d_all), vp(d_off), 2, None) == -1
    bad = np.array([0, 2, 1, 3], dtype=np.int64)
    assert L.mplb_fleet_map_edit(comm._h, mu._h, vp(d_rows), _lib.ptr(bad), 3, 100, vp(d_all), vp(d_off), 2, None) == -1
    d_all = torch.zeros((3, 3), dtype=torch.int32, device="cuda")
    assert L.mplb_fleet_map_edit(comm._h, mu._h, vp(d_rows), _lib.ptr(offs), 3, 100, vp(d_all), vp(d_off), 3, None) == 3
    assert np.array_equal(d_all.cpu().numpy(), rows) and list(d_off.cpu().numpy()) == [0, 1, 1, 3]
    g = mu.getMap().reshape(-1)
    nd = m.dim
    assert all(g[x + nd[0] * y + nd[0] * nd[1] * z] == 100 for x, y, z in rows)


def test_per_robot_maps_gather_only():
    """a fleet whose robots each own a map (potential-map and yaw sessions included) through mplb_fleet_plan with one rank:
    the gathered records and actions equal the same robots planned with planLPABatch"""
    comm = mdist.Comm(mdist.Comm.unique_id(), 0, 1)
    a = [Member_own(n) for n in PER_ROBOT]
    b = [Member_own(n) for n in PER_ROBOT]
    fl = mdist.ShardedFleet([x.pl for x in a], len(a), None, comm=comm)
    res, acts = fl.plan([x.s[0] for x in a], [x.g[0] for x in a], max_seg=256)
    mp.MapPlanner.planLPABatch([x.pl for x in b], [x.s[0] for x in b], [x.g[0] for x in b])
    for i, (x, y) in enumerate(zip(a, b)):
        assert same_result(res[i], np.array(y.pl.result(), dtype=_lib.RESULT_DTYPE)[()]), PER_ROBOT[i]
        assert np.array_equal(acts[i], actions_of(y, 256)), PER_ROBOT[i]
        assert state(x) == state(y), PER_ROBOT[i]
    assert sum(int(r["status"]) == 0 for r in res) >= 3


# ---- two GPUs: ranks 0 and 1 against the single-device reference run built from the same seeds

def _two_rank_worker(rank, world, idfile, out_dir):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import torch
    torch.cuda.set_device(rank)
    torch.zeros(1, device="cuda")
    from mpl_ros_b200 import dist as md
    if rank == 0:
        with open(idfile + ".tmp", "wb") as f:
            f.write(md.Comm.unique_id())
        os.replace(idfile + ".tmp", idfile)
    while not os.path.exists(idfile):
        time.sleep(0.05)
    comm = md.Comm(open(idfile, "rb").read(), rank, world)
    m, dim, specs = robot_specs("skir")
    sh = Sharded(comm, m, dim, specs, torch.device("cuda", rank))
    log = {}

    def dump(tag, extra=None):
        for k, i in enumerate(sh.idx):
            r = sh.rob[k]
            log["%s_state_%d" % (tag, i)] = np.frombuffer(b"".join(state(r)[:3]), dtype=np.uint8)
            log["%s_cap_%d" % (tag, i)] = np.array(list(state(r)[3].values()))
        log["%s_map_%d" % (tag, rank)] = sh.mu.getMap().reshape(-1)
        for key, v in (extra or {}).items():
            log["%s_%s" % (tag, key)] = v

    res, acts = sh.plan()
    dump("p0", {"res": res.view(np.uint8), "acts": acts} if rank == 0 else None)
    edits = np.load(os.path.join(out_dir, "edits.npz"))
    for cyc in range(3):
        lists = [edits["c%d_%d" % (cyc, i)] for i in sh.idx]
        sh.fleet.map_edit(lists, 100)
        cells, offs = sh.fleet.edit_cells(), sh.fleet.edit_offsets()
        dump("e%d" % cyc, {"cells_%d" % rank: cells, "offs_%d" % rank: offs})
        lk = sh.fleet.links()
        dump("l%d" % cyc, {"linked_%d" % i: lk[k] for k, i in enumerate(sh.idx)})
        sh.fleet.update(True)
        dump("u%d" % cyc)
        res, acts = sh.plan()
        dump("q%d" % cyc, {"res": res.view(np.uint8), "acts": acts} if rank == 0 else None)
        sh.subtree()
        dump("s%d" % cyc)
    # caps that differ between ranks: every rank fails alike, nothing applied
    import ctypes as C
    before = sh.mu.getMap().copy()
    d_all = torch.zeros((4096, 3), dtype=torch.int32, device="cuda")
    d_off = torch.zeros(len(specs) + 1, dtype=torch.int64, device="cuda")
    offs = np.zeros(len(sh.idx) + 1, dtype=np.int64)
    rc = _lib.lib().mplb_fleet_map_edit(comm._h, sh.mu._h, None, _lib.ptr(offs), len(sh.idx), 100, C.c_void_p(d_all.data_ptr()),
                                        C.c_void_p(d_off.data_ptr()), 4096 - rank, None)
    log["unequal_cap_rc_%d" % rank] = np.array([rc])
    assert np.array_equal(sh.mu.getMap(), before)
    # a fleet of per-robot maps (potential-map and yaw sessions included): only the plan is collective
    own = [Member_own(n) for n in PER_ROBOT]
    mine = [own[i] for i in md.shard_indices(len(own), rank, world)]
    fl = md.ShardedFleet([x.pl for x in mine], len(own), None, comm=comm)
    res, acts = fl.plan([x.s[0] for x in mine], [x.g[0] for x in mine], max_seg=256)
    if rank == 0:
        log["own_res"], log["own_acts"] = res.view(np.uint8), acts
    np.savez(os.path.join(out_dir, "rank%d.npz" % rank), **log)


PER_ROBOT = ("simple_pot_local", "corridor_pot_grad", "corridor_yaw", "skir_acc_flow")


class Member_own:
    """one robot with its own map: a tests/lpa_shaped_flow.py session, or the skir_acc flow"""

    def __init__(self, name):
        if name == "skir_acc_flow":
            _, self.mp_, p, dim, start, goal = lpa_flow.build(GpuMap, GpuPlanner, "skir")
            control = lpa_flow.ACC
        else:
            f = F.FLOWS[name]
            _, self.mp_, p, dim, start, goal = F.build(name, GpuMap, GpuPlanner)
            control = f["control"]
            if f.get("pot"):
                p.update_potential_map(np.r_[start, np.zeros(3 - dim)])
        self.pl = p.pl
        self.s = F.waypoints(start, control, F.FLOWS.get(name, {}).get("start_yaw", 0.0))
        self.g = F.waypoints(goal, control, 0.0)


def test_two_ranks_equal_the_single_device_run(tmp_path):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    import torch.multiprocessing as tmp
    m, dim, specs = robot_specs("skir")
    ref = Reference(m, dim, specs, with_oracle=False)
    R = len(specs)
    ref_log = {}

    def rdump(tag):
        for i, r in enumerate(ref.rob):
            ref_log["%s_state_%d" % (tag, i)] = np.frombuffer(b"".join(state(r)[:3]), dtype=np.uint8)
            ref_log["%s_cap_%d" % (tag, i)] = np.array(list(state(r)[3].values()))
        ref_log["%s_map" % tag] = ref.gm.mu.getMap().reshape(-1)

    def rplan(tag):
        res = ref.plan()
        ref_log[tag + "_res"] = np.array(res, dtype=oracle.RESULT_DTYPE)
        ref_log[tag + "_acts"] = np.array([actions_of(r, 256) for r in ref.rob])
        rdump(tag)

    rplan("p0")
    edits = {}
    for cyc in range(3):
        lists = ref.traced()
        if cyc == 1:  # only rank 1's robots edit
            lists = [c if i % 2 == 1 else np.zeros((0, 3), dtype=np.int32) for i, c in enumerate(lists)]
        if cyc == 2:  # robot 0 (rank 0) drops its edit on robot 1's (rank 1) trajectory
            path = ref.rob[1].lpa_best_child_states()[:, :dim]
            lists = [np.zeros((0, 3), dtype=np.int32) for _ in range(R)]
            lists[0] = mdist._rows3(lpa_flow.cells_on_path(m, dim, path[len(path) // 2:len(path) // 2 + 1], 1))
            before = ref.rob[1].lpa_best_child().copy()
        for i, c in enumerate(lists):
            edits["c%d_%d" % (cyc, i)] = c
        cells = ref.edit(lists)
        ref_log["e%d_cells" % cyc] = cells
        ref_log["e%d_offs" % cyc] = np.concatenate([[0], np.cumsum([len(c) for c in lists])]).astype(np.int64)
        rdump("e%d" % cyc)
        lk = ref.links()
        for i in range(R):
            ref_log["l%d_linked_%d" % (cyc, i)] = lk[i]
        rdump("l%d" % cyc)
        ref.update(cells)
        rdump("u%d" % cyc)
        rplan("q%d" % cyc)
        if cyc == 2:
            assert not np.array_equal(ref.rob[1].lpa_best_child(), before)  # robot 1 replanned around robot 0's edit
        ref.subtree()
        rdump("s%d" % cyc)
    np.savez(str(tmp_path / "edits.npz"), **edits)
    tmp.spawn(_two_rank_worker, args=(2, str(tmp_path / "nccl_id"), str(tmp_path)), nprocs=2, join=True)
    z = [np.load(str(tmp_path / ("rank%d.npz" % r))) for r in range(2)]
    tags = ["p0"] + ["%s%d" % (t, c) for c in range(3) for t in ("e", "l", "u", "q", "s")]
    for tag in tags:
        for i in range(R):
            zr = z[i % 2]
            assert np.array_equal(zr["%s_state_%d" % (tag, i)], ref_log["%s_state_%d" % (tag, i)]), (tag, i)
            assert np.array_equal(zr["%s_cap_%d" % (tag, i)], ref_log["%s_cap_%d" % (tag, i)]), (tag, i)
        for r in range(2):
            assert np.array_equal(z[r]["%s_map_%d" % (tag, r)], ref_log["%s_map" % tag]), (tag, r)
        if tag[0] in "pq":
            got = z[0][tag + "_res"].view(_lib.RESULT_DTYPE).reshape(-1)
            assert all(same_result(got[i], ref_log[tag + "_res"][i]) for i in range(R)), tag
            assert np.array_equal(z[0][tag + "_acts"], ref_log[tag + "_acts"]), tag
        if tag[0] == "e":
            for r in range(2):
                assert np.array_equal(z[r]["%s_cells_%d" % (tag, r)], ref_log[tag + "_cells"]), (tag, r)
                assert np.array_equal(z[r]["%s_offs_%d" % (tag, r)], ref_log[tag + "_offs"]), (tag, r)
        if tag[0] == "l":
            for i in range(R):
                assert np.array_equal(z[i % 2]["%s_linked_%d" % (tag, i)], ref_log["%s_linked_%d" % (tag, i)]), (tag, i)
    assert all(int(z[r]["unequal_cap_rc_%d" % r][0]) == -1 for r in range(2))
    # per-robot maps: the gathered plans equal each robot planned on one device
    own = [Member_own(n) for n in PER_ROBOT]
    mp.MapPlanner.planLPABatch([x.pl for x in own], [x.s[0] for x in own], [x.g[0] for x in own])
    got = z[0]["own_res"].view(_lib.RESULT_DTYPE).reshape(-1)
    for i, x in enumerate(own):
        assert same_result(got[i], np.array(x.pl.result(), dtype=_lib.RESULT_DTYPE)[()]), PER_ROBOT[i]
        assert np.array_equal(z[0]["own_acts"][i], actions_of(x, 256)), PER_ROBOT[i]
