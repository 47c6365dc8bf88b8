"""LPA* with a potential map and with yaw controls on the GPU (k_lpa_plan_shaped) against the checker in its correctly rounded
trig mode, EXACTLY (tolerance 0): result records, the state space in hm_ order (key, g, rhs, h, flags, hashes of the stored
successor and predecessor lists), the priority-queue array, best_child_, the linked points, the trajectory's action ids — over
the flows of tests/lpa_shaped_flow.py.  The potential-only flows (no trig involved) are also compared with the fixture recorded
from the reference's own LPA* sources (tests/golden/lpa_shaped_flows.npz).  A batch that mixes plain, potential, yaw and
potential + yaw replanners equals the same planners planned one by one, and seeded edit / replan sequences equal the checker."""
import ctypes as C
import os

import numpy as np
import pytest

import mpl_ros_b200 as mp
from mpl_ros_b200 import _lib
import oracle
import lpa_flow
import lpa_shaped_flow as F
from test_gpu_lpa import GpuMap, GpuPlanner as _GpuPlanner

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden", "lpa_shaped_flows.npz")


class GpuPlanner(_GpuPlanner):
    """the call shapes of tests/lpa_shaped_flow.py over the product's MapPlanner"""

    def set_param(self, key, v):
        setters = {"potential_weight": self.pl.setPotentialWeight, "gradient_weight": self.pl.setGradientWeight,
                   "wyaw": self.pl.setWyaw, "yaw_max": self.pl.setYawmax, "j_max": self.pl.setJmax}
        if key in setters:
            setters[key](v)
        else:
            super().set_param(key, v)

    def set_vec(self, key, v):
        {"potential_radius": self.pl.setPotentialRadius, "potential_map_range": self.pl.setPotentialMapRange}[key](np.asarray(v)[:self.dim])

    def update_potential_map(self, pos):
        self.pl.updatePotentialMap(np.asarray(pos)[:self.dim])


GPU_EXTRA = {"skir_jrk_yaw": {"lpa_init_nodes": 4096, "lpa_init_preds": 65536},  # small arrays: the plan grows and resumes
             "skir_snp_yaw": {"lpa_init_nodes": 1024, "lpa_init_preds": 16384}}


@pytest.mark.parametrize("name", list(F.FLOWS))
def test_flow_equals_oracle(name):
    a, opl = F.run_flow(name, oracle.OracleMap, F.OraclePlanner)
    b, gp = F.run_flow(name, GpuMap, GpuPlanner, GPU_EXTRA.get(name))
    lpa_flow.assert_same(a, b, name)
    if name in F.POT_ONLY:
        gold = np.load(GOLD)[name]
        d = F.digest(b)
        assert len(d) == len(gold), name
        for f in gold.dtype.names:
            assert np.array_equal(d[f], gold[f]), (name, f)
    last = b[-1]["res"] if b[-1]["res"] is not None else b[-2]["res"]
    if int(last["status"]) == 0:  # getTraj(): the oracle's recoverTraj action ids, primitives rebuilt with the yaw channel
        assert np.array_equal(gp.pl.getActions(), opl.lpa_actions())
        prims = gp.pl.getTraj().getPrimitives()
        assert len(prims) == int(last["n_seg"])
        if F.FLOWS[name]["control"] & F.YAW:
            states = opl.lpa_best_child_states()
            U = np.asarray(gp.pl.U_)
            for i, (pr, act) in enumerate(zip(prims, opl.lpa_actions())):
                assert pr.yaw_coeff is not None and pr.yaw_coeff[5] == states[i][12] and pr.yaw_coeff[4] == U[act][gp.dim]
    if name in GPU_EXTRA:
        assert gp.pl.lpaCapacity()["grows"] > 0


def _single(kind, extra=None):
    return F.build(kind, GpuMap, GpuPlanner, extra)


def test_mixed_batch_equals_single_plans():
    """16 replanners of four kinds in one mplb_lpa_plan_batch (one launch per kind) equal the same planners planned alone,
    including a relaunch for neighbours that outgrow their arrays"""
    kinds = ["corridor_plain", "corridor_pot_grad", "corridor_yaw", "corridor_pot_yaw"]
    F.FLOWS.setdefault("corridor_plain", dict(config="corridor", control=F.ACC, params={}))
    try:
        batch, singles, wps = [], [], []
        for i in range(16):
            kind = kinds[i % 4]
            extra = {"lpa_init_nodes": 1024, "lpa_init_preds": 16384} if i % 5 == 0 else None
            for lst in (batch, singles):
                m, mp_, pl, dim, start, goal = _single(kind, extra)
                if F.FLOWS[kind].get("pot"):
                    pl.update_potential_map(np.r_[start, 0.0])
                lst.append(pl)
            wps.append((start, goal, F.FLOWS[kind]["control"], F.FLOWS[kind].get("start_yaw", 0.0)))
        n = len(batch)
        s, g = mp.waypoints_array(n), mp.waypoints_array(n)
        for i, (st, gl, c, y) in enumerate(wps):
            s["pos"][i, :2], g["pos"][i, :2] = st, gl
            s["control"][i] = g["control"][i] = c
            s["yaw"][i] = y
        res = np.zeros(n, dtype=_lib.RESULT_DTYPE)
        handles = (C.c_void_p * n)(*[p.pl._h for p in batch])
        _lib.check(_lib.lib().mplb_lpa_plan_batch(handles, n, _lib.ptr(s), _lib.ptr(g), _lib.ptr(res)))
        grew = 0
        for i in range(n):
            r1 = singles[i].lpa_plan(s[i:i + 1], g[i:i + 1])
            for f in ("status", "n_seg", "cost", "pops", "n_nodes", "n_open", "n_closed", "n_prims", "n_valid", "pop_hash", "closed_hash"):
                assert res[i][f] == r1[f], (i, f, res[i][f], r1[f])
            a, b = batch[i].lpa_nodes(), singles[i].lpa_nodes()
            for f in a.dtype.names:
                assert np.array_equal(a[f], b[f]), (i, f)
            assert np.array_equal(batch[i].lpa_heap(), singles[i].lpa_heap()), i
            if res[i]["status"] == 0:
                assert np.array_equal(batch[i].pl.getActions(), singles[i].pl.getActions()), i
            grew += batch[i].pl.lpaCapacity()["grows"] > 0
        assert grew >= 2
        assert len({float(r["cost"]) for r in res}) > 1
    finally:
        F.FLOWS.pop("corridor_plain", None)


FUZZ = [("corridor_pot_grad", 1), ("corridor_pot_grad", 2), ("corridor_yaw", 1), ("corridor_yaw", 2), ("corridor_pot_yaw", 1)]


@pytest.mark.parametrize("name,seed", FUZZ)
def test_seeded_edit_sequences(name, seed, steps=int(os.environ.get("MPLB_LPA_SHAPED_FUZZ_STEPS", "24"))):
    """random blocks / clears near the current trajectory, re-stamps of the potential map and root moves, replanning after
    each, against the checker step by step"""
    rng = np.random.default_rng(seed)
    sides = []
    for cm, cp in ((oracle.OracleMap, F.OraclePlanner), (GpuMap, GpuPlanner)):
        m, mp_, pl, dim, start, goal = F.build(name, cm, cp)
        sides.append([m, mp_, pl, dim])
    f = F.FLOWS[name]
    pos3 = np.r_[start, 0.0]
    if f.get("pot"):
        for sd in sides:
            sd[2].update_potential_map(pos3)
    s = F.waypoints(start, f["control"], f.get("start_yaw", 0.0))
    g = F.waypoints(goal, f["control"], 0.0)
    m, dim = sides[0][0], sides[0][3]
    grid = m.data.reshape(-1).copy()
    blocked = []
    snaps = [[], []]
    for k, sd in enumerate(sides):
        snaps[k].append(lpa_flow.snapshot(sd[2], sd[2].lpa_plan(s, g)))
    for step in range(steps):
        op = rng.choice(["block", "clear", "restamp", "root"] if f.get("pot") else ["block", "clear", "root"], p=None)
        res = snaps[0][-1]["res"]
        if res is None or int(res["status"]) != 0:
            op = "clear" if blocked else "block"
        path = sides[0][2].lpa_best_child_states()[:, :3]
        if op == "block" and len(path):
            k = int(rng.integers(0, len(path)))
            cand = lpa_flow.cells_on_path(m, dim, path[k:k + 1], int(rng.integers(0, 3)))
            lin = cand[:, 0] + m.dim[0] * cand[:, 1]
            cells = cand[(grid[lin] >= 0) & (grid[lin] < 100)]
            grid[cells[:, 0] + m.dim[0] * cells[:, 1]] = 100
            blocked.extend(cells.tolist())
            for i, sd in enumerate(sides):
                sd[2].lpa_get_linked_nodes()
                sd[1].set_cells(cells, 100)
                sd[2].lpa_update_blocked_nodes(cells)
        elif op == "clear" and blocked:
            idx = rng.permutation(len(blocked))[: max(1, len(blocked) // 2)]
            cells = np.array([blocked[i] for i in idx], dtype=np.int32)
            blocked = [b for i, b in enumerate(blocked) if i not in set(idx.tolist())]
            grid[cells[:, 0] + m.dim[0] * cells[:, 1]] = 0
            for sd in sides:
                sd[2].lpa_get_linked_nodes()
                sd[1].set_cells(cells, 0)
                sd[2].lpa_update_cleared_nodes(cells)
        elif op == "restamp" and len(path):  # a local re-stamp (a whole-map one turns every cell with potential into an obstacle)
            pt = np.zeros(3)
            pt[:dim] = path[int(rng.integers(0, len(path)))][:dim]
            for sd in sides:
                sd[2].set_vec("potential_map_range", np.full(dim, 1.5))
                sd[2].update_potential_map(pt)
        elif op == "root" and len(path) >= 3:
            nxt = sides[0][2].lpa_waypoint(1)
            for sd in sides:
                sd[2].lpa_get_sub_state_space(1)
            s = nxt
        for k, sd in enumerate(sides):
            snaps[k].append(lpa_flow.snapshot(sd[2], sd[2].lpa_plan(s, g)))
        lpa_flow.assert_same(snaps[0][-2:], snaps[1][-2:], "%s seed %d step %d (%s)" % (name, seed, step, op))
