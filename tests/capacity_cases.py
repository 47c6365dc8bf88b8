"""Planning problems that reach the search kernel's capacity edges (tests/test_gpu_capacity.py), built so that the oracle
alone can say which edge each one reaches (oracle.OraclePlanner.peaks / heap).

The maps are rows of square free rooms walled off from each other: a query whose goal lies in another room exhausts its
own room (MPLB_PLAN_QUEUE_EMPTY) after a number of nodes fixed by the room's size, a query whose goal is a cell away ends
after a few pops.  With VEL controls of step 0.5 m, dt = 1 and res = 0.5 the lattice positions are exactly the cell
centres, so a 2D room of side L holds L^2 nodes: L = 180 fits a 32768-node arena tier (32400 + |U| <= 32768), L = 181
does not (32761 + |U| > 32768)."""
import numpy as np

import oracle
import mpl_ros_b200 as mp
from mpl_ros_b200 import maps
from helpers_gpu import make_pair

ORDER_CONTROL = {1: mp.VEL, 2: mp.ACC, 3: mp.JRK, 4: mp.SNP}
NOMEM = 8  # MPLB_PLAN_NOMEM
TIER0 = 32768  # first arena tier without a MaxExpandStep bound (mplb.cu run_batch_begin)


def rooms_2d(sizes, res=0.5):
    """(map, rooms): one row of square rooms of the given interior sides (cells), one-cell walls around each"""
    H = max(sizes) + 2
    W = sum(s + 1 for s in sizes) + 1
    g = np.full((H, W), 100, np.int8)
    rooms, x = [], 1
    for s in sizes:
        g[1:1 + s, x:x + s] = 0
        rooms.append((x, 1, s))
        x += s + 1
    return maps.GridMap([0.0, 0.0], [W, H], res, g.reshape(-1)), rooms


def box_3d(L, res=0.5):
    """(map, rooms): a free cube of side L cells and, behind a wall, a free column (the unreachable goal's room)"""
    n = L + 2
    g = np.full((n, n, n + 4), 100, np.int8)  # [z][y][x]
    g[1:1 + L, 1:1 + L, 1:1 + L] = 0
    g[1:1 + L, 1:1 + L, n + 2] = 0
    return maps.GridMap([0.0, 0.0, 0.0], [n + 4, n, n], res, g.reshape(-1)), [(1, 1, 1, L), (n + 2, 1, 1, 1)]


def centre(m, room, d=0):
    """centre cell of a room (shifted by d cells along x)"""
    if len(room) == 3:
        x, y, s = room
        return m.int_to_float([x + s // 2 + d, y + s // 2])
    x, y, z, s = room
    return m.int_to_float([x + s // 2 + d, y + s // 2, z + s // 2])


class Problem:
    """One planner configuration on both sides (GPU planner, oracle planner) plus a cache of single oracle plans."""

    def __init__(self, m, dim, params, U, control, shaped=False, exact_preds=None):
        self.m, self.dim, self.params, self.U, self.control, self.shaped = m, dim, params, U, control, shaped
        self.exact_preds = exact_preds
        self.nU = len(U)
        self._cache = {}
        self.pl = self.op = None

    def oracle(self):
        if self.op is None:
            om = oracle.OracleMap(self.m.origin, self.m.dim, self.m.data, self.m.res)
            om.free_unknown()
            op = oracle.OraclePlanner(self.dim)
            op.set_map(om)
            for k, v in self.params.items():
                op.set_param(k, v)
            op.set_controls(self.U)
            if self.shaped:
                op.set_search_region_mask(np.ones(self.m.data.size, np.uint8))
                op.set_potential_map(self.potential())
            op._keep = om
            self.op = op
        return self.op

    def gpu(self):
        if self.pl is None:
            pl, _ = make_pair(self.m, self.dim, self.params, self.U)
            if self.shaped:  # a search region over the whole map and a potential map: the POT instantiation
                pl.setSearchRegionMask(np.ones(self.m.data.size, np.uint8))
                pl.setPotentialMap(self.potential())
            if self.exact_preds is not None:
                pl.setExactPreds(self.exact_preds)
            self.pl = pl
        return self.pl

    def potential(self):
        """occupied cells 100 (the potential map is what the shaped kernels test for collisions, em:104-118), free cells
        a random cost in [0, 60)"""
        pot = np.random.default_rng(5).integers(0, 60, size=self.m.data.size).astype(np.int8)
        return np.where(self.m.data == 100, np.int8(100), pot)

    def waypoints(self, S, G):
        """(GPU starts, GPU goals, oracle starts, oracle goals)"""
        S, G = np.atleast_2d(S), np.atleast_2d(G)
        out = []
        for P in (S, G):
            a, b = mp.waypoints_array(len(P)), oracle.make_waypoints(len(P))
            for w in (a, b):
                w["pos"][:, :self.dim] = P
                w["control"] = self.control
            out.append((a, b))
        return out[0][0], out[1][0], out[0][1], out[1][1]

    def single(self, s, g, max_seg):
        """the oracle's plan of one query: (result, action row of max_seg entries, peaks, heap array), cached"""
        key = (tuple(np.ravel(s)), tuple(np.ravel(g)), max_seg)
        if key not in self._cache:
            op = self.oracle()
            _, _, so, go = self.waypoints(s, g)
            ro = op.plan(so, go)
            row = np.full(max(max_seg, 0), -1, np.int32)
            if ro["status"] == 0 and max_seg > 0:
                a = op.actions(int(ro["n_seg"]))[:max_seg]
                row[:len(a)] = a
            self._cache[key] = (ro.copy(), row, op.peaks(), op.heap())
        return self._cache[key]

    def overflows(self, peaks, cap, log_cap):
        """whether a plan with these oracle peaks outgrows a tier of capacity cap (mplb_search.cuh capacity check)"""
        return (peaks["nodes"] + self.nU > cap or peaks["heap"] + self.nU + 1 > cap or
                (log_cap > 0 and peaks["records"] + self.nU > log_cap))


def vel_rooms(sizes, nu_class=1, **kw):
    """2D VEL on a row of rooms: |U| = 25 (steps of 0.5 m in [-1, 1]) or, nu_class 4, |U| = 49 (in [-1.5, 1.5])"""
    m, rooms = rooms_2d(sizes)
    U = maps.make_U(1.0, 2, 2) if nu_class == 1 else maps.make_U(1.5, 3, 2)
    params = dict(v_max=float(np.abs(U).max()), dt=1.0, tol_pos=0.5)
    params.update(kw)
    return Problem(m, 2, params, U, mp.VEL), rooms


def room_queries(m, rooms, picks):
    """picks: list of (room index, kind) with kind 'exhaust' (goal in the next room) or 'near' (goal 2 cells away)"""
    S, G = [], []
    for r, kind in picks:
        S.append(centre(m, rooms[r]))
        G.append(centre(m, rooms[(r + 1) % len(rooms)]) if kind == "exhaust" else centre(m, rooms[r], 2))
    return np.array(S), np.array(G)


HEAP_MAX_NUM = {(2, 1): 5000, (2, 2): 200, (2, 3): 200, (2, 4): 200, (3, 1): 2500, (3, 2): 300, (3, 3): 300, (3, 4): 450}


def heap_cell(dim, order, shaped, eps, exhaust=False):
    """regime (a): |U| <= 32 on the (DIM, ORD) cell, plain or shaped: (problem, query).  The query's goal lies behind a
    wall, so the plan either stops at MaxExpandStep with a deep heap or (exhaust, VEL only) empties its room after a peak
    heap above 512."""
    ctl = ORDER_CONTROL[order]
    if dim == 2:
        m, rooms = rooms_2d([150, 12])
        U = maps.make_U(1.0, 2, 2)
    else:
        m, rooms = box_3d(30)
        U = maps.make_U(1.0, 1, 3)
    params = dict(v_max=2.0, a_max=1.0, j_max=1.0, dt=1.0, tol_pos=0.5, epsilon=eps)
    if order == 1:
        params["v_max"] = 1.0  # the control bound: no predecessor log
    if not exhaust:
        params["max_num"] = HEAP_MAX_NUM[(dim, order)]
    P = Problem(m, dim, params, U, ctl, shaped=shaped)
    return P, (centre(m, rooms[0]), centre(m, rooms[1]))


def near_queries(P, n, seed):
    """n queries whose goal is two cells from the start (few pops), on free cells of P's map"""
    S, _ = maps.sample_queries(P.m, n, seed=seed, min_dist=0.0)
    G = S.copy()
    G[:, 0] += 2 * P.m.res
    return S, G
