"""Seeded random planning problems steered to one instantiation of the search kernel, and the one place that says which
instantiation a problem launches.

mplb.cu's DISPATCH selects astar_batch_kernel<DIM, ORD, MAXU, POT> from the dimension, the control order (control & 15),
the control-set size (MAXU = 1 for |U| <= 32, else 4) and whether the plan is shaped (a potential map, a search region or
yaw controls; shaped plans need |U| <= 32, so there is no shaped MAXU = 4 kernel): 16 plain and 8 shaped cells.
`make_case(cell, seed)` draws a box map, planner settings and a query for one cell, reusing rand_case of
test_oracle_fuzz_vs_reference.py for the map and the parameters, and then varies what rand_case keeps fixed: the
control-set size class, epsilon in {0, 1, 2, 3.5}, tol_acc, VEL with v_max below the control bound (the predecessor-log
mode), non-dyadic resolutions, map origins of 1e5 .. 5e6 m, and the cost-shaping inputs."""
import numpy as np

import oracle
import mpl_ros_b200 as mp
from mpl_ros_b200 import maps
from helpers_gpu import make_pair
from test_oracle_fuzz_vs_reference import rand_case

CONTROL_OF_ORDER = {1: mp.VEL, 2: mp.ACC, 3: mp.JRK, 4: mp.SNP}
ORDER_OF_CONTROL = {mp.VEL: 1, mp.ACC: 2, mp.JRK: 3, mp.SNP: 4}
ORDER_NAME = {1: "VEL", 2: "ACC", 3: "JRK", 4: "SNP"}

CELLS = ([(dim, order, maxu, False) for dim in (2, 3) for order in (1, 2, 3, 4) for maxu in (1, 4)] +
         [(dim, order, 1, True) for dim in (2, 3) for order in (1, 2, 3, 4)])


def instantiation(dim, control, n_controls, shaped):
    """(DIM, ORD, MAXU, POT) of the astar_batch_kernel that mplb.cu's DISPATCH / launch_any run for this plan."""
    return dim, ORDER_OF_CONTROL[control & 15], (1 if n_controls <= 32 else 4), bool(shaped)


def cell_name(cell):
    dim, order, maxu, shaped = cell
    return "%dD-%s-U%s%s" % (dim, ORDER_NAME[order], "le32" if maxu == 1 else "gt32", "-shaped" if shaped else "")


class Case:
    """One problem: map, planner parameters, controls, a single query, and the cost-shaping inputs (None when absent)."""

    def __init__(self, **kw):
        self.__dict__.update(kw)

    @property
    def cell(self):
        return instantiation(self.dim, self.control, len(self.U), self.shaped)

    @property
    def shaped(self):
        return self.pot is not None or self.region is not None or bool(self.control & 16)

    def build(self):
        """(GPU planner, oracle planner) with the map, parameters, controls and shaping of this case applied to both."""
        pl, op = make_pair(self.map, self.dim, self.params, self.U)
        if self.pot is not None:
            pl.setPotentialWeight(self.pot["weight"])
            pl.setGradientWeight(self.pot["gradient"])
            pl.setPotentialRadius(self.pot["radius"])
            pl.setPotentialMapRange(self.pot["range"])
            pl.updatePotentialMap(self.start)
        if self.region is not None:
            pl.setSearchRadius(self.region["radius"])
            pl.setSearchRegion(self.region["path"][:, :self.dim], dense=self.region["dense"])
        self._shape_oracle(op)
        return pl, op

    def build_oracle(self):
        """The oracle planner alone (CPU), configured like the oracle half of build()."""
        om = oracle.OracleMap(self.map.origin, self.map.dim, self.map.data, self.map.res)
        om.free_unknown()
        op = oracle.OraclePlanner(self.dim)
        op.set_map(om)
        for k, v in self.params.items():
            op.set_param(k, v)
        op.set_controls(self.U)
        self._shape_oracle(op)
        return op

    def _shape_oracle(self, op):
        if self.control & 16:
            op.set_param("trig_mode", 1)  # the product's correctly rounded cos/sin (test_gpu_yaw.py)
        if self.pot is not None:
            op.set_param("potential_weight", self.pot["weight"])
            op.set_param("gradient_weight", self.pot["gradient"])
            op.set_vec("potential_radius", self.pot["radius"])
            op.set_vec("potential_map_range", self.pot["range"])
            op.update_potential_map(_vec3(self.start))
        if self.region is not None:
            op.set_vec("search_radius", self.region["radius"])
            op.set_search_region(self.region["path"], dense=self.region["dense"])

    def batch_waypoints(self, seed):
        """(GPU starts, GPU goals, oracle starts, oracle goals) of n_batch queries, with random start yaws for yaw controls."""
        S, G = self.queries(self.n_batch, seed)
        yaws = np.random.default_rng(seed).uniform(-3, 3, size=len(S)) if self.control & 16 else None
        sg, so = self.waypoints(S, yaw=yaws)
        gg, go = self.waypoints(G)
        return sg, gg, so, go

    def waypoints(self, pos, vel=None, yaw=None):
        """(GPU, oracle) waypoint arrays at `pos` [n, dim] with this case's control."""
        pos = np.atleast_2d(pos)
        a, b = mp.waypoints_array(len(pos)), oracle.make_waypoints(len(pos))
        for w in (a, b):
            w["pos"][:, :self.dim] = pos
            if vel is not None:
                w["vel"][:, :self.dim] = vel
            if yaw is not None:
                w["yaw"] = yaw
            w["control"] = self.control
        return a, b

    def queries(self, n, seed):
        """n (start, goal) pairs on free cell centres at least a few cells apart (maps.sample_queries)."""
        extent = float(np.min(self.map.dim)) * self.map.res
        return maps.sample_queries(self.map, n, seed=seed, min_dist=min(4 * self.map.res, 0.25 * extent))


def _vec3(v):
    out = np.zeros(3)
    out[:len(v)] = v
    return out


def _controls(rng, dim, maxu, yaw, u):
    if yaw:  # Dim + 1 columns; <= 27 rows
        uy = float(rng.choice([0.4, 0.5, 1.0]))
        if dim == 2:  # test_planner_2d_with_yaw.cpp:49-57
            return np.array([[dx, dy, dyaw] for dx in (-u, 0.0, u) for dy in (-u, 0.0, u) for dyaw in (-uy, 0.0, uy)])
        return np.array([[dx, dy, dz, float(rng.choice([-uy, 0.0, uy]))]
                         for dx in (-u, 0.0, u) for dy in (-u, 0.0, u) for dz in (-u, 0.0, u)])
    if maxu == 1:
        return maps.make_U(u, int(rng.choice([1, 2])) if dim == 2 else 1, dim)  # 9 or 25 / 27 rows
    if dim == 2:
        return maps.make_U(u, int(rng.choice([3, 4])), 2)  # 49 or 81 rows
    U = maps.make_U(u, 2, 3)  # 125 rows, of which 33 .. 64
    return U[rng.choice(len(U), int(rng.integers(33, 65)), replace=False)]


def make_case(cell, seed):
    dim, order, maxu, shaped = cell
    rng = np.random.default_rng([seed, dim, order, maxu, int(shaped)])
    nd, origin, res, data, _, _, prm, start, goal, _ = rand_case(rng, dim)
    cs, cg = np.rint((start - origin) / res - 0.5), np.rint((goal - origin) / res - 0.5)  # the query's cells
    frame = rng.random()
    if frame < 0.25:  # resolutions that are not binary fractions
        res = float(rng.choice([0.15, 0.3, float(np.float32(0.1))]))
    elif frame < 0.45:  # map frames far from the origin (UTM-like); keys round(pos / 0.01) stay inside int32
        origin = (rng.uniform(1e5, 5e6, size=dim) + rng.uniform(0, 1, size=dim)).round(3)
    start, goal = (cs + 0.5) * res + origin, (cg + 0.5) * res + origin
    m = maps.GridMap(origin, nd, res, data)

    kinds = dict(pot=False, region=False, yaw=False)
    while shaped and not any(kinds.values()):
        kinds = dict(pot=rng.random() < 0.5, region=rng.random() < 0.5, yaw=rng.random() < 0.5)
    control = CONTROL_OF_ORDER[order] | (16 if kinds["yaw"] else 0)
    u = float(rng.choice([0.5, 1.0]))
    U = _controls(rng, dim, maxu, kinds["yaw"], u)

    params = {k: prm[k] for k in ("v_max", "a_max", "j_max", "dt", "w", "max_num", "tol_pos")}
    params["epsilon"] = float(rng.choice([0.0, 1.0, 1.0, 2.0, 3.5]))
    if order >= 2 and rng.random() < 0.3:
        params["tol_vel"] = float(rng.choice([0.0, 0.5, 1.0]))
    if order >= 3 and rng.random() < 0.2:
        params["tol_acc"] = float(rng.choice([0.5, 1.0]))
    if order == 1 and rng.random() < 0.35:  # v_max below the control bound: the kernel keeps predecessor records
        params["v_max"] = 0.75 * float(np.abs(U[:, :dim]).max())
    if kinds["yaw"]:
        params["yaw_max"] = float(rng.choice([-1.0, 0.7, 1.3]))
        params["wyaw"] = float(rng.choice([0.0, 1.0, 2.5]))
    vel = rng.choice([0.0, 0.5, -0.5], size=dim) if (order >= 2 and rng.random() < 0.4) else np.zeros(dim)
    yaw = float(rng.uniform(-3, 3)) if kinds["yaw"] else 0.0

    pot = region = None
    if kinds["pot"]:
        radius = np.zeros(3)
        radius[:dim] = rng.choice([0.3, 0.6, 1.0])
        if dim == 3:
            radius[2] = rng.choice([0.2, 0.5])
        rngv = np.zeros(3)  # zero: the whole map
        if rng.random() < 0.5:
            rngv[:dim] = rng.choice([1.0, 2.0, 3.0], size=dim)
        pot = dict(weight=float(rng.choice([0.1, 0.5])), gradient=float(rng.choice([0.0, 0.3])), radius=radius, range=rngv)
    if kinds["region"]:
        npts = int(rng.integers(2, 6))
        path = np.zeros((npts, 3))
        path[0, :dim], path[-1, :dim] = start, goal
        for i in range(1, npts - 1):
            path[i, :dim] = origin + rng.random(dim) * nd * res
        radius = np.zeros(3)
        radius[:dim] = rng.choice([0.3, 0.8, 1.5])
        region = dict(radius=radius, path=path, dense=bool(rng.random() < 0.3))
    return Case(seed=seed, map=m, dim=dim, control=control, U=U, params=params, start=start, goal=goal, vel=vel, yaw=yaw,
                pot=pot, region=region, max_seg=int(rng.choice([3, 5, 8])), n_batch=int(rng.integers(16, 65)))
