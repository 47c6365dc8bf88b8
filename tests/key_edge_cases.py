"""Planning problems at the edges of the search kernel's configuration (build_cfg, mplb.cu): wide lattice keys, the exact
collision-sampling path and starts / goals outside the packable key range.

`key_layout` and `sampler` restate build_cfg's key packing and its `use_fast` rule; they only *choose* the cases here.
The GPU test (test_gpu_key_edges.py) asserts that they agree with what the library reports (mplb_planner_key_layout), so
a case meant to cover a branch is known to have taken it.

Every problem is small enough for the oracle to answer in well under a second."""
import math

import numpy as np

import oracle
import mpl_ros_b200 as mp
from mpl_ros_b200 import maps
from fuzz_cases import Case, ORDER_OF_CONTROL
from test_gpu_filters import filter_bounds

NCAP, TT_CAP = 64, 1024  # MPLB_NCAP, MPLB_TT_CAP (mplb_search.cuh)


def _bits_for(n):
    b = 1
    while (1 << b) < n:
        b += 1
    return b


def _bounds(prm):
    return [0.0, prm.get("v_max", -1.0), prm.get("a_max", -1.0), prm.get("j_max", -1.0)]


def key_layout(dim, order, m, prm, U, shaped, use_yaw):
    """build_cfg's lattice-key packing: (fields, key_bits); fields[f] = (lo, bits, shift, word) for f = axis * order + d,
    then the yaw field of shaped plans."""
    umax = float(np.abs(U[:, :dim]).max())
    margin = max(2.0, 2.0 * (prm["v_max"] if order >= 2 else umax) * prm["dt"])
    bounds, fields, bitpos = _bounds(prm), [], 0

    def place(lo, bits):
        nonlocal bitpos
        if bitpos % 64 + bits > 64:
            bitpos = (bitpos // 64 + 1) * 64
        fields.append((lo, bits, bitpos % 64, bitpos // 64))
        bitpos += bits

    for ax in range(dim):
        for d in range(order):
            if d == 0:
                lo = math.floor((m.origin[ax] - margin) / 0.01) - 2
                hi = math.ceil((m.origin[ax] + int(m.dim[ax]) * m.res + margin) / 0.01) + 2
            else:
                hi = math.ceil((bounds[d] if bounds[d] > 0 else 100.0) / 0.1) + 2
                lo = -hi
            place(lo, _bits_for(hi - lo + 1))
    if shaped:
        place(-256 if use_yaw else 0, 9 if use_yaw else 1)
    return fields, bitpos


def pack(fields, ints):
    """(k0, k1) of a lattice tuple, or None outside the packable range (pack_key_nohash)."""
    k = [0, 0]
    for (lo, bits, shift, word), v in zip(fields, ints):
        if not 0 <= v - lo < (1 << bits):
            return None
        k[word] |= (v - lo) << shift
    return k[0], k[1]


def packable_end(fields, f):
    """Largest lattice int field f packs (its lower end + 2^bits - 1)."""
    return fields[f][0] + (1 << fields[f][1]) - 1


def sampler(dim, order, m, prm, U):
    """build_cfg's sample-time tables and filtered-sampler switch: dict(use_fast, known, n_hi, tt_total, delta)."""
    umax = float(np.abs(U[:, :dim]).max())
    vmax_eff = prm["v_max"] if order >= 2 else umax
    dt = prm["dt"]
    n_hi = max(5, math.ceil(vmax_eff * dt / m.res)) + 1
    tt = 0
    for n in range(5, n_hi + 1):
        t, dts = 0.0, dt / n
        while t < dt:
            tt += 1
            t += dts
    b = _bounds(prm)
    known = all(b[d] > 0 for d in range(1, order))
    _, delta = filter_bounds(order, m.dim, m.res, m.origin, U[:, :dim], dt, *b[1:])
    return dict(use_fast=int(known and n_hi < NCAP and tt <= TT_CAP and delta <= 1e-6), known=known, n_hi=n_hi, tt_total=tt,
                delta=delta)


def box_map(dim, nd, res, seed, origin=None, nbox=8):
    """Random axis-aligned boxes of occupied cells on a free map."""
    rng = np.random.default_rng(seed)
    nd = np.array(nd)
    g = np.zeros(tuple(nd[::-1]), np.int8)
    for _ in range(nbox):
        lo = [int(rng.integers(0, n)) for n in nd]
        sz = [int(rng.integers(1, max(2, n // 5))) for n in nd]
        g[tuple(slice(lo[k], lo[k] + sz[k]) for k in range(dim))[::-1]] = 100
    return maps.GridMap(np.zeros(dim) if origin is None else np.asarray(origin, np.float64), nd, res, g.reshape(-1))


def yaw_controls(dim, u, uy):
    """test_planner_2d_with_yaw.cpp:49-57 (27 rows), and a 3D form with a z rate (27 rows, yaw rate by the x rate)."""
    if dim == 2:
        return np.array([[dx, dy, dyaw] for dx in (-u, 0.0, u) for dy in (-u, 0.0, u) for dyaw in (-uy, 0.0, uy)])
    return np.array([[dx, dy, dz, math.copysign(uy, dx) if dx else 0.0]
                     for dx in (-u, 0.0, u) for dy in (-u, 0.0, u) for dz in (-u, 0.0, u)])


def controls(dim, order, maxu, u):
    """|U| <= 32 (9 or 27 rows) or > 32 (49 or 63 rows) plain control sets."""
    if maxu == 1:
        return maps.make_U(u, 1, dim)
    if dim == 2:
        return maps.make_U(u, 3, 2)
    return maps.make_U(u, 2, 3)[::2]  # 63 rows


def make(m, dim, control, U, prm, seed=0, n_batch=24, max_seg=6, near_goals=False):
    """A Case (fuzz_cases) on map m with start / goal from maps.sample_queries; near_goals: the batch's goals lie 0.7 m
    from their starts along x."""
    extent = float(np.max(m.dim)) * m.res  # the single query's goal lies outside the start's goal region
    S, G = maps.sample_queries(m, 1, seed=seed, min_dist=min(1.2 * prm.get("tol_pos", 0.5), 0.5 * extent))
    return Case(seed=seed, map=m, dim=dim, control=control, U=U, params=dict(prm), start=S[0], goal=G[0], vel=np.zeros(dim),
                yaw=0.0, pot=None, region=None, max_seg=max_seg, n_batch=n_batch, near_goals=near_goals)


def order_of(control):
    return ORDER_OF_CONTROL[control & 15]


def state_waypoints(c, pos, vel=None, acc=None, jrk=None, yaw=None):
    """(GPU, oracle) waypoint arrays at pos [n, dim] with optional derivative rows and yaws, control of the case."""
    pos = np.atleast_2d(pos)
    a, b = mp.waypoints_array(len(pos)), oracle.make_waypoints(len(pos))
    for w in (a, b):
        w["pos"][:, :c.dim] = pos
        for name, v in (("vel", vel), ("acc", acc), ("jrk", jrk)):
            if v is not None:
                w[name][:, :c.dim] = v
        if yaw is not None:
            w["yaw"] = yaw
        w["control"] = c.control
    return a, b


# ---- the out-of-range start and goal values (per field kind), inside the packable range first
YAWS_INSIDE = (25.5, -25.5)             # round(yaw / 0.1) + 256 in [0, 512)
YAWS_OUTSIDE = (25.7, -25.7, 30.0, -40.0, 1000.0)


def derivative_values(fields, f, bound):
    """(inside, outside) values of derivative field f: the bound plus 0.24 / 0.26 / 1, the packable end, one step past it."""
    end = packable_end(fields, f) * 0.1
    vals = [bound + 0.24, bound + 0.26, bound + 1.0, end, end + 0.1, -(end + 0.1) - 0.2]
    ins = [v for v in vals if pack_one(fields, f, v)]
    outs = [v for v in vals if not pack_one(fields, f, v)]
    return ins, outs


def pack_one(fields, f, x):
    lo, bits = fields[f][:2]
    return 0 <= round_haz(x / 0.1) - lo < (1 << bits)


def round_haz(x):
    """std::round: halfway cases away from zero."""
    r = math.trunc(x)
    if abs(x - r) >= 0.5:
        r += math.copysign(1.0, x)
    return int(r)


# ---- the catalogue: (name, branch, Case, singles, batch)
# singles: list of (start fields, goal fields) dicts for state_waypoints; batch: (start fields, goal fields) lists that are
# dealt round-robin to every other start / every third goal of a batch of in-range queries (None: plain queries only).
PRM = dict(tol_pos=0.5)


def wide_cases():
    """Keys of more than 96 bits on 3D SNP, plain (both |U| classes) and shaped with yaw; and the 96-bit boundary.  At
    dt = 0.25 and j_max = 7, controls that differ in z often lead to nodes that differ only in their z jerk, the field
    packed above bit 96.  The single plans run out of pops (many nodes); the batches' goals lie 0.7 m from their starts
    and the search is greedy (epsilon 20, 100 with 63 controls), so that they find paths."""
    out = []
    prm = dict(PRM, v_max=3.0, a_max=3.0, j_max=7.0, dt=0.25, max_num=400, epsilon=20.0)
    for maxu in (1, 4):
        c = make(box_map(3, [120, 120, 40], 0.1, 1), 3, mp.SNP, controls(3, 4, maxu, 2.0),
                 dict(prm, epsilon=20.0 if maxu == 1 else 100.0), seed=1, near_goals=True)
        out.append(("3D SNP 12x12x4 m", "wide", c, [({}, {})], None))
    c = make(box_map(3, [75, 75, 30], 0.1, 2), 3, mp.SNPxYAW, yaw_controls(3, 2.0, 0.5),
             dict(prm, yaw_max=-1.0, wyaw=1.0), seed=2, near_goals=True)
    out.append(("3D SNPxYAW 7.5x7.5x3 m", "wide", c, [({"yaw": 0.4}, {})], None))
    for nx in (60, 100):  # 96 bits (word 1 still fits the table slot), then more
        c = make(box_map(3, [nx, 60, 30], 0.1, 3), 3, mp.SNP, controls(3, 4, 1, 2.0), prm, seed=3, near_goals=True)
        out.append(("3D SNP %gx6x3 m" % (nx * 0.1), "wide" if nx != 60 else "96 bits", c, [({}, {})], None))
    return out


def exact_cases():
    """use_fast == 0 on every plain instantiation: the table-size trigger (res 0.045, v dt = 2: 1092 sample times; res
    0.05 just inside with 870), the bound trigger on JRK / SNP, the guard-band trigger alone (origin 1.5e7 at res 0.01;
    1e7 just inside), 200 samples per primitive, and the largest sample divisor the host accepts (4096)."""
    out = []
    ctl = {1: mp.VEL, 2: mp.ACC, 3: mp.JRK, 4: mp.SNP}
    for dim in (2, 3):
        for order in (1, 2, 3, 4):
            for maxu in (1, 4):
                U = controls(dim, order, maxu, 2.0 if order == 1 else 1.0)
                prm = dict(PRM, v_max=2.0, a_max=2.0, j_max=2.0, dt=1.0, max_num=120)
                for res, branch in ((0.045, "exact: table"), (0.05, "fast: table inside")):
                    nd = [int(4.0 / res)] * 2 if dim == 2 else [int(3.0 / res), int(3.0 / res), int(1.2 / res)]
                    c = make(box_map(dim, nd, res, 10 + order), dim, ctl[order], U, prm, seed=order, n_batch=16)
                    out.append(("table res %g" % res, branch, c, [({}, {})], None))
                if order >= 3:
                    drop = ("a_max",) if order == 3 else (("j_max",) if maxu == 4 else ("a_max", "j_max"))
                    p = {k: v for k, v in prm.items() if k not in drop}
                    nd = [40, 40] if dim == 2 else [24, 24, 10]
                    c = make(box_map(dim, nd, 0.1, 20 + order), dim, ctl[order], U, p, seed=order, n_batch=16)
                    out.append(("unset " + "/".join(drop), "exact: bound", c, [({}, {})], None))
    for dim in (2, 3):
        nd = [150, 150] if dim == 2 else [60, 60, 24]
        prm = dict(PRM, v_max=0.3, a_max=0.5, dt=1.0, max_num=120, tol_pos=0.2)
        for org, branch in ((1.5e7, "exact: guard band"), (1.0e7, "fast: guard band inside")):
            c = make(box_map(dim, nd, 0.01, 30 + dim, origin=[org] * dim), dim, mp.ACC, maps.make_U(0.25, 1, dim), prm,
                     seed=dim, n_batch=16)
            out.append(("origin %g res 0.01" % org, branch, c, [({}, {})], None))
    c = make(box_map(2, [200, 200], 0.02, 40), 2, mp.VEL, maps.make_U(2.0, 1, 2), dict(PRM, v_max=2.0, dt=2.0, max_num=60),
             seed=4, n_batch=16)
    out.append(("200 samples per primitive", "exact: table", c, [({}, {})], None))
    c = make(box_map(2, [40, 40], 0.25, 41), 2, mp.VEL, maps.make_U(1023.75, 1, 2), dict(PRM, v_max=2.0, dt=1.0, max_num=3),
             seed=5, n_batch=16)
    out.append(("4096 sample divisors", "exact: table", c, [({}, {})], None))
    return out


def too_many_samples_case():
    """v dt / res one step past the last accepted value: n_hi = 4097 is rejected."""
    return make(box_map(2, [40, 40], 0.25, 41), 2, mp.VEL, maps.make_U(1024.0, 1, 2), dict(PRM, v_max=2.0, dt=1.0, max_num=3),
                seed=5)


def shaped_exact_case():
    """A yaw plan whose sample tables do not fit the fast path: the shaped kernels have no exact path."""
    return make(box_map(2, [90, 90], 0.045, 42), 2, mp.ACCxYAW, yaw_controls(2, 1.0, 0.5),
                dict(PRM, v_max=2.0, a_max=2.0, dt=1.0, max_num=50, yaw_max=1.3), seed=6)


def oor_cases():
    """Starts and goals outside the packable key range (and just inside it): yaw, velocity, acceleration and jerk, 2D and
    3D, plain and shaped."""
    out = []
    yaw_singles = [({"yaw": y}, {}) for y in YAWS_INSIDE + YAWS_OUTSIDE] + [({"yaw": 1000.0}, {"yaw": 30.0}),
                                                                            ({"yaw": 0.3}, {"yaw": -40.0})]
    yaw_batch = ([{"yaw": y} for y in YAWS_OUTSIDE + YAWS_INSIDE], [{"yaw": 30.0}, {"yaw": -25.7}])
    prm = dict(PRM, v_max=2.0, a_max=1.0, dt=1.0, max_num=300, yaw_max=1.3, wyaw=1.0)
    for dim, ctl, nd in ((2, mp.ACCxYAW, [40, 40]), (3, mp.ACCxYAW, [24, 24, 10]), (2, mp.VELxYAW, [40, 40])):
        c = make(box_map(dim, nd, 0.1, 50 + dim), dim, ctl, yaw_controls(dim, 1.0, 0.5), prm, seed=dim)
        out.append(("start / goal yaw", "out-of-range yaw", c, yaw_singles, yaw_batch))
    specs = [(2, mp.ACC, 1, "vel", "v_max", [40, 40]), (3, mp.ACC, 4, "vel", "v_max", [24, 24, 10]),
             (2, mp.JRK, 1, "acc", "a_max", [40, 40]), (3, mp.JRK, 1, "acc", "a_max", [24, 24, 10]),
             (2, mp.SNP, 4, "jrk", "j_max", [40, 40]), (3, mp.SNP, 1, "jrk", "j_max", [24, 24, 10]),
             (2, mp.ACCxYAW, 1, "vel", "v_max", [40, 40])]
    prm = dict(PRM, v_max=2.0, a_max=1.0, j_max=1.5, dt=1.0, max_num=300)
    for dim, ctl, maxu, kind, bname, nd in specs:
        order = order_of(ctl)
        U = yaw_controls(dim, 1.0, 0.5) if ctl & 16 else controls(dim, order, maxu, 1.0)
        p = dict(prm, yaw_max=-1.0) if ctl & 16 else prm
        c = make(box_map(dim, nd, 0.1, 60 + order), dim, ctl, U, p, seed=order + dim)
        fields, _ = key_layout(dim, order, c.map, p, U, bool(ctl & 16), bool(ctl & 16))
        d = {"vel": 1, "acc": 2, "jrk": 3}[kind]
        ins, outs = derivative_values(fields, d, p[bname])  # field of axis 0, derivative d
        vec = lambda x: np.eye(dim)[0] * x  # noqa: E731
        singles = [({kind: vec(x)}, {}) for x in ins + outs] + [({}, {kind: vec(outs[0])}), ({kind: vec(outs[-1])}, {kind: vec(outs[0])})]
        batch = ([{kind: vec(x)} for x in outs + ins], [{kind: vec(x)} for x in outs])
        out.append(("start / goal %s" % kind, "out-of-range " + kind, c, singles, batch))
    return out
