"""The search kernel's filtered collision sampler against exact arithmetic, and plans on maps far from the origin.

The reference's voxel of a collision sample is round((p(t) - origin)/res - 0.5) (map_util.h:103-108) with p(t) in
primitive.h's operation order (primitive.h:128-131).  The search kernel decides most samples with a filter
(filtered_w and clear_of_tie in mplb_search.cuh): w = (p(t) - origin)/res - 0.5 as one FP64 Horner chain in cells, "sure" when w lies
farther than the guard band fast_delta from a rounding tie, the exact formula otherwise.  mplb_probe_samples runs the
kernel's own filter code on arbitrary states; every row it returns is checked here against a float64 model of the
reference and against exact rational arithmetic, on map origins up to UTM scale (5e5 .. 1e7 m), where the reference's
own rounding of p = (... + v t) + p0 is larger than the filter's error.
"""
import math
from fractions import Fraction

import numpy as np
import pytest

import oracle
import mpl_ros_b200 as mp
from mpl_ros_b200 import maps
from helpers_gpu import assert_results_equal, make_pair, waypoint_pair

ORDER = {mp.VEL: 1, mp.ACC: 2, mp.JRK: 3, mp.SNP: 4}
RES = (0.05, float(np.float32(0.1)), 0.1, 0.15, 0.3)
ORIGINS = (0.0, -2.37, 1234.5, -4.1e5, 5e5, 5.3e6, "9.9e6 on one axis")
KMAX = 2 ** 31 - 1


# ---------------------------------------------------------------- exact arithmetic and the reference's float64 model
class Dy:
    """Exact dyadic rationals n / 2**s, elementwise over arrays (Python ints in object arrays).  Every float64 is one,
    and so is every sum and product of them: this is exact rational arithmetic like fractions.Fraction
    (test_dyadic_matches_fraction), fast enough to cover every row of a probe."""

    def __init__(self, n, s):
        self.n, self.s = n, s

    @staticmethod
    def of(x):
        x = np.asarray(x, dtype=np.float64).ravel()
        fr = [float(v).as_integer_ratio() for v in x]
        s = max([d.bit_length() - 1 for _, d in fr] + [0])
        return Dy(np.array([n << (s - d.bit_length() + 1) for n, d in fr], dtype=object), s)

    def _align(self, o):
        s = max(self.s, o.s)
        return self.n * (1 << (s - self.s)), o.n * (1 << (s - o.s)), s

    def __add__(self, o):
        a, b, s = self._align(o)
        return Dy(a + b, s)

    def __sub__(self, o):
        a, b, s = self._align(o)
        return Dy(a - b, s)

    def __mul__(self, o):
        if isinstance(o, int):
            return Dy(self.n * o, self.s)
        return Dy(self.n * o.n, self.s + o.s)

    __rmul__ = __mul__

    def abs(self):
        return Dy(np.abs(self.n), self.s)

    def __lt__(self, o):
        a, b, _ = self._align(o)
        return np.asarray(a < b, dtype=bool)

    def __le__(self, o):
        a, b, _ = self._align(o)
        return np.asarray(a <= b, dtype=bool)

    def fraction(self, i):
        return Fraction(int(self.n[i]), 1 << self.s)


def ref_p(ordr, p0, v, a, j, u, t):
    """Axis p(t) in primitive.h:128-131's order, in float64 (numpy: IEEE round-to-nearest per operation, no
    contraction).  c(0) is 0 for every control; adding the products of the structurally-zero coefficients adds exact
    zeros, which cannot change a non-zero sum, so they are left out.  power(t, k) multiplies left to right."""
    t3 = (t * t) * t
    if ordr == 1:
        s = u * t
    elif ordr == 2:
        s = (u / 2 * t) * t + v * t
    elif ordr == 3:
        s = (u / 6 * t3 + (a / 2 * t) * t) + v * t
    else:
        s = ((u / 24 * (t3 * t) + j / 6 * t3) + (a / 2 * t) * t) + v * t
    return s + p0


def round_haz(x):
    """std::round: half away from zero."""
    r = np.trunc(x)
    return r + np.where(np.abs(x - r) >= 0.5, np.copysign(1.0, x), 0.0)


def ref_cell(p, origin, res):
    """map_util.h:103-108: y = (p - origin)/res - 0.5 in float64, and round(y)."""
    y = (p - origin) / res - 0.5
    return y, round_haz(y).astype(np.int64)


def filter_bounds(ordr, nd, res, origin, U, dt, v_max, a_max, j_max):
    """The host's magnitude bound M and guard band of the filtered sampler (build_cfg, mplb.cu), in the same
    operation order: the filter's own error is < 2^-45 M, the band is 2^-40 M + 2^-50 P / res."""
    umax = float(np.abs(U).max())
    vmax_eff = v_max if ordr >= 2 else umax
    bnd = [0.0, v_max, a_max, j_max, 0.0]
    bnd[ordr] = umax
    dsum, tp, fact = 0.0, 1.0, 1.0
    for d in range(1, ordr + 1):
        tp *= dt
        fact *= d
        dsum += abs(bnd[d]) * tp / fact / res
    margin = max(2.0, 2.0 * vmax_eff * dt)
    M = max(float(n) for n in nd) + margin / res + dsum + 2.0
    P = max(abs(float(origin[i])) + int(nd[i]) * res + margin for i in range(len(nd)))
    return M, math.ldexp(M, -40) + math.ldexp(P / res, -50)


def check_probe(pl, sts, ordr, m, dt, bounds, ctx, tally):
    """Every row of one probe: the four properties of the module docstring.  Violations are counted in `tally`
    (per origin) and the first few are kept for the report; nothing here asserts, so one run shows them all."""
    rows, use_fast, delta = pl.probe_samples(sts)
    M, band = bounds
    dim = len(m.dim)
    t_ = tally.setdefault(ctx[0], dict(rows=0, unsure=0, sure_wrong=0, model=0, own=0, band=0, use_fast=0, delta=0, ex=[]))
    t_["rows"] += len(rows)
    t_["unsure"] += int((rows["sure"] == 0).sum())
    if use_fast != 1:
        t_["use_fast"] += 1
    if delta != band:
        t_["delta"] += 1
        t_["ex"].append((ctx, "fast_delta", delta, band))
    if len(rows) == 0:
        return 0
    sure = rows["sure"] != 0
    wrong = sure & np.any(rows["cell_fast"][:, :dim] != rows["cell_exact"][:, :dim], axis=1)
    t_["sure_wrong"] += int(wrong.sum())
    for i in np.flatnonzero(wrong)[:3]:
        t_["ex"].append((ctx, "sure but wrong", rows[i]))
    si, ui, t = rows["state"], rows["control"], rows["t"]
    U = pl.U_
    T = Dy.of(t)
    E24R = Dy.of(np.ldexp(M, -45)) * Dy.of(m.res) * 24
    R24 = Dy.of(m.res) * 24
    D = Dy.of(delta)
    half = Dy.of(0.5)
    weights = {1: 24, 2: 12, 3: 4, 4: 1}  # 24 / d!
    for ax in range(dim):
        o = float(m.origin[ax])
        p0, u = sts["pos"][si, ax], U[ui, ax]
        v, a, j = sts["vel"][si, ax], sts["acc"][si, ax], sts["jrk"][si, ax]
        y_ref, cell = ref_cell(ref_p(ordr, p0, v, a, j, u, t), o, m.res)
        bad = cell != rows["cell_exact"][:, ax]
        t_["model"] += int(bad.sum())
        for i in np.flatnonzero(bad)[:3]:
            t_["ex"].append((ctx, "exact cell != float64 model", ax, rows[i], cell[i]))
        # 24 res (y_true + 0.5) = 24 (p0 - o) + sum_d 24/d! coef_d t^d, exactly
        coefs = {1: v, 2: a, 3: j}
        acc = (Dy.of(p0) - Dy.of(o)) * 24
        tp = T
        for d in range(1, ordr + 1):
            acc = acc + Dy.of(u if d == ordr else coefs[d]) * tp * weights[d]
            tp = tp * T
        W = Dy.of(rows["w"][:, ax])
        own = ~((R24 * (W + half) - acc).abs() <= E24R)  # |w - y_true| <= 2^-45 M
        t_["own"] += int(own.sum())
        for i in np.flatnonzero(own)[:3]:
            t_["ex"].append((ctx, "filter error above 2^-45 M", ax, rows[i]))
        far = ~((W - Dy.of(y_ref)).abs() < D)  # |w - y_ref| < fast_delta
        t_["band"] += int(far.sum())
        for i in np.flatnonzero(far)[:3]:
            t_["ex"].append((ctx, "|w - y_ref| >= fast_delta", ax, rows[i], float((W - Dy.of(y_ref)).abs().fraction(i)), delta))
    return len(rows)


# ---------------------------------------------------------------- problem builders
def origin_of(name, dim):
    if name == "9.9e6 on one axis":
        return np.array([9.9e6, -2.37, 1234.5][:dim])
    return np.full(dim, float(name))


def box_map(dim, res, origin, seed):
    nd = [64, 64] if dim == 2 else [32, 32, 12]
    rs = np.random.RandomState(seed)
    g = np.zeros(tuple(nd[::-1]), dtype=np.int8)
    for _ in range(10 if dim == 2 else 14):
        sz = rs.randint(2, 9, size=dim)
        lo = [rs.randint(0, nd[k] - sz[k]) for k in range(dim)]
        sl = tuple(slice(lo[k], lo[k] + sz[k]) for k in range(dim))[::-1]
        g[sl] = 100
    return maps.GridMap(origin, nd, res, g.reshape(-1))


def salt_map(dim, res, origin, seed, frac=0.15):
    nd = [72, 72] if dim == 2 else [28, 28, 10]
    rs = np.random.RandomState(seed)
    data = np.where(rs.rand(int(np.prod(nd))) < frac, 100, 0).astype(np.int8)
    return maps.GridMap(origin, nd, res, data)


def controls_for(dim):
    U = maps.make_U(1.0, 1, dim)
    return U if dim == 2 else U[::4]  # 7 of the 27: every z value, and every x and y value


def params_for(ctrl, dt):
    p = dict(v_max=2.0, a_max=1.0, dt=dt, tol_pos=0.5, max_num=40)
    if ORDER[ctrl] == 4:
        p["j_max"] = 1.0
    return p


def states_of(nodes, ctrl, dim, sel):
    st = nodes["state"][sel]
    g, _ = waypoint_pair(st[:, 0:dim], ctrl, vel=st[:, 3:3 + dim], acc=st[:, 6:6 + dim])
    g["jrk"][:, :dim] = st[:, 9:9 + dim]
    return g


def adversarial_states(pl, base, ordr, m, rng):
    """Parent positions whose reference-order p(t) lands on a cell boundary at a sampled time of one control, on every
    axis at once, then stepped by -64 .. 64 ulps (np.nextafter): this fills the window between the guard band and the
    reference's own rounding error of p."""
    rows, _, _ = pl.probe_samples(base)
    rows = rows[rows["t"] > 0]
    if len(rows) == 0:
        return base[:0]
    r = rows[rng.randint(len(rows))]
    s0, u = base[int(r["state"])], pl.U_[int(r["control"])]
    dim = len(m.dim)
    p0 = np.zeros(dim)
    for ax in range(dim):
        s = ref_p(ordr, 0.0, s0["vel"][ax], s0["acc"][ax], s0["jrk"][ax], u[ax], float(r["t"]))
        o = float(m.origin[ax])
        k = round((s0["pos"][ax] + s - o) / m.res)
        p0[ax] = (o + k * m.res) - s
    steps = list(range(-64, 65))
    out = np.repeat(base[int(r["state"]):int(r["state"]) + 1], len(steps))
    for q, n in enumerate(steps):
        for ax in range(dim):
            x = p0[ax]
            for _ in range(abs(n)):
                x = np.nextafter(x, np.inf if n > 0 else -np.inf)
            out["pos"][q, ax] = x
    return out


# ---------------------------------------------------------------- 1. the probe matrix
def test_dyadic_matches_fraction():
    """The exact helper agrees with fractions.Fraction, and the float64 model reproduces a known hazard: at
    p0 = 500011.22, v = u = 1, t = 0.6 (ACC) the reference rounds p to exactly 500012.0, cell 120 of a map at
    origin 5e5 with res 0.1, although the real p(t) is below 500012 (cell 119)."""
    rs = np.random.RandomState(0)
    x = rs.standard_normal(50) * 10.0 ** rs.randint(-20, 20, size=50)
    y = rs.standard_normal(50) * 10.0 ** rs.randint(-20, 20, size=50)
    X, Y = Dy.of(x), Dy.of(y)
    e = (X * Y + X * 3 - Y).abs()
    for i in range(50):
        fx, fy = Fraction(x[i]), Fraction(y[i])
        assert e.fraction(i) == abs(fx * fy + 3 * fx - fy)
    assert list(X < Y) == [Fraction(a) < Fraction(b) for a, b in zip(x, y)]
    p = ref_p(2, np.array([500011.22]), np.array([1.0]), 0, 0, np.array([1.0]), np.array([0.6]))
    assert p[0] == 500012.0
    y_ref, cell = ref_cell(p, 5e5, 0.1)
    assert y_ref[0] == 119.5 and cell[0] == 120
    assert Fraction(500011.22) + Fraction(0.6) + Fraction(1, 2) * Fraction(0.6) ** 2 < 500012


@pytest.mark.gpu
def test_probe_filter_is_sound():
    """Every sample of every primitive that needs sampling, over dims 2/3 x VEL/ACC/JRK/SNP x res x origin x dt, from
    (a) node states of a short oracle plan on a random-box map and (b) adversarial states on cell boundaries:
      1. sure => the filtered cell is the exact cell;
      2. the exact cell is the float64 model of the reference (ref_p, ref_cell);
      3. exactly: |w - y_true| <= 2^-45 M (the filter's own error) and |w - y_ref| < fast_delta on every row;
      4. use_fast is on, fast_delta is the documented band, and fewer than 40 % of the samples are unsure.
    Most probe states are adversarial ones, so the unsure share here is far above the search's; the printed table shows
    it per origin (measured on an H100: 9 % at 5e5 .. 5.3e6, up to 30 % at origin 0 where lattice states put many
    samples exactly on voxel boundaries)."""
    rng = np.random.RandomState(7)
    tally, n_cfg = {}, 0
    for dim in (2, 3):
        U = controls_for(dim)
        for oname in ORIGINS:
            origin = origin_of(oname, dim)
            for ri, res in enumerate(RES):
                m = box_map(dim, res, origin, seed=ri)
                sc, gc = maps.sample_queries(m, 1, seed=ri, min_dist=1.0, max_dist=2.5)
                for ctrl in (mp.VEL, mp.ACC, mp.JRK, mp.SNP):
                    ordr = ORDER[ctrl]
                    for dt in (0.5, 1.0):
                        params = params_for(ctrl, dt)
                        pl, op = make_pair(m, dim, params, U)
                        _, so = waypoint_pair(sc, ctrl)
                        _, go = waypoint_pair(gc, ctrl)
                        ro = op.plan(so, go)
                        nodes = op.nodes(ro["n_nodes"])
                        sel = rng.choice(len(nodes), size=min(6, len(nodes)), replace=False)
                        real = states_of(nodes, ctrl, dim, sel)
                        adv = adversarial_states(pl, real[-1:], ordr, m, rng)
                        sts = np.concatenate([real, adv[::4], adv[60:69]])  # steps -64, -60, .., 64 and -4 .. 4
                        bounds = filter_bounds(ordr, m.dim, res, m.origin, U, dt, params["v_max"], params["a_max"],
                                               params.get("j_max", 0.0))
                        check_probe(pl, sts, ordr, m, dt, bounds, (oname, dim, ctrl, res, dt), tally)
                        n_cfg += 1
    print("\nfiltered sampler over %d configurations:" % n_cfg)
    for oname, t_ in tally.items():
        print("  origin %-18s rows %8d  unsure %5.1f %%  sure-but-wrong %d  model %d  own-bound %d  band %d  "
              "use_fast-off %d  delta %d" % (oname, t_["rows"], 100.0 * t_["unsure"] / max(t_["rows"], 1), t_["sure_wrong"],
                                             t_["model"], t_["own"], t_["band"], t_["use_fast"], t_["delta"]))
    ex = [e for t_ in tally.values() for e in t_["ex"]][:12]
    for k in ("sure_wrong", "model", "own", "band", "use_fast", "delta"):
        assert sum(t_[k] for t_ in tally.values()) == 0, (k, ex)
    for oname, t_ in tally.items():
        assert t_["rows"] > 10000, oname
        assert t_["unsure"] < 0.4 * t_["rows"], (oname, t_["unsure"], t_["rows"])


# ---------------------------------------------------------------- 2. whole plans on UTM-scale origins
def _batch_parity(pl, op, m, ctrl, n, seed, ctx):
    S, G = maps.sample_queries(m, n, seed=seed, min_dist=1.0, max_dist=4.0)
    sg, so = waypoint_pair(S, ctrl)
    gg, go = waypoint_pair(G, ctrl)
    rg, ag, _ = pl.plan_batch(sg, gg, max_seg=64, want_states=True)
    ro, ao = op.plan_batch(so, go, nthreads=8, max_seg=64)
    for i in range(n):
        assert_results_equal(rg[i], ro[i], (ctx, i))
    assert np.array_equal(ag, ao), ctx
    assert (ro["status"] == 0).sum() >= n // 8, (ctx, np.unique(ro["status"], return_counts=True))
    return ro


CASES = [  # (dim, control, U, res, dt)
    (2, mp.ACC, maps.make_U(1.0, 1, 2), 0.1, 1.0),
    (3, mp.ACC, maps.make_U(1.0, 1, 3), 0.15, 1.0),
    (2, mp.JRK, maps.make_U(1.0, 1, 2), float(np.float32(0.1)), 0.5),
]


@pytest.mark.gpu
@pytest.mark.parametrize("origin", [5e5, 5.3e6])
@pytest.mark.parametrize("case", range(len(CASES)))
def test_large_origin_plans_match_oracle(case, origin):
    """256 plans per case on salt-and-pepper maps (15 % occupied, so a one-voxel error flips a verdict) placed at
    UTM-scale origins with non-dyadic resolutions: every result field and every action row equals the oracle's."""
    dim, ctrl, U, res, dt = CASES[case]
    m = salt_map(dim, res, np.full(dim, origin) + np.arange(dim) * 0.37, seed=case)
    params = dict(v_max=2.0, a_max=1.0, dt=dt, tol_pos=0.5, max_num=1500)
    pl, op = make_pair(m, dim, params, U)
    _batch_parity(pl, op, m, ctrl, 256, seed=case, ctx=(case, origin))


@pytest.mark.gpu
def test_large_origin_shaped_plans_match_oracle():
    """The shaped kernels sample through cell_filtered: a search region mask on the same kind of map at 5.3e6."""
    m = salt_map(2, 0.15, np.array([5.3e6, 4.1e6]), seed=11)
    U = maps.make_U(1.0, 1, 2)
    pl, op = make_pair(m, 2, dict(v_max=2.0, a_max=1.0, dt=1.0, tol_pos=0.5, max_num=1500), U)
    mask = (np.random.RandomState(12).rand(int(np.prod(m.dim))) > 0.05).astype(np.uint8)
    pl.setSearchRegionMask(mask)
    op.set_search_region_mask(mask)
    _batch_parity(pl, op, m, mp.ACC, 256, seed=13, ctx="shaped")


# ---------------------------------------------------------------- 3. the other two filters of get_succ
TRACE_FIELDS = ("verdict", "n", "n_tested", "block_idx", "cost", "succ", "key")


@pytest.mark.gpu
@pytest.mark.parametrize("ctrl,v_max,dt,res", [(mp.ACC, 2.0, 1.0, 0.1), (mp.ACC, 1.5, 1.0, 0.15), (mp.JRK, 3.0, 0.5, 0.3)])
def test_expand_trace_adversarial(ctrl, v_max, dt, res):
    """get_succ rows (mplb_expand) against the oracle on states made for lattice_int and sample_divisor: positions at
    lattice half-steps (k + 0.5) * 0.01 on both sides of 2^30 * 0.01 (the end of lattice_int's fast path), derivatives
    at (k + 0.5) * 0.1 and at k * 0.1, with v_max * dt / res an integer."""
    cut = 2 ** 30
    dim = 2
    lo = (cut - 600) * 0.01
    m = salt_map(dim, res, np.array([lo, lo - 3.0]), seed=5, frac=0.1)
    U = maps.make_U(1.0, 1, dim)
    params = dict(v_max=v_max, a_max=1.0, dt=dt, tol_pos=0.5)
    pl, op = make_pair(m, dim, params, U)
    rs = np.random.RandomState(6)
    n = 240
    kx = rs.randint(cut - 400, cut + 400, size=n)
    ky = rs.randint(cut - 700, cut + 100, size=n)
    pos = np.stack([(kx + 0.5) * 0.01, (ky + 0.5) * 0.01], axis=1)
    half = rs.rand(n, 1) < 0.5
    kv = rs.randint(-int(v_max * 10) + 1, int(v_max * 10) - 1, size=(n, dim))
    vel = np.where(half, (kv + 0.5) * 0.1, kv * 0.1)
    ka = rs.randint(-9, 9, size=(n, dim))
    acc = np.where(half, (ka + 0.5) * 0.1, ka * 0.1) if ORDER[ctrl] >= 3 else None
    sg, so = waypoint_pair(pos, ctrl, vel=vel, acc=acc)
    assert np.any(np.abs(pos / 0.01) < cut) and np.any(np.abs(pos / 0.01) > cut)
    rows = pl.expand(sg)
    verdicts = set()
    for i in range(n):
        tr = op.succ_trace(so[i:i + 1])
        for f in TRACE_FIELDS:
            assert np.array_equal(rows[i][f], tr[f]), (i, f, rows[i][f], tr[f], sg[i])
        verdicts |= set(tr["verdict"].tolist())
    assert {2, 3} <= verdicts, verdicts


# ---------------------------------------------------------------- 4. lattice keys that leave int32
@pytest.mark.gpu
def test_key_range_rejected():
    """round(pos / 0.01) of the reference is an int: a map whose positions leave that range is refused, one just inside
    it plans like the oracle."""
    U = maps.make_U(1.0, 1, 2)
    params = dict(v_max=2.0, a_max=1.0, dt=1.0, tol_pos=0.5, max_num=1500)
    far = salt_map(2, 0.1, np.array([2.5e7, 100.0]), seed=1, frac=0.05)
    pl, _ = make_pair(far, 2, params, U)
    S, G = maps.sample_queries(far, 4, seed=1, min_dist=1.0, max_dist=4.0)
    sg, _ = waypoint_pair(S, mp.ACC)
    gg, _ = waypoint_pair(G, mp.ACC)
    with pytest.raises(mp.MplbError, match="int32"):
        pl.plan_batch(sg, gg)
    near = salt_map(2, 0.1, np.array([2.0e7, -2.0e7]), seed=2, frac=0.05)
    pl, op = make_pair(near, 2, params, U)
    _batch_parity(pl, op, near, mp.ACC, 32, seed=2, ctx="2.0e7")
