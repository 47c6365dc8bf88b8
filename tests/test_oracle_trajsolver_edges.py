"""The TrajSolver oracle (oracle/poly_oracle.cpp) on the batched solver's edge cases (tests/trajsolver_edge_cases.py), CPU only:
(1) against the reference's own traj_solver.h / poly_solver.cpp compiled here (oracle/_ref; where it is absent, against
    what those sources returned when recorded, tests/ref_record.py) — bit for bit, NaN placement included;
(2) against numpy's LAPACK on the long and extreme lists — the rounding-level difference a real Eigen build shows;
(3) against the same closed form solved with mpmath at 256 bits on short lists — the oracle's own error, which is also the
    GPU's, since the GPU equals the oracle bit for bit (tests/test_gpu_trajsolver_edges.py)."""
import functools
import math

import mpmath
import numpy as np
import pytest

import oracle
import ref_record as R
from oracle import ref
from trajsolver_cases import ACC, JRK, VEL
import trajsolver_edge_cases as E
from trajsolver_numpy import numpy_poly_solve

ALL = {c.name: c for c in E.cases() + E.mixed_batch() + E.one_global_batch() + E.mpmath_cases() if c.W >= 2}


@functools.lru_cache(maxsize=None)
def solved(name):
    c = ALL[name]
    return oracle.traj_solve(c.dim, c.control, c.wps, c.dts, c.yaw_control)


def coef_error(got, want):
    """(per-coefficient error, normwise error) of one solve's rows [S, ncol, 6]: the first is max |got - want| over each
    (axis, polynomial order) divided by the largest |want| of that (axis, order) along the trajectory, so a 5e6 m position
    does not hide the error of a velocity term; the second divides by the largest |want| of the whole solve."""
    scale = np.abs(want).max(axis=0)
    err = np.abs(got - want)
    assert not err[:, scale == 0].any()  # orders the solver does not use stay exactly zero
    per = float((err.max(axis=0)[scale > 0] / scale[scale > 0]).max())
    return per, float(err.max() / np.abs(want).max())


def test_edge_cases_take_their_paths():
    """The generator places every boundary where the kernel's work-space formula puts it (H100 opt-in shared memory)."""
    cs = {c.name: c for c in E.cases()}
    fit = lambda c, ncol: E.largest_fitting(E.ORDER[c][0], ncol)  # noqa: E731
    if E.smem_doubles() == (E.H100_SMEM_OPTIN - 1024) // 8:  # 28 928 doubles
        assert (fit(JRK, 3), fit(JRK, 2), fit(ACC, 3), fit(VEL, 3), fit(VEL, 2)) == (49, 50, 77, 159, 160)
        assert (fit(JRK, 1), fit(ACC, 1), fit(VEL, 1)) == (50, 78, 161)
    split = [c for c in cs.values() if "smem" in c.tags and E.pos_global(c.W, c.dim, c.control) != E.yaw_global(c.W, c.yaw_control)]
    assert any(c.dim == 3 and c.control == JRK and c.yaw_control == JRK and c.W == fit(JRK, 3) + 1 for c in split)
    assert any(c.control == JRK and c.yaw_control == ACC and fit(JRK, 3) < c.W <= fit(ACC, 1) for c in split)
    for dim, c in ((2, VEL), (3, VEL), (2, ACC), (3, ACC), (2, JRK), (3, JRK)):
        Ws = {x.W for x in cs.values() if "smem" in x.tags and x.dim == dim and x.control == c}
        assert {fit(c, dim), fit(c, dim) + 1} <= Ws
    assert {257, 258, 259} <= {c.W for c in cs.values() if "seg>256" in c.tags}
    assert {255, 256, 257, 258} == {E.nfree(c.wps, c.control) for c in cs.values() if "nfree" in c.tags}
    assert E.nfree(cs["threads_seg_3d_JRK_258"].wps, JRK) > 257
    ph4 = {(c.dim, (c.W - 1) * c.dim) for c in cs.values() if "phase4" in c.tags}
    assert {(3, 255), (3, 258), (2, 254), (2, 256), (2, 258)} == ph4
    assert sum(c.W > 200 for c in ALL.values()) <= 10
    mixed = [c for c in E.mixed_batch() if c.W >= 2]
    assert any(E.pos_global(c.W, 2, ACC) for c in mixed) and any(not E.pos_global(c.W, 2, ACC) for c in mixed)
    assert sum(E.pos_global(c.W, 3, JRK) or E.yaw_global(c.W, JRK) for c in E.one_global_batch()) == 1


@pytest.mark.parametrize("name", sorted(ALL))
def test_oracle_equals_reference_sources(name):
    c = ALL[name]
    a = solved(name)
    assert a.shape == (c.W - 1, c.dim + 1, 6)
    live = lambda: ref.traj_solve(c.dim, c.control, c.wps, c.dts, c.yaw_control)  # noqa: E731
    if "degenerate" in c.tags:  # stored whole: NaN placement and every other value
        b = R.value(name, live)
        nan = np.isnan(a)
        assert nan.any() and not nan.all(), name
        assert np.array_equal(nan, np.isnan(b)) and np.array_equal(a[~nan], b[~nan]), name
    else:
        assert np.isfinite(a).all(), name
        assert R.same(name, a, live), name


LAPACK = [n for n, c in ALL.items() if c.W > 100 or set(c.tags) & {"extreme", "offset", "equal"}]


def _lapack(c):
    N, Rr = E.ORDER[c.control]
    pos = numpy_poly_solve(c.dim, N, Rr, c.wps, c.dts, lambda w, k: (w["pos"], w["vel"], w["acc"])[k][:c.dim])
    ys = c.wps.copy()  # the yaw solve (traj_solver.h:86-103): interior VEL, the ends yaw_control, key frames = yaw
    ys["control"] = VEL
    ys["control"][0] = ys["control"][-1] = c.yaw_control
    Ny, Ry = E.ORDER[c.yaw_control]
    yaw = numpy_poly_solve(1, Ny, Ry, ys, c.dts, lambda w, k: np.array([w["yaw"] if k == 0 else 0.0]))
    return pos, yaw


@pytest.mark.parametrize("name", LAPACK)
def test_against_numpy_lapack(name):
    """Per case the worst relative difference between the oracle and LAPACK (per coefficient and normwise).  Durations in
    [0.4, 2.5] and coordinates of metres: < 1e-11 per coefficient at every length up to 300.  Durations over 1e-3 .. 1e3, or a
    5e6 m offset, alone: < 1e-9 normwise.  Both together: printed only — there the 1e-6 does not hold (DESIGN.md 4.11)."""
    c = ALL[name]
    got = solved(name)
    pos, yaw = _lapack(c)
    per_p, norm_p = coef_error(got[:, :c.dim], pos)
    per_y, norm_y = coef_error(got[:, c.dim:], yaw)
    print("%-28s W=%3d  position: %.1e per coefficient, %.1e normwise   yaw: %.1e, %.1e" % (name, c.W, per_p, norm_p, per_y, norm_y))
    hard = set(c.tags) & {"extreme", "offset"}
    if not hard:
        assert max(per_p, per_y) < 1e-11, (name, per_p, per_y)
    elif len(hard) == 1:
        assert max(norm_p, norm_y) < 1e-9, (name, norm_p, norm_y)


def mp_solve(dim, N, Rr, flags, values, dts, prec=256):
    """The closed form of poly_solver.cpp:23-221 in exact-input, `prec`-bit arithmetic: block-diagonal A and Q, the same
    fixed/free ordering, R = Mᵀ blockdiag(A_s⁻ᵀ Q_s A_s⁻¹) M, Dp = -Rpp⁻¹ Rpf Df, p_s = A_s⁻¹ d_s, coeff_k = p_k k!.
    flags[w]: control bits of waypoint w; values(w, k) -> dim floats.  Returns [S, dim, 6] floats and cond_2(Rpp)."""
    with mpmath.workprec(prec):
        W, S, H = len(flags), len(flags) - 1, N // 2
        mf = mpmath.mpf
        Ainv, K = [], []
        for s in range(S):
            T = mf(float(dts[s]))
            A = mpmath.zeros(N, N)
            Q = mpmath.zeros(N, N)
            for n in range(N):
                if n < H:
                    A[n, n] = math.factorial(n)
                for r in range(H):
                    if r <= n:
                        A[H + r, n] = mf(math.factorial(n) // math.factorial(n - r)) * T ** (n - r)
                for r in range(N):
                    if r >= Rr and n >= Rr:
                        val = 1
                        for m in range(Rr):
                            val *= (r - m) * (n - m)
                        Q[r, n] = val * T ** (r + n - 2 * Rr + 1) / (r + n - 2 * Rr + 1)
            Ai = mpmath.inverse(A)
            Ainv.append(Ai)
            K.append(Ai.T * Q * Ai)
        use = lambda w, k: (int(flags[w]) >> k) & 1  # noqa: E731
        nfixed = sum(use(w, k) for w in range(W) for k in range(H))
        Wd = W * H
        rows = {}  # new id -> [(segment, local row)]
        fix = fre = 0
        for w in range(W):
            for k in range(H):
                nid = fix if use(w, k) else nfixed + fre
                att = []
                if w < W - 1:
                    att.append((w, k))      # start of segment w
                if w > 0:
                    att.append((w - 1, H + k))  # end of segment w - 1
                rows[nid] = (w, k, att)
                if use(w, k):
                    fix += 1
                else:
                    fre += 1
        Rm = mpmath.zeros(Wd, Wd)
        for i in range(Wd):
            for j in range(Wd):
                acc = mf(0)
                for si, li in rows[i][2]:
                    for sj, lj in rows[j][2]:
                        if si == sj:
                            acc += K[si][li, lj]
                Rm[i, j] = acc
        D = mpmath.zeros(Wd, dim)
        for nid in range(nfixed):
            w, k, _ = rows[nid]
            v = values(w, k)
            for a in range(dim):
                D[nid, a] = mf(float(v[a]))
        nfree = Wd - nfixed
        cond = 1.0
        if W > 2 and nfree > 0:
            Rpp = Rm[nfixed:, nfixed:]
            Rpf = Rm[nfixed:, :nfixed]
            rhs = Rpf * D[:nfixed, :]
            Dp = mpmath.inverse(Rpp) * rhs
            for i in range(nfree):
                for a in range(dim):
                    D[nfixed + i, a] = -Dp[i, a]
            cond = float(np.linalg.cond(np.array(Rpp.tolist(), dtype=np.float64)))
        out = np.zeros((S, dim, 6))
        for s in range(S):
            d = mpmath.zeros(N, dim)
            for k in range(H):
                for a in range(dim):
                    d[k, a] = D[_nid(rows, s, k), a]
                    d[H + k, a] = D[_nid(rows, s + 1, k), a]
            p = Ainv[s] * d
            for a in range(dim):
                for k in range(N):
                    out[s, a, 5 - k] = float(p[k, a] * math.factorial(k))
        return out, cond


def _nid(rows, w, k):
    for nid, (ww, kk, _) in rows.items():
        if ww == w and kk == k:
            return nid
    raise KeyError((w, k))


def hp_solve(c):
    N, Rr = E.ORDER[c.control]
    pos, cp = mp_solve(c.dim, N, Rr, c.wps["control"], lambda w, k: (c.wps["pos"], c.wps["vel"], c.wps["acc"])[k][w][:c.dim], c.dts)
    yflags = [VEL] * c.W
    yflags[0] = yflags[-1] = c.yaw_control
    Ny, Ry = E.ORDER[c.yaw_control]
    yaw, cy = mp_solve(1, Ny, Ry, yflags, lambda w, k: [c.wps["yaw"][w] if k == 0 else 0.0], c.dts)
    return pos, yaw, cp, cy


@pytest.mark.parametrize("name", [c.name for c in E.mpmath_cases()])
def test_against_high_precision(name):
    """The oracle's error against a 256-bit solve.  Well-conditioned lists (durations in [0.4, 2.5], coordinates of metres):
    at most 1e-9 per coefficient.  Extreme durations and 5e6 m offsets: printed with the condition number of Rpp."""
    c = ALL[name]
    got = solved(name)
    pos, yaw, cp, cy = hp_solve(c)
    per_p, norm_p = coef_error(got[:, :c.dim], pos)
    per_y, norm_y = coef_error(got[:, c.dim:], yaw)
    print("%-22s W=%2d  position: %.1e per coefficient, %.1e normwise, cond(Rpp) %.1e   yaw: %.1e, %.1e, cond %.1e"
          % (name, c.W, per_p, norm_p, cp, per_y, norm_y, cy))
    assert np.isfinite(got).all()
    if "good" in c.tags:
        assert max(per_p, per_y) <= 1e-9, (name, per_p, per_y)


def test_high_precision_solve_is_the_closed_form():
    """The 256-bit solve and numpy's LAPACK agree on a well-conditioned list to double rounding, and the 256-bit solve does
    not move between 256 and 320 bits, so it measures the oracle and not itself."""
    c = ALL[E.mpmath_cases()[2].name]
    pos, yaw, _, _ = hp_solve(c)
    lp, ly = _lapack(c)
    assert coef_error(lp, pos)[0] < 1e-11 and coef_error(ly, yaw)[0] < 1e-11
    N, Rr = E.ORDER[c.control]
    hi, _ = mp_solve(c.dim, N, Rr, c.wps["control"], lambda w, k: (c.wps["pos"], c.wps["vel"], c.wps["acc"])[k][w][:c.dim], c.dts, prec=320)
    assert np.array_equal(hi, pos)
