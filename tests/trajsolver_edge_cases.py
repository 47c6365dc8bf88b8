"""Seeded TrajSolver inputs at the batched solver's size and arithmetic edges (shared by the CPU and GPU tests).

Every case carries the kernel path it is there for (`tags`): the shared-memory / global-scratch split of each CTA, the
thread-stride loops of the 256-thread CTA, flag patterns, extreme segment times and coordinates, and degenerate input.
`ws_doubles` restates the kernel's work-space size (ts_ws_doubles in mpl_ros_b200/csrc/mplb_trajsolve.cu) so that the
boundaries are placed from the same formula the launch uses."""
import functools

import numpy as np

from trajsolver_cases import ACC, JRK, VEL, WAYPOINT_DTYPE, path_case

THREADS = 256                     # TS_THREADS
ORDER = {VEL: (2, 1), ACC: (4, 2), JRK: (6, 3)}  # control -> (N, R)
H100_SMEM_OPTIN = 232448          # cudaDevAttrMaxSharedMemoryPerBlockOptin of an H100 (227 KB)


@functools.lru_cache(maxsize=None)
def smem_doubles():
    """Doubles of work space a CTA may keep in shared memory: the opt-in limit less the 1 KB the launch keeps back."""
    optin = H100_SMEM_OPTIN
    try:
        import torch
        if torch.cuda.is_available():
            optin = torch.cuda.get_device_properties(0).shared_memory_per_block_optin
    except ImportError:
        pass
    return (optin - 1024) // 8


def ws_doubles(W, N, ncol):
    S, Wd = W - 1, W * N // 2
    d = 3 * S * N * N + Wd * ncol + Wd * Wd + Wd * ncol
    ints = 2 * S * N + 2 * Wd + 8
    return d + (ints + 1) // 2


def pos_global(W, dim, control):
    return ws_doubles(W, ORDER[control][0], dim) > smem_doubles()


def yaw_global(W, yaw_control):
    return ws_doubles(W, ORDER[yaw_control][0], 1) > smem_doubles()


def largest_fitting(N, ncol):
    W = 2
    while ws_doubles(W + 1, N, ncol) <= smem_doubles():
        W += 1
    return W


def nfree(wps, control):
    """Free derivatives of the position solve: W * N/2 minus the fixed ones (poly_solver.cpp:78-88)."""
    H = ORDER[control][0] // 2
    return len(wps) * H - sum(bin(int(c) & ((1 << H) - 1)).count("1") for c in wps["control"])


class Case:
    def __init__(self, name, tags, dim, control, yaw_control, wps, dts):
        self.name, self.tags, self.dim, self.control, self.yaw_control = name, tuple(tags), dim, control, yaw_control
        self.wps, self.dts = wps, np.asarray(dts, dtype=np.float64)

    @property
    def W(self):
        return len(self.wps)

    def __repr__(self):
        return "%s(W=%d)" % (self.name, self.W)


def make_list(rs, dim, W, end_control, interior=(VEL,), dts=None, offset=0.0, step=2.0):
    w = np.zeros(W, dtype=WAYPOINT_DTYPE)
    w["pos"][:, :dim] = offset + np.cumsum(rs.uniform(-step, step, size=(W, dim)), axis=0)
    for f in ("vel", "acc", "jrk"):
        w[f][:, :dim] = rs.uniform(-1, 1, size=(W, dim))
    w["yaw"] = rs.uniform(-3, 3, size=W)
    w["control"] = [interior[i % len(interior)] for i in range(W)]
    w["control"][0] = w["control"][-1] = end_control
    if dts is None:
        dts = rs.uniform(0.4, 2.5, size=W - 1)
    return w, np.asarray(dts, dtype=np.float64)


def extreme_dts(rs, n):
    """Durations spread log-uniformly over 1e-3 .. 1e3, both ends present, in random order."""
    d = 10.0 ** rs.uniform(-3, 3, size=n)
    if n >= 2:
        d[rs.choice(n, 2, replace=False)] = (1e-3, 1e3)
    return d


def cases():
    out = []
    rs = np.random.RandomState(2024)
    names = {VEL: "VEL", ACC: "ACC", JRK: "JRK"}

    # ---- shared memory vs global scratch: for every (dim, control, yaw_control) the largest W whose two CTAs both fit and
    # W + 1, and where the yaw CTA crosses later than the position CTA, its own last fitting W and W + 1 (a split pair)
    for dim in (2, 3):
        for c in (VEL, ACC, JRK):
            for yc in (VEL, ACC, JRK):
                wp, wy = largest_fitting(ORDER[c][0], dim), largest_fitting(ORDER[yc][0], 1)
                for W in sorted({min(wp, wy), min(wp, wy) + 1, wy, wy + 1}):
                    w, d = make_list(rs, dim, W, c)
                    out.append(Case("smem_%dd_%s_%s_%d" % (dim, names[c], names[yc], W), ["smem"], dim, c, yc, w, d))

    # ---- thread-stride loops
    for W in (257, 258, 259):  # phase 1: a second pass over the segments (S > 256)
        w, d = make_list(rs, 2, W, VEL)
        out.append(Case("threads_seg_2d_VEL_%d" % W, ["threads", "seg>256"], 2, VEL, VEL, w, d))
    w, d = make_list(rs, 3, 258, JRK, (VEL, VEL, ACC))
    out.append(Case("threads_seg_3d_JRK_258", ["threads", "seg>256", "nfree>257"], 3, JRK, VEL, w, d))
    for nf in (255, 256, 257, 258):  # phases 3b / 3c: JRK ends, VEL interior -> nfree = 2 (W - 2); one ACC interior point -> -1
        W = (nf + 1) // 2 + 2
        w, d = make_list(rs, 3, W, JRK)
        if nf % 2:
            w["control"][W // 2] = ACC
        assert nfree(w, JRK) == nf
        out.append(Case("threads_nfree_%d" % nf, ["threads", "nfree"], 3, JRK, VEL, w, d))
    for dim, Ss in ((3, (85, 86)), (2, (127, 128, 129))):  # phase 4: S * ncol around 256
        for S in Ss:
            w, d = make_list(rs, dim, S + 1, ACC)
            out.append(Case("threads_phase4_%dd_S%d" % (dim, S), ["threads", "phase4"], dim, ACC, VEL, w, d))

    # ---- flag patterns
    w, d = make_list(rs, 3, 9, JRK, (JRK,))  # everything fixed: nfree = 0 in both solves
    out.append(Case("flags_all_fixed", ["flags"], 3, JRK, VEL, w, d))
    w, d = make_list(rs, 2, 14, VEL, (VEL,))  # VEL ends under a JRK solver: velocity and acceleration free at the ends
    out.append(Case("flags_vel_ends_jrk", ["flags"], 2, JRK, JRK, w, d))
    w, d = make_list(rs, 3, 16, JRK, (VEL, ACC, JRK))  # alternating interiors
    out.append(Case("flags_alternating_3d", ["flags"], 3, JRK, ACC, w, d))
    w, d = make_list(rs, 2, 15, ACC, (JRK, VEL, ACC))
    out.append(Case("flags_alternating_2d", ["flags"], 2, ACC, JRK, w, d))
    for c in (VEL, ACC, JRK):
        w, d = make_list(rs, 3, 2, c)
        out.append(Case("flags_two_%s" % names[c], ["flags"], 3, c, c, w, d))

    # ---- segment times and coordinates
    for dim, c, W, dt in ((3, JRK, 40, 1.0), (2, ACC, 33, 0.2), (3, ACC, 300, 0.2)):  # refinement: one dt everywhere
        w, d = make_list(rs, dim, W, c, dts=np.full(W - 1, dt), step=dt)
        out.append(Case("equal_dt_%dd_%s_%d" % (dim, names[c], W), ["times", "equal"] + (["long"] if W > 200 else []), dim, c, VEL, w, d))
    for dim, c, W in ((3, JRK, 12), (2, ACC, 30), (3, VEL, 40)):
        w, d = make_list(rs, dim, W, c, dts=extreme_dts(rs, W - 1))
        out.append(Case("extreme_dt_%dd_%s_%d" % (dim, names[c], W), ["times", "extreme"], dim, c, JRK, w, d))
    for dim, c, W in ((3, JRK, 12), (2, JRK, 36)):
        w, d = make_list(rs, dim, W, c, offset=5e6)
        out.append(Case("offset_%dd_%s_%d" % (dim, names[c], W), ["coords", "offset"], dim, c, ACC, w, d))
    for dim, c, W in ((3, JRK, 10), (2, ACC, 28)):
        w, d = make_list(rs, dim, W, c, dts=extreme_dts(rs, W - 1), offset=5e6)
        out.append(Case("offset_extreme_%dd_%s_%d" % (dim, names[c], W), ["coords", "offset", "extreme"], dim, c, VEL, w, d))

    # ---- degenerate input: setPath with a repeated point gives a zero duration (NaN coefficients in the reference)
    path = [(0, 0, 0), (1, 0, 0.5), (1, 0, 0.5), (3, 2, 1), (3, 3, 0), (4, 3, 1)]
    for dim in (2, 3):
        for c in (VEL, ACC, JRK):
            w, d = path_case(dim, c, [p[:dim] for p in path])
            assert (d == 0).sum() == 1
            out.append(Case("degenerate_%dd_%s" % (dim, names[c]), ["degenerate"], dim, c, ACC, w, d))
    return out


def mixed_batch():
    """One launch: W from 2 to 300 in shuffled order, 2-D ACC with a VEL yaw, both scratch kinds for both CTAs, plus the two
    lists the reference leaves empty (W = 0 and W = 1)."""
    rs = np.random.RandomState(77)
    Ws = [2, 3, 5, 9, 17, 33, 49, 64, 77, 78, 100, 129, 160, 161, 162, 200, 300, 0, 1]
    rs.shuffle(Ws)
    out = []
    for W in Ws:
        if W < 2:
            w, d = np.zeros(W, dtype=WAYPOINT_DTYPE), np.zeros(0)
        else:
            w, d = make_list(rs, 2, W, ACC, (VEL, VEL, ACC))
        out.append(Case("mixed_%d" % W, ["mixed"], 2, ACC, VEL, w, d))
    return out


def one_global_batch():
    """3-D JRK / JRK: twenty lists that fit shared memory and one (W = 50) whose position CTA alone needs global scratch."""
    rs = np.random.RandomState(78)
    Ws = list(rs.randint(2, 50, size=20))
    Ws.insert(7, 50)
    return [Case("one_global_%d_%d" % (i, W), ["one_global"], 3, JRK, JRK, *make_list(rs, 3, int(W), JRK)) for i, W in enumerate(Ws)]


def mpmath_cases():
    """Short lists (W <= 12) for the high-precision solve: well-conditioned ones (durations in [0.4, 2.5], coordinates of a few
    metres) and the extreme-duration / 5e6-offset ones, every solver order."""
    rs = np.random.RandomState(99)
    out = []
    for dim, c, yc, W in ((2, VEL, VEL, 7), (3, ACC, JRK, 9), (3, JRK, ACC, 12), (2, JRK, JRK, 10)):
        w, d = make_list(rs, dim, W, c, (VEL, ACC))
        out.append(Case("mp_good_%d" % len(out), ["good"], dim, c, yc, w, d))
    for dim, c, W in ((3, JRK, 12), (2, ACC, 10)):
        w, d = make_list(rs, dim, W, c, dts=extreme_dts(rs, W - 1))
        out.append(Case("mp_extreme_%d" % len(out), ["extreme"], dim, c, JRK, w, d))
    for dim, c, W in ((3, JRK, 12), (2, ACC, 11)):
        w, d = make_list(rs, dim, W, c, offset=5e6)
        out.append(Case("mp_offset_%d" % len(out), ["offset"], dim, c, ACC, w, d))
    w, d = make_list(rs, 3, 10, JRK, dts=extreme_dts(rs, 9), offset=5e6)
    out.append(Case("mp_offset_extreme_%d" % len(out), ["offset", "extreme"], 3, JRK, JRK, w, d))
    return out
