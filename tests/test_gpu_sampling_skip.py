"""The search kernel's sampler skips every collision sample whose index is not below the first blocked sample already
found for its primitive (sample_granules over the wave-major granule list of b1_warp).  Results must not change: a
primitive's verdict and n_samples (first blocked index + 1) are what the reference computes.

These plans are chosen so that the skip matters: box obstacles at fine resolutions make primitives of 20 to 40 samples
(3 to 6 granules of 8) whose first blocked sample often lies in a later granule, and both the |U| <= 32 kernel (NB = 1)
and the |U| > 32 kernel (NB = 4, four 32-control batches in one wave-major list) are covered."""
import numpy as np
import pytest

import mpl_ros_b200 as mp
from mpl_ros_b200 import maps
from helpers_gpu import assert_results_equal, make_pair, waypoint_pair

pytestmark = pytest.mark.gpu


def box_map(nd, res, seed, n_boxes):
    rs = np.random.RandomState(seed)
    dim = len(nd)
    g = np.zeros(tuple(nd[::-1]), dtype=np.int8)
    for _ in range(n_boxes):
        sz = [rs.randint(2, max(3, nd[k] // 4)) for k in range(dim)]
        lo = [rs.randint(0, nd[k] - sz[k]) for k in range(dim)]
        g[tuple(slice(lo[k], lo[k] + sz[k]) for k in range(dim))[::-1]] = 100
    return maps.GridMap(np.full(dim, -0.3), nd, res, g.reshape(-1))


CASES = [  # (nd, res, control, U, dt)
    ([48, 48, 16], 0.1, mp.ACC, maps.make_U(1.0, 1, 3), 1.0),   # |U| = 27, 21 samples per moving primitive
    ([48, 48, 16], 0.1, mp.ACC, maps.make_U(1.0, 2, 3), 1.0),   # |U| = 125
    ([96, 96], 0.05, mp.JRK, maps.make_U(1.0, 1, 2), 1.0),      # up to 41 samples
    ([96, 96], 0.05, mp.ACC, maps.make_U(1.0, 5, 2), 1.0),      # |U| = 121
]


@pytest.mark.parametrize("case", range(len(CASES)))
def test_plans_with_late_blocked_samples_match_oracle(case):
    nd, res, ctrl, U, dt = CASES[case]
    dim = len(nd)
    m = box_map(nd, res, seed=case, n_boxes=24 if dim == 3 else 30)
    params = dict(v_max=2.0, a_max=1.0, dt=dt, tol_pos=0.5, max_num=1500)
    if ctrl == mp.JRK:
        params["j_max"] = 1.0
    pl, op = make_pair(m, dim, params, U)
    S, G = maps.sample_queries(m, 128, seed=case, min_dist=1.0, max_dist=4.0)
    sg, so = waypoint_pair(S, ctrl)
    gg, go = waypoint_pair(G, ctrl)
    rg, ag, _ = pl.plan_batch(sg, gg, max_seg=64, want_states=True)
    ro, ao = op.plan_batch(so, go, nthreads=8, max_seg=64)
    for i in range(len(ro)):
        assert_results_equal(rg[i], ro[i], (case, i))
    assert np.array_equal(ag, ao), case
    assert ro["n_samples"].sum() > 0 and ro["n_valid"].sum() < ro["n_prims"].sum(), case  # the plans do meet obstacles
