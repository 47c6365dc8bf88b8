"""The case generator of the GPU fuzz (tests/fuzz_cases.py) reaches every astar_batch_kernel instantiation, and in every
one the oracle's plans include successes and plans whose primitives meet obstacles, so that no cell of the GPU fuzz
degenerates into blocked starts or empty searches.  CPU only: the oracle plans the same cases the GPU test runs."""
import numpy as np

import fuzz_cases as F

SEEDS = 4  # the default number of seeds per cell of tests/test_gpu_fuzz.py


def test_instantiation_mapping():
    assert len(F.CELLS) == len(set(F.CELLS)) == 24
    assert F.instantiation(2, F.mp.SNP, 33, False) == (2, 4, 4, False)
    assert F.instantiation(3, F.mp.VEL | 16, 27, True) == (3, 1, 1, True)
    assert F.instantiation(3, F.mp.JRK, 32, False) == (3, 3, 1, False)


def test_generator_covers_every_instantiation():
    seen = {}
    for cell in F.CELLS:
        runs = ok = met = truncated = 0
        for seed in range(SEEDS):
            c = F.make_case(cell, seed)
            assert c.cell == cell, (F.cell_name(cell), seed, c.cell)
            op = c.build_oracle()
            so, go = c.waypoints(c.start, vel=c.vel, yaw=c.yaw)
            gs = c.waypoints(c.goal)[1]
            r = op.plan(so, gs)
            _, _, bso, bgo = c.batch_waypoints(seed)
            rb, _ = op.plan_batch(bso, bgo, nthreads=8, max_seg=c.max_seg)
            rs = np.concatenate([[r], rb])
            runs += len(rs)
            ok += int((rs["status"] == 0).sum())
            met += int((rs["n_valid"] < rs["n_prims"]).sum())
            truncated += int(((rb["status"] == 0) & (rb["n_seg"] > c.max_seg)).sum())
        seen[cell] = (runs, ok, met, truncated)
    bad = {F.cell_name(c): v for c, v in seen.items() if not (v[1] > 0 and v[2] > 0)}
    assert not bad, bad
    assert sum(v[3] for v in seen.values()) > 0  # some batch plans are longer than max_seg


def test_generator_varies_the_frame_and_the_shaping():
    cases = [F.make_case(cell, seed) for cell in F.CELLS for seed in range(SEEDS)]
    shaped = [c for c in cases if c.shaped]
    assert any(abs(c.map.origin).max() > 1e5 for c in cases)
    assert {0.15, 0.3, float(np.float32(0.1))} <= {c.map.res for c in cases}
    assert {0.0, 1.0, 2.0, 3.5} <= {c.params["epsilon"] for c in cases}
    assert any(c.control & 15 == F.mp.VEL and c.params["v_max"] < np.abs(c.U[:, :c.dim]).max() for c in cases)
    assert any(c.pot is not None for c in shaped) and any(c.region is not None for c in shaped)
    assert any(c.control & 16 for c in shaped)
    assert any(c.pot is not None and c.region is not None for c in shaped)
