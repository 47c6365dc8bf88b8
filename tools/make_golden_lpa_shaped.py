"""Records tests/golden/lpa_shaped_flows.npz from the REFERENCE'S OWN LPA* sources (oracle/_ref, see tools/make_golden_lpa.py)
over the potential-map and yaw replanning flows of tests/lpa_shaped_flow.py: one digest row per step (state-space dump in hm_
order, heap array, best_child_, linked points, result).  The checker in libm trig mode (the reference's cos / sin) is asserted
identical step by step while recording.  Needs oracle/_ref/libmplref.so:  python tools/make_golden_lpa_shaped.py"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from oracle import ref  # noqa: E402
import oracle  # noqa: E402
import lpa_flow  # noqa: E402
import lpa_shaped_flow as F  # noqa: E402

PATH = os.path.join(ROOT, "tests", "golden", "lpa_shaped_flows.npz")


def record():
    """name -> digest rows of the reference's run (the checker in libm mode must agree step by step)"""
    out = {}
    for name in F.FLOWS:
        a, _ = F.run_flow(name, ref.RefMap, ref.RefPlanner)
        b, _ = F.run_flow(name, oracle.OracleMap, F.OraclePlannerLibm)
        lpa_flow.assert_same(b, a, name)
        out[name] = F.digest(a)
    return out


def main():
    if not ref.available():
        raise SystemExit("needs oracle/_ref/libmplref.so (build() makes it where the reference tree is present)")
    out = record()
    for name, d in out.items():
        print(name, len(d), "steps", [(int(r["status"]), float(r["cost"]), int(r["pops"])) for r in d if r["status"] != -9])
    np.savez_compressed(PATH, **out)


if __name__ == "__main__":
    main()
