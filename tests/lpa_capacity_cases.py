"""Cases for the LPA* capacity paths (DESIGN.md section 4.12): array growth in first plans, replans and after re-rooting,
predecessor-pool growth, the exact fill that leaves no room for a new start node, batches whose sessions grow in different
relaunch rounds, and trajectories longer than the 4096 rows one k_lpa_plan launch keeps per plan.  Shared by the host build of
the device core (tests/test_oracle_lpa_capacity.py) and the GPU (tests/test_gpu_lpa_capacity.py).

The initial sizes below were chosen on the host build of the core, which makes the same growth decisions as the device (same
pop-time check, same host policy).  Every test also asserts through the capacity export that its branch was taken, so a case
that stops reaching its branch fails instead of passing vacuously."""
import numpy as np

import oracle
from test_oracle_lpa_fuzz import sequence_case

# (flow of lpa_flow.FLOWS, initial node capacity): the first growth happens in the replan that follows updateBlockedNodes /
# updateClearedNodes of the flow's first round (corridor_jrk: 11 965 nodes after the first plan, 11 971 after the blocked replan)
BLOCKED_GROWTH = ("corridor_jrk", 11970)
CLEARED_GROWTH = ("corridor_jrk", 11976)
# getSubStateSpace with a predecessor pool smaller than (stored edges + 16) + |U|: skir_acc keeps 4 067 node records after its
# first plans, the re-root drops most of them from hm_, and the blocked replan after it grows the arrays to 7 932 records
REROOT = ("skir_acc", 4067 + 27, 65536)
# growth driven by the predecessor pool alone: corridor_acc never has more than 2 514 node records
PRED_ONLY = ("corridor_acc", 8192, 128)
# (dim, sequence seed of test_oracle_lpa_fuzz, F): the first plan ends with exactly F node records and, planned with F as the
# initial size, never grows: its last pop created |U| new nodes in exactly the room that was left
EXACT_FILL = [(2, 9, 382), (3, 7, 513)]
# batch: 8 random replanners of test_oracle_lpa_fuzz per dimension (|U| = 9 and 25 in 2D, 27 and 40 in 3D) as (seed, d): the
# initial node size is the first plan's node count N shifted right by d, so the session doubles at least d times; None keeps
# the default size and never grows
BATCH = {2: [(2, 4), (10, 3), (1, 1), (11, None), (5, 1), (13, None), (9, 1), (12, None)],
         3: [(4, 3), (14, 1), (6, 4), (2, 3), (9, None), (0, 1), (13, None), (7, 1)]}


def sizes(nodes, preds=None):
    """planner parameters for the initial sizes (names shared by the GPU adaptor and the host build)"""
    out = {"lpa_init_nodes": int(nodes)}
    if preds is not None:
        out["lpa_init_preds"] = int(preds)
    return out


class CapacityLog:
    """Mixin for an LpaMixin-shaped planner with lpa_capacity(): after every LPA* call, the capacity export, hm_'s size and
    the predecessor records its nodes list, in self.cap_log"""

    def _logged(self, op, out):
        nodes = self.lpa_nodes()
        c = self.lpa_capacity()
        c.update(op=op, hm=len(nodes), live_preds=int(nodes["n_pred"].sum()) if len(nodes) else 0)
        self.__dict__.setdefault("cap_log", []).append(c)
        return out

    def lpa_plan(self, s, g):
        return self._logged("plan", super().lpa_plan(s, g))

    def lpa_update_blocked_nodes(self, c):
        return self._logged("block", super().lpa_update_blocked_nodes(c))

    def lpa_update_cleared_nodes(self, c):
        return self._logged("clear", super().lpa_update_cleared_nodes(c))

    def lpa_get_sub_state_space(self, k):
        return self._logged("sub", super().lpa_get_sub_state_space(k))


def peak(log):
    """(peak node records, peak predecessor records listed by hm_ members) over a capacity log"""
    return max(c["n_nodes_physical"] for c in log), max(c["live_preds"] for c in log)


def random_planner(cm, cp, case, dim, extra=None):
    nd, origin, res, data, ctl, U, prm, _, _, _ = case
    m = cm(origin, nd, data, res)
    m.free_unknown()
    p = cp(dim)
    p.set_map(m)
    for k, v in dict(prm, **(extra or {})).items():
        p.set_param(k, v)
    p.set_controls(U)
    p._lpa_control = ctl
    return m, p


def random_waypoints(case, dim):
    _, _, _, _, ctl, _, _, start, goal, vel = case
    s, g = oracle.make_waypoints(1), oracle.make_waypoints(1)
    s["pos"][0, :dim], g["pos"][0, :dim], s["vel"][0, :dim] = start, goal, vel
    s["control"] = g["control"] = ctl
    return s, g


def fuzz_case(dim, seed):
    return sequence_case(seed, dim)[1]


def off_lattice_start(s):
    """the start moved 0.0137 m along x: another lattice key (0.01 m steps), off the lattice the first plan built (the tests
    assert that no state of the first plan has that key)"""
    s2 = s.copy()
    s2["pos"][0, 0] += 0.0137
    return s2


def lattice_key(w, dim):
    """Waypoint's lattice ints (waypoint.h:92-125 / make_key of mplb_lpa_core.h), padded to 16 with the count last"""
    order = {1: 1, 3: 2, 7: 3, 15: 4}[int(w["control"][0]) & 15]
    key = []
    for i in range(dim):
        key.append(int(np.round(w["pos"][0, i] / 0.01)))
        for d, f in ((2, "vel"), (3, "acc"), (4, "jrk")):
            if order >= d:
                key.append(int(np.round(w[f][0, i] / 0.1)))
    return np.array(key + [0] * (15 - len(key)) + [len(key)], dtype=np.int32)


# ---- trajectories longer than one launch's 4096 rows: 2D, VEL controls {-1, 0, 1}^2 (|U| = 9), dt = 0.01 s on a free strip
# one 0.01 m cell wide between two walls; every step moves one key unit along x, sideways steps hit a wall, so the plan expands
# about one state per segment (plus the few behind the start)
STRIP_DT = 0.01
LONG_SEG = 5000
SHORT_SEG = 4096


def strip_case(n_seg):
    nx = n_seg + 120
    data = np.zeros((3, nx), dtype=np.int8)  # [y][x], x fastest
    data[0, :] = 100
    data[2, :] = 100
    origin = np.array([0.0, 0.0])
    nd = np.array([nx, 3], dtype=np.int32)
    U = np.array([[dx, dy] for dx in (-1.0, 0.0, 1.0) for dy in (-1.0, 0.0, 1.0)])
    prm = dict(v_max=1.0, dt=STRIP_DT, w=10.0, epsilon=1.0, tol_pos=0.004)
    start = np.array([0.5013, 0.0137])  # away from key rounding ties (x / 0.01 = k + 0.5), which would merge neighbours
    goal = np.array([0.5013 + n_seg * STRIP_DT, 0.0137])
    return nd, origin, 0.01, data.reshape(-1), 1, U, prm, start, goal, np.zeros(2)


# ---- what each case must show through the capacity export (cap_log of CapacityLog)
def check_first_growth_after(log, op):
    """no growth in the first plan; the first growth happens in the plan right after `op` ("block" / "clear")"""
    assert log[0]["op"] == "plan" and log[0]["grows"] == 0, log[0]
    i = next(k for k, c in enumerate(log) if c["grows"] > 0)
    assert log[i]["op"] == "plan" and log[i - 1]["op"] == op, [(c["op"], c["grows"]) for c in log[:i + 1]]
    return i


def check_reroot_growth(log, init_nodes, nU):
    """getSubStateSpace resizes the pool to (stored edges + 16) + |U| records, drops nodes from hm_ (their records stay), and
    a later plan doubles every array: the key table is rebuilt with the dropped records in it and some of them are reset in
    place when the plan reaches their keys again"""
    k = next(i for i, c in enumerate(log) if c["op"] == "sub")
    sub = log[k]
    assert all(c["grows"] == 0 for c in log[:k + 1]), [(c["op"], c["grows"]) for c in log[:k + 1]]
    assert sub["cap_pred"] == sub["n_nodes_physical"] * nU + 16 + nU, sub
    assert sub["hm"] < sub["n_nodes_physical"] == log[k - 1]["n_nodes_physical"], sub
    j = next(i for i, c in enumerate(log) if c["grows"] > 0)
    grown = log[j]
    assert j > k and grown["op"] == "plan", (j, k)
    assert grown["cap_pred"] == sub["cap_pred"] << grown["grows"], grown
    assert grown["cap_nodes"] == init_nodes << grown["grows"], grown
    assert grown["hm"] - sub["hm"] > grown["n_nodes_physical"] - sub["n_nodes_physical"], (sub, grown)  # re-created in place


def check_pred_only_growth(log, init_nodes):
    """the node arrays doubled although the node records never came near their initial size"""
    last = log[-1]
    assert last["grows"] >= 1 and last["cap_nodes"] == init_nodes << last["grows"], last
    assert max(c["n_nodes_physical"] for c in log) < init_nodes


def check_doublings(log, init_nodes):
    """capacity is the initial size doubled `grows` times, and it grew wherever the node records outgrew the initial size"""
    last = log[-1]
    assert last["cap_nodes"] == init_nodes << last["grows"], last
    assert last["n_nodes_physical"] <= last["cap_nodes"]
    if peak(log)[0] > init_nodes:
        assert last["grows"] >= 1, last
