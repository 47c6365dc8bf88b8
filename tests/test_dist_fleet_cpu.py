"""world_size-2 gloo test of the sharded fleet's plumbing (mpl_ros_b200.dist.ShardedFleet without a libmplb communicator): the
exchange of the cycle's map edits and the gather of the cycle's plans.  Robot i lives on rank i mod 2.  libmplb has no CPU path,
so each rank applies the edit to a host grid and "plans" with a stand-in whose records and action rows name the robot; the
concatenation, its offsets, every replica and the gathered records must equal a single-process run in robot order."""
import os
import socket
import sys

import numpy as np
import torch.multiprocessing as tmp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ND = (20, 16, 4)
# (R, which robots edit): R < N, R not divisible by N, every robot, only rank 1's robots, a rank whose robots contribute
# nothing, no edits at all
CASES = [(1, "all"), (5, "all"), (6, "all"), (6, "odd"), (7, "even"), (4, "none")]


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def robot_edit(case, i):
    """robot i's cell list in case `case`: seeded, of varying length; empty where the case says so and for every third robot"""
    R, who = CASES[case]
    if who == "none" or (who == "odd" and i % 2 == 0) or (who == "even" and i % 2 == 1) or i % 3 == 2:
        return np.zeros((0, 3), dtype=np.int32)
    rng = np.random.default_rng(100 * case + i)
    n = int(rng.integers(1, 9))
    return np.stack([rng.integers(0, d, n) for d in ND], axis=1).astype(np.int32)


def _fleet(*args, **kw):
    """ShardedFleet with the rank-local work done on the host: a grid as the map replica, records naming the robot (the class is
    made here because a spawned worker imports the package only after it has set up its path)"""
    from mpl_ros_b200 import _lib, dist as mdist

    class Fleet(mdist.ShardedFleet):
        def _set_cells(self, cells, value):
            self.map_util[cells[:, 0] + ND[0] * cells[:, 1] + ND[0] * ND[1] * cells[:, 2]] = value

        def _plan_local(self, starts, goals, max_seg):
            res = np.zeros(len(self.planners), dtype=_lib.RESULT_DTYPE)
            acts = np.full((len(self.planners), max_seg), -1, dtype=np.int32)
            for k, i in enumerate(self.planners):
                res[k]["pops"], res[k]["n_seg"], res[k]["cost"] = i, i % 4, 0.5 * i
                acts[k, :i % 4] = i
            return res, acts
    return Fleet(*args, **kw)


def single_process(case):
    R, _ = CASES[case]
    lists = [robot_edit(case, i) for i in range(R)]
    cells = np.concatenate(lists) if lists else np.zeros((0, 3), dtype=np.int32)
    offs = np.concatenate([[0], np.cumsum([len(c) for c in lists])]).astype(np.int64)
    grid = np.zeros(int(np.prod(ND)), dtype=np.int8)
    if len(cells):
        grid[cells[:, 0] + ND[0] * cells[:, 1] + ND[0] * ND[1] * cells[:, 2]] = 100
    return cells.reshape(-1, 3), offs, grid


def _worker(rank, world, port, out_path):
    sys.path.insert(0, ROOT)
    import torch
    import torch.distributed as dist
    from mpl_ros_b200 import dist as mdist
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    out = {}
    for case, (R, _) in enumerate(CASES):
        mine = list(mdist.shard_indices(R, rank, world))
        fleet = _fleet(mine, R, np.zeros(int(np.prod(ND)), dtype=np.int8), device=torch.device("cpu"))
        T = fleet.map_edit([robot_edit(case, i) for i in mine], 100)
        cells, offs = fleet.edit_cells(), fleet.edit_offsets()
        assert T == len(cells)
        res, acts = fleet.plan(None, None, max_seg=4)
        out["cells%d" % case], out["offs%d" % case], out["grid%d_%d" % (case, rank)] = cells, offs, fleet.map_util
        if rank == 0:
            out["res%d" % case], out["acts%d" % case] = res.view(np.uint8), acts
        else:
            assert res is None and acts is None
    grids = {k: v for k, v in out.items() if k.startswith("grid")}
    gathered = [None] * world
    dist.all_gather_object(gathered, grids)
    if rank == 0:
        for g in gathered:
            out.update(g)
        np.savez(out_path, **out)
    else:  # every rank holds the same concatenation
        z = {k: v for k, v in out.items() if k.startswith(("cells", "offs"))}
        np.savez(out_path + ".r1.npz", **z)
    dist.barrier()
    dist.destroy_process_group()


def test_sharded_fleet_exchange_and_gather_gloo(tmp_path):
    out = str(tmp_path / "fleet.npz")
    tmp.spawn(_worker, args=(2, _free_port(), out), nprocs=2, join=True)
    sys.path.insert(0, ROOT)
    from mpl_ros_b200 import _lib
    z, z1 = np.load(out), np.load(out + ".r1.npz")
    for case, (R, _) in enumerate(CASES):
        cells, offs, grid = single_process(case)
        for zz in (z, z1):
            assert np.array_equal(zz["cells%d" % case], cells), case
            assert np.array_equal(zz["offs%d" % case], offs), case
        for r in range(2):
            assert np.array_equal(z["grid%d_%d" % (case, r)], grid), (case, r)
        res = z["res%d" % case].view(_lib.RESULT_DTYPE).reshape(-1)
        assert np.array_equal(res["pops"], np.arange(R)) and np.array_equal(res["n_seg"], np.arange(R) % 4), case
        acts = z["acts%d" % case]
        for i in range(R):
            assert np.array_equal(acts[i], [i if k < i % 4 else -1 for k in range(4)]), (case, i)
    assert len(z["cells3"]) > 0 and len(z["cells5"]) == 0


def test_merge_is_robot_ordered_and_independent_of_arrival():
    """merge_edits puts robot i's rows at the prefix of robots 0 .. i-1 whatever the payloads' order of arrival: the payload of
    rank r is always read from slot r"""
    from mpl_ros_b200 import dist as mdist
    for R, world in ((0, 3), (2, 3), (7, 3), (9, 4)):
        lists = [np.full((i % 3, 3), i, dtype=np.int32) for i in range(R)]
        parts = [mdist.pack_edits([lists[i] for i in mdist.shard_indices(R, r, world)]) for r in range(world)]
        cells, offs = mdist.merge_edits(parts, R)
        want = np.concatenate(lists) if R else np.zeros((0, 3), dtype=np.int32)
        assert np.array_equal(cells, want.reshape(-1, 3)) and list(offs) == [0] + list(np.cumsum([len(c) for c in lists]))
