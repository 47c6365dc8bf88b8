"""Multi-GPU sharding of a query batch: one process per GPU, torch.distributed for the plumbing.

The path shards by query (plans are independent and read-only on the map, SURVEY.md §8e).  There are exactly
two collectives on the data path: one broadcast of the voxel grid per map, and one gather of fixed-stride result
records per batch (plus, at set-up, one broadcast of the query list when only one rank holds it).  Within one plan
there is nothing to shard.

Works with backend "nccl" (GPU tensors, NVLink/NVSwitch) and "gloo" (CPU tensors; used by the CPU tests with a
stand-in planner, since libmplb has no CPU path), and without a process group at all (world size 1).
"""
import numpy as np
import torch
import torch.distributed as dist

from . import _lib


def _rank_world():
    if dist.is_available() and dist.is_initialized():
        return dist.get_rank(), dist.get_world_size()
    return 0, 1


def shard_indices(n, rank, world):
    """Query i goes to rank i mod world (static striping: neighbouring queries have unrelated cost)."""
    return np.arange(rank, n, world)


def broadcast_map(origin, dim, res, data, device, src=0):
    """Rank `src` supplies the map; every rank returns (origin, dim, res, grid tensor on `device`).
    One broadcast of a small header and one of the int8 grid."""
    rank, world = _rank_world()
    if world == 1:
        dimv = np.asarray(dim, dtype=np.int32)
        grid = torch.as_tensor(np.ascontiguousarray(data, dtype=np.int8).reshape(-1)).to(device)
        return np.asarray(origin, dtype=np.float64).copy(), dimv, float(res), grid
    hdr = torch.zeros(8, dtype=torch.float64, device=device)
    if rank == src:
        nd = len(dim)
        hdr[0] = nd
        hdr[1:1 + nd] = torch.as_tensor(np.asarray(origin, dtype=np.float64))
        hdr[4:4 + nd] = torch.as_tensor(np.asarray(dim, dtype=np.float64))
        hdr[7] = res
    dist.broadcast(hdr, src)
    h = hdr.cpu().numpy()
    nd = int(h[0])
    origin, dimv, res = h[1:1 + nd].copy(), h[4:4 + nd].astype(np.int32), float(h[7])
    ncell = int(np.prod(dimv.astype(np.int64)))
    if rank == src:
        grid = torch.as_tensor(np.ascontiguousarray(data, dtype=np.int8).reshape(-1)).to(device)
    else:
        grid = torch.empty(ncell, dtype=torch.int8, device=device)
    dist.broadcast(grid, src)
    return origin, dimv, res, grid


def gather_results(local_results, local_actions, n_total, max_seg, device, dst=0):
    """Gather per-rank result records (and action rows) to rank `dst`, restoring global query order.
    local_results: numpy structured array (RESULT_DTYPE) for queries shard_indices(n_total, rank, world).
    Returns (results[n_total], actions[n_total, max_seg]) on dst, (None, None) elsewhere."""
    rank, world = _rank_world()
    if world == 1:
        acts = np.ascontiguousarray(local_actions, dtype=np.int32) if max_seg else np.full((n_total, 0), -1, dtype=np.int32)
        return local_results, acts
    per = (n_total + world - 1) // world
    rec = _lib.RESULT_DTYPE.itemsize
    row = rec + 4 * max_seg
    buf = np.zeros((per, row), dtype=np.uint8)
    k = len(local_results)
    buf[:k, :rec] = local_results.view(np.uint8).reshape(k, rec)
    if max_seg:
        buf[:k, rec:] = np.ascontiguousarray(local_actions, dtype=np.int32).view(np.uint8).reshape(k, 4 * max_seg)
    t = torch.as_tensor(buf).to(device)
    outs = [torch.empty_like(t) for _ in range(world)] if rank == dst else None
    dist.gather(t, outs, dst)  # NCCL: grouped send/recv to dst; gloo: native gather
    if rank != dst:
        return None, None
    results = np.zeros(n_total, dtype=_lib.RESULT_DTYPE)
    actions = np.full((n_total, max_seg), -1, dtype=np.int32)
    for r in range(world):
        idx = shard_indices(n_total, r, world)
        b = outs[r].cpu().numpy()[:len(idx)]
        results[idx] = np.ascontiguousarray(b[:, :rec]).view(_lib.RESULT_DTYPE).reshape(-1)
        if max_seg:
            actions[idx] = np.ascontiguousarray(b[:, rec:]).view(np.int32).reshape(len(idx), max_seg)
    return results, actions


class Comm:
    """libmplb's own NCCL communicator (include/mplb.h, mplb_comm_*): the map broadcast and the result gather of the
    sharded batch run inside the C ABI, so a C++ caller without Python gets the same path.  The 128-byte id of rank 0
    has to reach the other ranks out of band (here: torch.distributed, a file, an environment variable ...)."""

    def __init__(self, id_bytes, rank, nranks):
        import ctypes as C
        h = C.c_void_p()
        buf = np.frombuffer(bytes(id_bytes), dtype=np.uint8).copy()
        _lib.check(_lib.lib().mplb_comm_create(_lib.ptr(buf), int(rank), int(nranks), C.byref(h)))
        self._h, self.rank, self.size = h, int(rank), int(nranks)

    @staticmethod
    def unique_id():
        buf = np.zeros(128, dtype=np.uint8)
        _lib.check(_lib.lib().mplb_comm_unique_id(_lib.ptr(buf)))
        return buf.tobytes()

    @classmethod
    def from_process_group(cls, device):
        """Rank 0 creates the id, the default torch.distributed group carries it to the others (set-up plumbing only)."""
        rank, world = _rank_world()
        t = torch.zeros(128, dtype=torch.uint8, device=device)
        if rank == 0:
            t.copy_(torch.frombuffer(bytearray(cls.unique_id()), dtype=torch.uint8))
        if world > 1:
            dist.broadcast(t, 0)
        return cls(t.cpu().numpy().tobytes(), rank, world)

    def broadcast_map(self, dim, origin=None, ndim=None, res=0.0, data=None, root=0):
        """One ncclBroadcast of the grid: returns a planner.MapUtil on this rank's device."""
        import ctypes as C
        from .planner import MapUtil
        h = C.c_void_p()
        if self.rank == root:
            o = np.ascontiguousarray(origin, dtype=np.float64)
            nd = np.ascontiguousarray(ndim, dtype=np.int32)
            dt = np.ascontiguousarray(data, dtype=np.int8).reshape(-1)
            _lib.check(_lib.lib().mplb_comm_broadcast_map(self._h, root, int(dim), _lib.ptr(nd), _lib.ptr(o), float(res), _lib.ptr(dt),
                                                        C.byref(h)))
        else:
            _lib.check(_lib.lib().mplb_comm_broadcast_map(self._h, root, 0, None, None, 0.0, None, C.byref(h)))
        mu = MapUtil(0)
        mu._h = h
        mu.dim = len(mu._info_raw()[0])
        return mu

    def __del__(self):
        try:
            _lib.lib().mplb_comm_destroy(self._h)
        except Exception:
            pass


class ShardedBatchPlanner:
    """plan_batch over all ranks.

    Without `comm`: torch.distributed collectives (works on gloo for the CPU tests); `make_planner(origin, dim, res,
    grid_tensor)` builds this rank's planner on its device from the broadcast grid.
    With `comm` (a dist.Comm): the broadcast and the gather run inside libmplb (mplb_comm_broadcast_map,
    mplb_plan_batch_sharded, mplb_plan_stripe_gather_device); `make_planner(origin, dim, res, map_util)` then receives the
    ready planner.MapUtil instead of a tensor."""

    def __init__(self, make_planner, device, comm=None):
        self.make_planner = make_planner
        self.device = device
        self.planner = None
        self.comm = comm

    def _rw(self):
        """(rank, world): the communicator's when one is attached, else the default torch.distributed group's"""
        return (self.comm.rank, self.comm.size) if self.comm is not None else _rank_world()

    def set_map(self, origin=None, dim=None, res=None, data=None, src=0):
        if self.comm is not None:
            mu = self.comm.broadcast_map(len(dim) if dim is not None else 0, origin, dim, res if res is not None else 0.0, data, src)
            d, o, r = mu._info()
            self.planner = self.make_planner(o, d, r, mu)
            return o, d, r
        o, d, r, grid = broadcast_map(origin, dim, res, data, self.device, src)
        self._grid = grid  # keep the receive buffer alive until the planner has copied it
        self.planner = self.make_planner(o, d, r, grid)
        return o, d, r

    def set_cost_shaping(self, potential=None, region=None, src=0):
        """Install a potential map (int8 per cell, env_map::set_potential_map) and / or a search-region mask (one byte
        per cell, env_base::set_search_region) on every rank's planner: rank `src` supplies them (e.g. the map its own
        planner rewrote with updatePotentialMap), the others receive them with one broadcast each.  None on `src`
        clears that piece everywhere."""
        rank, world = self._rw()
        flags = torch.zeros(2, dtype=torch.int64, device=self.device)
        if rank == src:
            flags[0] = 0 if potential is None else int(np.asarray(potential).size)
            flags[1] = 0 if region is None else int(np.asarray(region).size)
        if world > 1:
            dist.broadcast(flags, src)
        n_pot, n_reg = (int(x) for x in flags.cpu().numpy())
        for n, arr, dtype, setter in ((n_pot, potential, np.int8, "setPotentialMap"), (n_reg, region, np.uint8, "setSearchRegionMask")):
            if n == 0:
                getattr(self.planner, setter)(None)
                continue
            tdt = torch.int8 if dtype == np.int8 else torch.uint8
            if rank == src:
                t = torch.as_tensor(np.ascontiguousarray(arr, dtype=dtype).reshape(-1)).to(self.device)
            else:
                t = torch.empty(n, dtype=tdt, device=self.device)
            if world > 1:
                dist.broadcast(t, src)
            getattr(self.planner, setter)(t.cpu().numpy())

    def broadcast_queries(self, starts, goals, src=0):
        """Rank `src` holds the query list; every rank returns it (one broadcast of the two waypoint arrays)."""
        rank, world = self._rw()
        if world == 1:
            return starts, goals
        n = len(starts)
        host = np.concatenate([starts.view(np.uint8).reshape(n, -1), goals.view(np.uint8).reshape(n, -1)]) if rank == src else None
        t = torch.as_tensor(host).to(self.device) if rank == src else torch.empty((2 * n, _lib.WAYPOINT_DTYPE.itemsize), dtype=torch.uint8,
                                                                                 device=self.device)
        dist.broadcast(t, src)
        b = t.cpu().numpy()
        return (np.ascontiguousarray(b[:n]).view(_lib.WAYPOINT_DTYPE).reshape(-1),
                np.ascontiguousarray(b[n:]).view(_lib.WAYPOINT_DTYPE).reshape(-1))

    # ---- device-resident stripes (inputs and outputs stay in HBM; the gather moves device buffers)
    def make_device_buffers(self, n_total, max_seg, dst=0):
        rank, world = self._rw()
        per = (n_total + world - 1) // world
        b = {"res": torch.zeros(per, _lib.RESULT_DTYPE.itemsize, dtype=torch.uint8, device=self.device),
             "act": torch.zeros(per, max(max_seg, 1), dtype=torch.int32, device=self.device), "gres": None, "gact": None}
        if world > 1 and rank == dst:
            b["gres"] = [torch.empty_like(b["res"]) for _ in range(world)]
            b["gact"] = [torch.empty_like(b["act"]) for _ in range(world)]
        return b

    def plan_stripe_device(self, d_starts, d_goals, n_local, bufs, max_seg, stream=None, dst=0):
        """This rank's stripe (device tensors of waypoint records) through mplb_plan_batch_device, then the one gather of
        result records and action rows on `dst`."""
        rank, world = self._rw()
        if self.comm is not None:
            import ctypes as C
            vp = lambda x: C.c_void_p(int(x)) if x else None  # noqa: E731
            _lib.check(_lib.lib().mplb_plan_stripe_gather_device(
                self.planner._h, self.comm._h, vp(d_starts.data_ptr()), vp(d_goals.data_ptr()), n_local, bufs["res"].shape[0],
                vp(bufs["res"].data_ptr()), vp(bufs["act"].data_ptr() if max_seg else 0), max_seg, dst,
                vp(stream.cuda_stream if stream is not None else 0)))
            return
        self.planner.plan_batch_device(d_starts.data_ptr(), d_goals.data_ptr(), n_local, bufs["res"].data_ptr(),
                                       bufs["act"].data_ptr() if max_seg else 0, 0, max_seg,
                                       stream.cuda_stream if stream is not None else 0)
        if world > 1:
            dist.gather(bufs["res"], bufs["gres"], dst=dst)
            dist.gather(bufs["act"], bufs["gact"], dst=dst)

    # ---- one batch in flight per planner (mplb_plan_stripe_begin / _end, mplb_plan_batch_sharded_begin / _end): two
    # ShardedBatchPlanner objects on one map and one communicator, alternating, overlap the drain of a launch with the
    # start of the next one
    def begin_stripe_device(self, d_starts, d_goals, n_local, bufs, max_seg, stream=None):
        import ctypes as C
        vp = lambda x: C.c_void_p(int(x)) if x else None  # noqa: E731
        _lib.check(_lib.lib().mplb_plan_stripe_begin(self.planner._h, vp(d_starts.data_ptr()), vp(d_goals.data_ptr()), n_local,
                                                   vp(bufs["res"].data_ptr()), vp(bufs["act"].data_ptr() if max_seg else 0), max_seg,
                                                   vp(stream.cuda_stream if stream is not None else 0)))

    def end_stripe_device(self, bufs, dst=0):
        _lib.check(_lib.lib().mplb_plan_stripe_end(self.planner._h, self.comm._h, bufs["res"].shape[0], dst))

    def begin_batch(self, starts, goals, max_seg=64):
        self._pending = (len(starts), max_seg)
        _lib.check(_lib.lib().mplb_plan_batch_sharded_begin(self.planner._h, self.comm._h, _lib.ptr(starts), _lib.ptr(goals), len(starts),
                                                          max_seg))

    def end_batch(self, dst=0):
        n, max_seg = self._pending
        rank, world = self._rw()
        res = np.zeros(n, dtype=_lib.RESULT_DTYPE) if rank == dst else None
        acts = np.full((n, max_seg), -1, dtype=np.int32) if (rank == dst and max_seg) else None
        _lib.check(_lib.lib().mplb_plan_batch_sharded_end(self.planner._h, self.comm._h, n, _lib.ptr(res), _lib.ptr(acts), dst))
        return res, acts

    def unstripe(self, bufs, n_total, max_seg):
        """On the gather destination: (results[n_total], actions[n_total, max_seg]) in global query order."""
        rank, world = self._rw()
        results = np.zeros(n_total, dtype=_lib.RESULT_DTYPE)
        actions = np.full((n_total, max_seg), -1, dtype=np.int32)
        if self.comm is not None:
            _lib.check(_lib.lib().mplb_comm_unstripe(self.comm._h, n_total, bufs["res"].shape[0], max_seg, _lib.ptr(results),
                                                   _lib.ptr(actions) if max_seg else None))
            return results, actions
        parts = zip(bufs["gres"], bufs["gact"]) if world > 1 else [(bufs["res"], bufs["act"])]
        for r, (tr, ta) in enumerate(parts):
            idx = shard_indices(n_total, r, world)
            results[idx] = np.ascontiguousarray(tr.cpu().numpy()[:len(idx)]).view(_lib.RESULT_DTYPE).reshape(-1)
            if max_seg:
                actions[idx] = ta.cpu().numpy()[:len(idx), :max_seg]
        return results, actions

    def plan_batch_local(self, starts_local, goals_local, n_total, max_seg=64, dst=0):
        """Host buffers holding only this rank's stripe (queries shard_indices(n_total, rank, world))."""
        res, acts, _ = self.planner.plan_batch(starts_local, goals_local, max_seg=max_seg)
        return gather_results(res, acts, n_total, max_seg, self.device, dst)

    def plan_batch(self, starts, goals, max_seg=64, dst=0):
        """starts/goals: full arrays on every rank (host, WAYPOINT_DTYPE). Each rank plans its stripe."""
        rank, world = self._rw()
        if self.comm is not None:
            n = len(starts)
            res = np.zeros(n, dtype=_lib.RESULT_DTYPE) if rank == dst else None
            acts = np.full((n, max_seg), -1, dtype=np.int32) if (rank == dst and max_seg) else None
            _lib.check(_lib.lib().mplb_plan_batch_sharded(self.planner._h, self.comm._h, _lib.ptr(starts), _lib.ptr(goals), n,
                                                        _lib.ptr(res), _lib.ptr(acts), max_seg, dst))
            return res, acts
        idx = shard_indices(len(starts), rank, world)
        res, acts, _ = self.planner.plan_batch(np.ascontiguousarray(starts[idx]), np.ascontiguousarray(goals[idx]),
                                               max_seg=max_seg)
        return gather_results(res, acts, len(starts), max_seg, self.device, dst)


# ---- a fleet of LPA* replanners sharded over ranks (mplb_fleet_map_edit / mplb_fleet_plan, DESIGN.md section 6.1): robot i lives
# on rank i mod N; every rank holds a replica of the shared map.  A replan cycle is the single-device fleet cycle with the map
# edit and the plan distributed: every replica applies the concatenation of all robots' edits in robot order, and the plans
# come back to one root in robot order.

def _rows3(cells):
    """rows of 2 or 3 ints -> rows of 3 int32 (the third 0 in 2D)"""
    c = np.asarray(cells, dtype=np.int32).reshape(len(cells), -1) if len(cells) else np.zeros((0, 3), dtype=np.int32)
    out = np.zeros((len(c), 3), dtype=np.int32)
    out[:, :c.shape[1]] = c
    return out


def pack_edits(cells_local):
    """This rank's robots' edit lists -> (per-robot row counts int64, rows int32 [k, 3]): the send payload of the exchange."""
    c3 = [np.asarray(c, dtype=np.int32).reshape(-1, 3) for c in cells_local]
    counts = np.array([len(c) for c in c3], dtype=np.int64)
    rows = np.concatenate(c3) if c3 else np.zeros((0, 3), dtype=np.int32)
    return counts, np.ascontiguousarray(rows, dtype=np.int32)


def merge_edits(parts, n_total):
    """The received payloads (counts, rows) of ranks 0 .. N-1 -> the concatenation c_0 || ... || c_{R-1} in robot order (robot i
    = the (i / N)-th robot of rank i mod N) and its R + 1 offsets.  Independent of the order the payloads arrived in."""
    world = len(parts)
    starts = [np.concatenate([[0], np.cumsum(c)]).astype(np.int64) for c, _ in parts]
    lists, offs = [], np.zeros(n_total + 1, dtype=np.int64)
    for i in range(n_total):
        r, k = i % world, i // world
        lists.append(parts[r][1][starts[r][k]:starts[r][k + 1]])
        offs[i + 1] = offs[i] + len(lists[-1])
    cells = np.concatenate(lists) if lists else np.zeros((0, 3), dtype=np.int32)
    return np.ascontiguousarray(cells, dtype=np.int32).reshape(-1, 3), offs


def exchange_edits(cells_local, n_total, device):
    """torch.distributed stand-in of mplb_fleet_map_edit's exchange (gloo on a CPU box): one all-gather of the payload sizes,
    one of the payloads (padded to the largest), then merge_edits.  Returns (cells [T, 3] int32, offsets [R + 1]) on every rank."""
    rank, world = _rank_world()
    counts, rows = pack_edits(cells_local)
    if world == 1:
        return merge_edits([(counts, rows)], n_total)
    words = np.concatenate([counts.astype(np.int32), rows.reshape(-1)]).astype(np.int32)
    size = torch.tensor([len(counts), len(rows)], dtype=torch.int64, device=device)
    sizes = [torch.empty_like(size) for _ in range(world)]
    dist.all_gather(sizes, size)
    sizes = [tuple(int(v) for v in s.cpu().numpy()) for s in sizes]
    width = max(max(n + 3 * k for n, k in sizes), 1)
    buf = torch.zeros(width, dtype=torch.int32, device=device)
    buf[:len(words)] = torch.as_tensor(words)
    bufs = [torch.empty_like(buf) for _ in range(world)]
    dist.all_gather(bufs, buf)
    parts = []
    for (n, k), b in zip(sizes, bufs):
        w = b.cpu().numpy()
        parts.append((w[:n].astype(np.int64), w[n:n + 3 * k].reshape(k, 3)))
    return merge_edits(parts, n_total)


class ShardedFleet:
    """This rank's robots of a fleet of R LPA* replanners (robot i on rank i mod N) and one replan cycle over all ranks.

    planners: this rank's MapPlanner objects (LPA* on), robots rank, rank + N, ... in that order.  map_util: this rank's replica
    of the shared map (None for a fleet whose robots each own a map: then only the plan is collective).  With `comm` (a dist.Comm)
    the edit and the gather run inside libmplb on the device; without it the default torch.distributed group carries them
    (gloo works), and `_set_cells` / `_plan_local` do the rank-local work, which a CPU test may replace with stand-ins."""

    def __init__(self, planners, n_total, map_util=None, comm=None, device=None):
        self.planners, self.n_total, self.map_util, self.comm, self.device = list(planners), int(n_total), map_util, comm, device
        self.rank, self.world = (comm.rank, comm.size) if comm is not None else _rank_world()
        self.local = shard_indices(self.n_total, self.rank, self.world)
        if len(self.local) != len(self.planners):
            raise ValueError("rank %d of %d holds robots %s of %d, not %d planners" % (self.rank, self.world, list(self.local),
                                                                                      self.n_total, len(self.planners)))
        self.cells, self.offsets = np.zeros((0, 3), dtype=np.int32), np.zeros(self.n_total + 1, dtype=np.int64)
        self._d_all = self._d_off = None
        self._T = 0

    # ---- step 1 and 2: every robot's edit reaches every replica, in robot order
    def map_edit(self, cells_local, value):
        """cells_local[k]: the edit of this rank's k-th robot (rows of 2 or 3 ints).  Every replica receives
        mplb_map_set_cells(c_0 || ... || c_{R-1}, value).  Returns the row count T of that concatenation, which stays on the
        device for update(); edit_cells() / edit_offsets() copy it and its R + 1 offsets to the host."""
        c3 = [_rows3(c) for c in cells_local]
        if self.comm is None:
            self.cells, self.offsets = exchange_edits(c3, self.n_total, self.device)
            self._T = len(self.cells)
            if self._T:
                self._set_cells(self.cells, value)
            return self._T
        import ctypes as C
        counts, rows = pack_edits(c3)
        offs = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
        d_rows = torch.as_tensor(rows).to(self.device) if len(rows) else None
        vp = lambda t: C.c_void_p(t.data_ptr()) if t is not None else None  # noqa: E731
        if self._d_off is None:
            self._d_off = torch.zeros(self.n_total + 1, dtype=torch.int64, device=self.device)
            self._d_all = torch.zeros((1024, 3), dtype=torch.int32, device=self.device)
        stream = C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)  # the stream d_rows was written on
        for _ in range(2):  # every rank holds the same cap, so T > cap on one rank is T > cap on all: all grow and call again
            total = _lib.check(_lib.lib().mplb_fleet_map_edit(self.comm._h, self.map_util._h, vp(d_rows), _lib.ptr(offs), len(c3),
                                                             int(value), vp(self._d_all), vp(self._d_off), self._d_all.shape[0], stream))
            if total <= self._d_all.shape[0]:
                break
            self._d_all = torch.zeros((total, 3), dtype=torch.int32, device=self.device)
        self._T = total
        return total

    def edit_cells(self):
        """the last map_edit's concatenation c_0 || ... || c_{R-1}, rows of 3 int32 on the host"""
        return self.cells if self.comm is None else self._d_all[:self._T].cpu().numpy()

    def edit_offsets(self):
        """its R + 1 offsets on the host: robot i's rows are edit_cells()[offsets[i]:offsets[i + 1]]"""
        return self.offsets if self.comm is None else self._d_off.cpu().numpy()

    def _set_cells(self, cells, value):
        self.map_util.setCells(cells, value)

    # ---- steps 3 to 6: rank-local, except the gather of the plans
    def links(self):
        from .planner import MapPlanner
        return MapPlanner.getLinkedNodesBatch(self.planners)

    def update(self, blocked, selection=None):
        """updateBlockedNodes (blocked) / updateClearedNodes of this rank's robots: by default every robot receives the whole
        concatenation of the last map_edit; selection[k] (rows of ints) replaces it for this rank's k-th robot."""
        from .planner import MapPlanner
        if selection is not None:
            return MapPlanner._update_batch(self.planners, selection, blocked)
        n, T = len(self.planners), self._T
        if self.comm is None or n == 0:
            return MapPlanner._update_batch(self.planners, [self.cells] * n, blocked)
        import ctypes as C
        # The batched update gives entry k the rows offsets[k] .. offsets[k+1]-1, so one list cannot be shared by several
        # entries: the device concatenation is repeated once per local robot (n T rows of 12 B), and entry k reads copy k.
        rep = self._d_all[:T].repeat(n, 1) if T else None
        offs = (np.arange(n + 1, dtype=np.int64) * T)
        torch.cuda.current_stream(self.device).synchronize()  # the update reads `rep` on the default stream
        visited = np.zeros(n, dtype=np.int32)
        _lib.check(_lib.lib().mplb_lpa_update_nodes_batch_device(MapPlanner._handles(self.planners), n, int(blocked),
                                                                 C.c_void_p(rep.data_ptr()) if rep is not None else None,
                                                                 _lib.ptr(offs), _lib.ptr(visited)))
        return [int(v) for v in visited]

    def plan(self, starts_local, goals_local, max_seg=64, root=0):
        """planLPABatch of this rank's robots, gathered: (results[R], actions[R, max_seg]) in robot order on `root`, (None, None)
        elsewhere.  Every local planner keeps result(), traj_ and traj_cost_ as plan() does."""
        if self.comm is not None:
            from .planner import MapPlanner
            return MapPlanner.planLPAFleet(self.comm, self.planners, self.n_total, starts_local, goals_local, max_seg, root)
        res, acts = self._plan_local(starts_local, goals_local, max_seg)
        return gather_results(res, acts, self.n_total, max_seg, self.device, root)

    def _plan_local(self, starts, goals, max_seg):
        from .planner import MapPlanner
        n = len(self.planners)
        MapPlanner.planLPABatch(self.planners, starts, goals)
        res = np.zeros(n, dtype=_lib.RESULT_DTYPE)
        acts = np.full((n, max_seg), -1, dtype=np.int32)
        for k, pl in enumerate(self.planners):
            res[k] = pl.result()
            if int(res[k]["status"]) == 0 and max_seg:
                a = pl.getActions()[:max_seg]
                acts[k, :len(a)] = a
        return res, acts

    def sub_state_space(self, time_steps_local):
        from .planner import MapPlanner
        return MapPlanner.getSubStateSpaceBatch(self.planners, time_steps_local)

    def cycle(self, cells_local, value, starts_local, goals_local, time_steps_local, selection=None, max_seg=64, root=0):
        """One replan cycle: edit, getLinkedNodes, update, plan, getSubStateSpace.  Returns the gathered plan (root) and sizes."""
        self.map_edit(cells_local, value)
        self.links()
        self.update(value == 100, selection)
        out = self.plan(starts_local, goals_local, max_seg, root)
        return out, self.sub_state_space(time_steps_local)
