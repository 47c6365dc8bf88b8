"""VoxelGrid of planning_ros_utils (include/planning_ros_utils/voxel_grid.h, src/mapping_utils/voxel_grid.cpp) over the C ABI.

Both int8 grids live on the GPU; member names follow the reference so that callers read like cloud_to_map.cpp and
map_replanner_node.cpp.  Points are rows of 3 (x, y, z); cells are rows of 3 ints.  See include/mplb.h for the behaviour the
library defines where the reference is undefined.
"""
import ctypes as C

import numpy as np

from ._lib import MplbError, check, lib, ptr
from .planner import VoxelMapUtil


def _rows3(a, dtype):
    a = np.ascontiguousarray(a, dtype=dtype)
    if a.size == 0:
        return a.reshape(0, 3)
    if a.ndim != 2 or a.shape[1] != 3:
        raise MplbError("expected rows of 3")
    return a


class VoxelGrid:
    """VoxelGrid(origin, dim, res) (voxel_grid.cpp:3-10): res is a float as in the reference."""

    def __init__(self, origin, dim, res):
        self._h = None
        o = np.ascontiguousarray(origin, dtype=np.float64)
        d = np.ascontiguousarray(dim, dtype=np.float64)
        h = C.c_void_p()
        check(lib().mplb_voxel_grid_create(ptr(o), ptr(d), float(np.float32(res)), C.byref(h)))
        self._h = h

    def __del__(self):
        try:
            if self._h is not None:
                lib().mplb_voxel_grid_destroy(self._h)
                self._h = None
        except Exception:
            pass

    # ---- geometry
    def info(self):
        """(dim_ int[3], origin_ int[3], origin_d_ float64[3], res_ as float32)"""
        dim, ori = np.zeros(3, dtype=np.int32), np.zeros(3, dtype=np.int32)
        ori_d, res = np.zeros(3, dtype=np.float64), C.c_float()
        check(lib().mplb_voxel_grid_get_info(self._h, ptr(dim), ptr(ori), ptr(ori_d), C.byref(res)))
        return dim, ori, ori_d, np.float32(res.value)

    def allocate(self, new_dim_d, new_ori_d):  # voxel_grid.cpp:129-172
        d = np.ascontiguousarray(new_dim_d, dtype=np.float64)
        o = np.ascontiguousarray(new_ori_d, dtype=np.float64)
        changed = C.c_int32()
        check(lib().mplb_voxel_grid_allocate(self._h, ptr(d), ptr(o), C.byref(changed)))
        return bool(changed.value)

    def _ncell(self):
        return int(np.prod(self.info()[0].astype(np.int64)))

    # ---- edits
    def clear(self, nx=None, ny=None):
        """clear() (both grids free) or clear(nx, ny) (one column of map_)"""
        if nx is None:
            check(lib().mplb_voxel_grid_clear(self._h))
        else:
            self.clearColumns([(nx, ny, 0)])

    def clearColumns(self, cells):
        c = _rows3(cells, np.int32)
        check(lib().mplb_voxel_grid_clear_columns(self._h, ptr(c), len(c)))

    def fill(self, nx, ny, nz=None):
        """fill(nx, ny) (a column) or fill(nx, ny, nz) (one cell) of map_"""
        if nz is None:
            self.fillColumns([(nx, ny, 0)])
        else:
            self.fillCells([(nx, ny, nz)])

    def fillColumns(self, cells):
        c = _rows3(cells, np.int32)
        check(lib().mplb_voxel_grid_fill(self._h, ptr(c), len(c), 1))

    def fillCells(self, cells):
        c = _rows3(cells, np.int32)
        check(lib().mplb_voxel_grid_fill(self._h, ptr(c), len(c), 0))

    def decay(self):  # voxel_grid.cpp:214-225
        check(lib().mplb_voxel_grid_decay(self._h))

    def addCloud(self, pts, ns=None):
        """addCloud(pts) (voxel_grid.cpp:174-180), or addCloud(pts, ns) (:182-199) which returns new_obs as int32 rows"""
        p = _rows3(pts, np.float64)
        if ns is None:
            check(lib().mplb_voxel_grid_add_cloud(self._h, ptr(p), len(p)))
            return None
        n3 = _rows3(ns, np.int32)
        cap = min(len(p) * len(n3), self._ncell())  # one call emits a cell at most once
        out = np.zeros((max(cap, 1), 3), dtype=np.int32)
        n = check(lib().mplb_voxel_grid_add_cloud_inflated(self._h, ptr(p), len(p), ptr(n3), len(n3), ptr(out), cap))
        return out[:n].copy()

    @staticmethod
    def _device_points(pts, n):
        """(pointer, n, fp32) of a CUDA (N, 3) float32/float64 tensor or of a raw device pointer (n required, fp64 assumed
        unless a (pointer, fp32) pair is given)"""
        if hasattr(pts, "data_ptr"):
            if not pts.is_cuda or pts.dim() != 2 or pts.shape[1] != 3 or not pts.is_contiguous():
                raise MplbError("expected a contiguous CUDA tensor of shape (N, 3)")
            name = str(pts.dtype)
            if name not in ("torch.float32", "torch.float64"):
                raise MplbError("points must be float32 or float64")
            return pts.data_ptr(), int(pts.shape[0]) if n is None else int(n), int(name == "torch.float32")
        if isinstance(pts, tuple):
            p, fp32 = pts
        else:
            p, fp32 = pts, 0
        if n is None:
            raise MplbError("n is required with a raw device pointer")
        return int(p), int(n), int(fp32)

    @staticmethod
    def _stream(pts, stream):
        if stream is not None:
            return C.c_void_p(int(getattr(stream, "cuda_stream", stream)) or None)
        if hasattr(pts, "data_ptr"):
            import torch
            return C.c_void_p(torch.cuda.current_stream(pts.device).cuda_stream or None)
        return None

    def addCloudDevice(self, pts, n=None, stream=None, ns=None, out=None):
        """addCloud on points already on the device.  With ns, new_obs goes to `out` (a CUDA int32 tensor of shape (cap, 3))
        and the row count is returned, or, when out is None, new_obs is returned as a CUDA int32 tensor."""
        p, cnt, fp32 = self._device_points(pts, n)
        s = self._stream(pts, stream)
        if ns is None:
            check(lib().mplb_voxel_grid_add_cloud_device(self._h, C.c_void_p(p), cnt, fp32, s))
            return None
        n3 = _rows3(ns, np.int32)
        if out is not None:
            return check(lib().mplb_voxel_grid_add_cloud_inflated_device(self._h, C.c_void_p(p), cnt, fp32, ptr(n3), len(n3),
                                                                        C.c_void_p(out.data_ptr()), int(out.shape[0]), s))
        import torch
        cap = min(cnt * len(n3), self._ncell())  # one call emits a cell at most once
        buf = torch.empty((max(cap, 1), 3), dtype=torch.int32, device=getattr(pts, "device", "cuda"))
        k = check(lib().mplb_voxel_grid_add_cloud_inflated_device(self._h, C.c_void_p(p), cnt, fp32, ptr(n3), len(n3),
                                                                 C.c_void_p(buf.data_ptr()), cap, s))
        return buf[:k]

    def setChunkPoints(self, n):
        """points per internal pass of the inflated insertion (0 = default); results do not depend on it"""
        check(lib().mplb_voxel_grid_set_chunk_points(self._h, int(n)))

    # ---- outputs
    def _cloud(self, call, *args):
        n = check(call(self._h, *args, None, 0))
        out = np.zeros((max(n, 1), 3), dtype=np.float64)
        n2 = check(call(self._h, *args, ptr(out), n))
        assert n2 == n
        return out[:n]

    def getCloud(self):  # voxel_grid.cpp:18-29
        return self._cloud(lib().mplb_voxel_grid_get_cloud)

    def getLocalCloud(self, pos, ori, dim):  # voxel_grid.cpp:47-69
        a = [np.ascontiguousarray(v, dtype=np.float64) for v in (pos, ori, dim)]
        return self._cloud(lib().mplb_voxel_grid_get_local_cloud, *[ptr(v) for v in a])

    def getMapData(self, inflated=False):
        """data of getMap() / getInflatedMap() (voxel_grid.cpp:71-127): 100 / 0, x fastest"""
        out = np.zeros(max(self._ncell(), 1), dtype=np.int8)
        check(lib().mplb_voxel_grid_get_map(self._h, int(bool(inflated)), ptr(out), out.size))
        return out[:self._ncell()]

    def getMap(self):
        """planning_ros_msgs::VoxelMap fields as a dict: origin, dim, resolution (float32), data"""
        dim, _, ori_d, res = self.info()
        return dict(origin=ori_d, dim=dim, resolution=res, data=self.getMapData(False))

    def getInflatedMap(self):
        dim, _, ori_d, res = self.info()
        return dict(origin=ori_d, dim=dim, resolution=res, data=self.getMapData(True))

    def writeMap(self, map_util, inflated=False):
        """setMap(map_util, getMap()) on the device: map_util must already have the grid's geometry"""
        check(lib().mplb_voxel_grid_write_map(self._h, int(bool(inflated)), map_util._h))

    def toMapUtil(self, inflated=False):
        """a new VoxelMapUtil holding getMap() / getInflatedMap(), built device to device"""
        mu = VoxelMapUtil()
        h = C.c_void_p()
        check(lib().mplb_voxel_grid_create_map(self._h, int(bool(inflated)), C.byref(h)))
        mu._h = h
        return mu

