"""Voxel down-sampling of raw scans on the GPU (d3f_voxel_down_sample): Open3D 0.7's voxel_down_sample, the input
stage of every reference entry point (datasets/ThreeDMatch.py:349 at 0.03 m, datasets/ETH.py:169 at 0.0625 m,
datasets/KITTI.py:314-315 at first_subsampling_dl, demo_registration.py:24 at 0.03 m), for all clouds of a stack at
once and bit-exact:

    min_b = min over the cloud's finite rows - v * 0.5;   i = (int)floor((p - min_b) / v)   (fp64, one rounding each)
    voxel point = fp64 sum of its rows in input order / count, rounded to fp32.

Deviations from Open3D: voxels come per cloud in ascending (iz, iy, ix) (Open3D: std::unordered_map order); the
output is fp32; rows with a non-finite coordinate are dropped; a voxel_size that is not finite and > 0 is a ValueError.

    pts, lens = voxel_down_sample(raw_points, raw_lengths, 0.03)

encoder.GraphPipeline(..., voxel_size=v) runs the same op in its static form at the head of the pyramid graph.
"""
import ctypes as C
import math
import numbers

import numpy as np
import torch

from . import _lib


def check_voxel_size(voxel_size, who):
    """The voxel size as the Python float (an IEEE double) the kernels use, or ValueError."""
    if not isinstance(voxel_size, numbers.Real) or isinstance(voxel_size, bool):
        raise ValueError("%s: voxel_size must be a real number, got %r" % (who, voxel_size))
    v = float(voxel_size)
    if not (math.isfinite(v) and v > 0):
        raise ValueError("%s: voxel_size=%r must be finite and > 0" % (who, voxel_size))
    return v


def _host_bbox(bbox, who):
    bb = np.ascontiguousarray(bbox, np.float32).reshape(-1)
    if bb.shape[0] != 6 or not np.isfinite(bb).all():
        raise ValueError("%s: bbox must be 6 finite numbers (min xyz, max xyz), got %r" % (who, bbox))
    return bb


def _widest_cloud_bbox(pts, lens):
    """float32[6] box [0, e] where e is the largest per-axis extent of any cloud's finite rows (one device->host read).
    The key only needs the widest cloud, not the span of all clouds: clouds far apart stay inside the key budget."""
    N, B = int(pts.shape[0]), int(lens.shape[0])
    if N == 0:
        return np.zeros((6,), np.float32)
    end = torch.cumsum(lens.to(torch.int64), 0)
    cloud = torch.searchsorted(end, torch.arange(N, device=pts.device), right=True)   # B: a row of no cloud
    cloud = torch.where(torch.isfinite(pts).all(1) & (cloud < B), cloud, B).unsqueeze(1).expand(N, 3)
    inf = float("inf")
    mn = torch.full((B + 1, 3), inf, device=pts.device).scatter_reduce(0, cloud, pts, "amin")[:B]
    mx = torch.full((B + 1, 3), -inf, device=pts.device).scatter_reduce(0, cloud, pts, "amax")[:B]
    ext = torch.where(mx >= mn, mx - mn, torch.zeros_like(mx)).amax(0).cpu().numpy()
    return np.concatenate([np.zeros(3), ext]).astype(np.float32)


def _stack_args(points, lengths, who):
    pts = _lib.tensor_arg(points, who + ": points", torch.float32, (None, 3))
    lens = _lib.tensor_arg(lengths, who + ": lengths", torch.int32, (None,), pts.device)
    B = int(lens.shape[0])
    if not 1 <= B <= 1024:
        raise ValueError("%s: lengths must hold 1 to 1024 clouds, got %d" % (who, B))
    return pts, lens


def voxel_down_sample(points, lengths, voxel_size, bbox=None):
    """points [N,3] float32 and lengths [B] int32 (CUDA) of B stacked raw clouds -> (points [M,3] float32, lengths [B]
    int32) on the device: every cloud voxelised at voxel_size (a double: 0.03 is the double 0.03). Clouds as in
    batch_grid_subsampling: rows at or past sum(lengths) belong to no cloud, lengths summing past N cut the last cloud.

    bbox (6 floats, optional) only sizes the sort key: any box at least as wide as every cloud (a cloud merely
    displaced outside it is still exact). Without it, the widest cloud's extent is read from the device. The
    number of voxels is read back: one synchronisation, like the TF subsampling op."""
    who = "voxel_down_sample"
    v = check_voxel_size(voxel_size, who)
    pts, lens = _stack_args(points, lengths, who)
    bb = _widest_cloud_bbox(pts, lens) if bbox is None else _host_bbox(bbox, who)
    dev = pts.device
    N, B = int(pts.shape[0]), int(lens.shape[0])
    lib = _lib.lib()
    out = torch.empty((max(N, 1), 3), dtype=torch.float32, device=dev)
    out_len = torch.empty((B,), dtype=torch.int32, device=dev)
    out_m = torch.empty((1,), dtype=torch.int32, device=dev)
    ws = _lib.workspace(lib.d3f_voxel_down_sample_workspace_bytes(N, B), dev)
    _lib.check(lib.d3f_voxel_down_sample(_lib.ptr(pts), _lib.ptr(lens), B, N, None, v, bb.ctypes.data_as(C.c_void_p),
                                         _lib.ptr(out), _lib.ptr(out_len), _lib.ptr(out_m), N, None, _lib.ptr(ws),
                                         ws.numel(), _lib.stream()), "d3f_voxel_down_sample")
    M = int(out_m.item())
    if M < 0:
        raise ValueError("%s: a cloud needs more voxels per axis than bbox %s allows" % (who, bb.tolist()))
    return out[:M], out_len


class VoxelStage:
    """The static form for one slot of encoder.GraphPipeline: raw points [raw_capacity,3], raw lengths [B] and the raw
    row count [1] (device) are loaded by the caller; run() voxelises them into a pyramid slot's points0 / lengths0 /
    n0 and ORs the overflow bits into its status word, with no device->host read, so it can be captured in a graph."""

    def __init__(self, raw_capacity, n_clouds, voxel_size, bbox, device):
        self.voxel_size = check_voxel_size(voxel_size, "GraphPipeline")
        self.capacity, self.n_clouds = max(int(raw_capacity), 1), int(n_clouds)
        self.bbox = _host_bbox(bbox, "GraphPipeline")
        self.points = torch.zeros((self.capacity, 3), dtype=torch.float32, device=device)
        self.lengths = torch.zeros((self.n_clouds,), dtype=torch.int32, device=device)
        self.n = torch.zeros((1,), dtype=torch.int32, device=device)
        self.ws = _lib.workspace(_lib.lib().d3f_voxel_down_sample_workspace_bytes(self.capacity, self.n_clouds), device)

    def run(self, out_points, out_lengths, out_n, status):
        _lib.check(_lib.lib().d3f_voxel_down_sample(
            _lib.ptr(self.points), _lib.ptr(self.lengths), self.n_clouds, self.capacity, _lib.ptr(self.n),
            self.voxel_size, self.bbox.ctypes.data_as(C.c_void_p), _lib.ptr(out_points), _lib.ptr(out_lengths),
            _lib.ptr(out_n), int(out_points.shape[0]), _lib.ptr(status), _lib.ptr(self.ws), self.ws.numel(),
            _lib.stream()), "d3f_voxel_down_sample")
