"""Input pyramid of the KPFCNN encoder -- mirror of Dataset.tf_descriptor_input (datasets/common.py:1301-1413)
with big_neighborhood_filter (:399-406) and calibrate_neighbors (:572-673), on the GPU.

The reference runs this loop on the CPU inside tf.data (13 radius searches + 4 grid subsamplings per batch).
Here the whole loop is ONE call into the library (d3f_pyramid_build): every level builds one hash grid per
(supports, radius) pair and reuses it for the searches that share it (conv_l, pool_l, up_{l-1}: 5 grid builds
instead of 13), the neighbour matrices are produced directly at the calibrated width (the reference computes the
full width and slices), and the only device->host reads are the number of cells after each subsampling plus one
bbox up front.
"""
import ctypes as C
import os

import numpy as np
import torch

from . import _lib
from . import tf_custom_ops as ops

MAX_LEVELS = 8


class PyramidSpec(C.Structure):
    """ctypes image of d3f_pyramid_spec (include/d3feat_b200.h)."""
    _fields_ = [("n_levels", C.c_int),
                ("conv_radius", C.c_float * MAX_LEVELS),
                ("sub_dl", C.c_float * MAX_LEVELS),
                ("pool_radius", C.c_float * MAX_LEVELS),
                ("up_radius", C.c_float * MAX_LEVELS),
                ("limit", C.c_int * MAX_LEVELS)]


def _level_radii(config):
    """(conv radius, subsample dl, pool radius, upsample radius) per level, exactly as the loop of
    tf_descriptor_input derives them (:1312-1396)."""
    r_normal = config.first_subsampling_dl * config.KP_extent * 2.5
    arch = list(config.architecture)
    layer_blocks = []
    levels = []
    for block_i, block in enumerate(arch):
        if "global" in block or "upsample" in block:
            break
        if not ("pool" in block or "strided" in block):
            layer_blocks.append(block)
            if block_i < len(arch) - 1 and "upsample" not in arch[block_i + 1]:
                continue
        lv = {}
        if layer_blocks:
            if np.any(["deformable" in b for b in layer_blocks[:-1]]):
                lv["conv_r"] = r_normal * config.density_parameter / (config.KP_extent * 2.5)
            else:
                lv["conv_r"] = r_normal
        else:
            lv["conv_r"] = None
        if "pool" in block or "strided" in block:
            lv["dl"] = 2 * r_normal / (config.KP_extent * 2.5)
            if "deformable" in block:
                lv["pool_r"] = r_normal * config.density_parameter / (config.KP_extent * 2.5)
            else:
                lv["pool_r"] = r_normal
            lv["up_r"] = 2 * lv["pool_r"]
        else:
            lv["dl"] = None
        levels.append(lv)
        r_normal *= 2
        layer_blocks = []
    return levels


def make_spec(config, neighborhood_limits):
    levels = _level_radii(config)
    if len(levels) > MAX_LEVELS:
        raise ValueError("pyramid: %d levels exceed D3F_MAX_LEVELS" % len(levels))
    spec = PyramidSpec()
    spec.n_levels = len(levels)
    for l, lv in enumerate(levels):
        spec.conv_radius[l] = float(lv["conv_r"]) if lv["conv_r"] is not None else -1.0
        spec.sub_dl[l] = float(lv["dl"]) if lv["dl"] is not None else -1.0
        spec.pool_radius[l] = float(lv.get("pool_r", -1.0)) if lv["dl"] is not None else -1.0
        spec.up_radius[l] = float(lv.get("up_r", -1.0)) if lv["dl"] is not None else -1.0
        spec.limit[l] = int(neighborhood_limits[l])
    return spec, levels


def _ptr_array(tensors):
    arr = (C.c_void_p * len(tensors))()
    for i, t in enumerate(tensors):
        arr[i] = t.data_ptr() if t is not None else None
    return arr


class PyramidBuffers:
    """Pre-allocated output matrices + workspace of one pyramid (a slot of BatchPipeline's ring): steady-state batches
    then touch no allocator at all.

    capacity: int (level-0 rows; every deeper level gets the same capacity -- a subsampled level can never have more
    points than its parent) or a per-level list (tight buckets for the static form, where launch grids are sized by
    capacity). `counts` (int32[L], device) receives the actual level sizes, `status` (int32[1]) the static form's
    error bits, `points0` / `lengths0` / `features0` are the static form's input buffers."""

    def __init__(self, config, neighborhood_limits, capacity, n_clouds, device, bbox=None):
        levels = _level_radii(config)
        L = len(levels)
        i32, f32 = torch.int32, torch.float32
        self.n_clouds, self.device = int(n_clouds), device
        self.caps = ([max(int(c), 1) for c in capacity] if isinstance(capacity, (list, tuple))
                     else [max(int(capacity), 1)] * L)
        assert len(self.caps) == L
        self.capacity = self.caps[0]
        self.limits = [int(neighborhood_limits[l]) for l in range(L)]
        self.pts = [None] + [torch.empty((self.caps[l], 3), dtype=f32, device=device) for l in range(1, L)]
        self.len = [None] + [torch.empty((n_clouds,), dtype=i32, device=device) for _ in range(1, L)]
        self.nb = [torch.empty((self.caps[l], self.limits[l]), dtype=i32, device=device)
                   if levels[l]["conv_r"] is not None else None for l in range(L)]
        self.pool = [torch.empty((self.caps[l + 1], self.limits[l]), dtype=i32, device=device)
                     if levels[l]["dl"] is not None and l + 1 < L else None for l in range(L)]
        self.up = [torch.empty((self.caps[l], self.limits[l]), dtype=i32, device=device)
                   if levels[l]["dl"] is not None and l + 1 < L else None for l in range(L)]
        self.counts = torch.zeros((MAX_LEVELS,), dtype=i32, device=device)
        self.status = torch.zeros((1,), dtype=i32, device=device)
        self.n0 = torch.zeros((1,), dtype=i32, device=device)
        self.points0 = torch.zeros((self.caps[0], 3), dtype=f32, device=device)
        self.lengths0 = torch.zeros((n_clouds,), dtype=i32, device=device)
        self.features0 = torch.ones((self.caps[0], config.in_features_dim), dtype=f32, device=device)
        self.bbox = None if bbox is None else np.ascontiguousarray(bbox, np.float32)
        self.ws = None

    def fits(self, n_points, n_clouds, limits):
        return n_points <= self.capacity and n_clouds == self.n_clouds and [int(x) for x in limits] == self.limits

    def workspace(self, nbytes):
        if self.ws is None or self.ws.numel() < nbytes:
            self.ws = torch.empty((int(nbytes * 1.25) + 256,), dtype=torch.uint8, device=self.device)
        return self.ws


def bucket_capacities(level_sizes, slack=1.125, quantum=256):
    """Per-level capacities of a shape bucket from the level sizes of a representative batch."""
    return [int(-(-int(n * slack + 64) // quantum) * quantum) for n in level_sizes]


def descriptor_input(config, stacked_points, stacked_lengths, neighborhood_limits, bbox=None, buffers=None,
                     static=False):
    """Returns the dict the blocks consume: points[L], neighbors[L], pools[L], upsamples[L], lengths[L]
    (placeholders of the reference's shapes at the last level, :1374-1377).

    neighborhood_limits: per-level column caps (Dataset.neighborhood_limits). Neighbour matrices are emitted
    with exactly `limit` columns, padded with the shadow index; when the true maximum count is below the
    limit the extra columns are all-shadow and do not change any downstream result.

    static=True (needs `buffers` with a bbox): the sync-free form. Nothing is read back from the device; every returned
    tensor is a whole capacity-sized buffer and inputs["rows"][l] is a device scalar with the level's actual row count
    (inputs["counts"], inputs["status"] hold all of them / the error bits). stacked_points / stacked_lengths must
    already be buffers.points0 / buffers.lengths0 (the caller copies each batch into them) with buffers.n0 set.
    The launch sequence is then the same for every batch of the bucket -- it can be captured in a CUDA graph.
    """
    dev = stacked_points.device
    pts = _lib.f32(stacked_points, dev)
    lens = _lib.i32(stacked_lengths, dev)
    if static:
        if buffers is None or buffers.bbox is None:
            raise ValueError("pyramid: the static form needs pre-allocated buffers with a scene bbox")
        bbox = buffers.bbox
    if bbox is None:
        bbox = ops.host_bbox(pts)
    bb = np.ascontiguousarray(bbox, dtype=np.float32)
    bbp = bb.ctypes.data_as(C.c_void_p)
    spec, levels = make_spec(config, neighborhood_limits)
    L = spec.n_levels
    N0, B = int(pts.shape[0]), int(lens.shape[0])
    # a subsampled level can never have more points than its parent: every level gets the level-0 capacity
    cap = [max(N0, 1)] * L
    lib = _lib.lib()
    i32, f32 = torch.int32, torch.float32
    if buffers is not None:
        if not buffers.fits(N0, B, [neighborhood_limits[l] for l in range(L)]):
            raise ValueError("pyramid: buffers (capacity %d, %d clouds) do not fit this batch (%d points, %d clouds)"
                             % (buffers.capacity, buffers.n_clouds, N0, B))
        cap = list(buffers.caps)
        out_pts, out_len, out_nb, out_pool, out_up = buffers.pts, buffers.len, buffers.nb, buffers.pool, buffers.up
    else:
        out_pts = [None] + [torch.empty((cap[l], 3), dtype=f32, device=dev) for l in range(1, L)]
        out_len = [None] + [torch.empty((B,), dtype=i32, device=dev) for l in range(1, L)]
        lim = [int(neighborhood_limits[l]) for l in range(L)]
        out_nb = [torch.empty((cap[l], lim[l]), dtype=i32, device=dev) if levels[l]["conv_r"] is not None else None
                  for l in range(L)]
        out_pool = [torch.empty((cap[l + 1], lim[l]), dtype=i32, device=dev)
                    if levels[l]["dl"] is not None and l + 1 < L else None for l in range(L)]
        out_up = [torch.empty((cap[l], lim[l]), dtype=i32, device=dev)
                  if levels[l]["dl"] is not None and l + 1 < L else None for l in range(L)]
    cap_arr = (C.c_int * L)(*cap)
    nbytes = lib.d3f_pyramid_workspace_bytes(B, C.byref(spec), cap_arr, bbp)
    if nbytes == 0:
        raise _lib.D3FError("pyramid: hash grid too large for bbox %s" % bb.tolist())
    ws = buffers.workspace(nbytes) if buffers is not None else _lib.workspace(nbytes, dev)
    empty_i = torch.zeros((0, 1), dtype=i32, device=dev)
    out = dict(points=[], neighbors=[], pools=[], upsamples=[], lengths=[], orders=[])
    if static:
        _lib.check(lib.d3f_pyramid_build(_lib.ptr(pts), _lib.ptr(lens), B, N0, C.byref(spec), bbp,
                                         _ptr_array(out_pts), _ptr_array(out_len), _ptr_array(out_nb),
                                         _ptr_array(out_pool), _ptr_array(out_up), cap_arr, None, _lib.ptr(ws),
                                         ws.numel(), _lib.stream(), _lib.ptr(buffers.counts),
                                         _lib.ptr(buffers.status), _lib.ptr(buffers.n0)), "d3f_pyramid_build")
        for l in range(L):
            out["points"].append(pts if l == 0 else out_pts[l])
            out["lengths"].append(lens if l == 0 else out_len[l])
            out["neighbors"].append(out_nb[l] if out_nb[l] is not None else empty_i)
            out["pools"].append(out_pool[l] if out_pool[l] is not None else empty_i)
            out["upsamples"].append(out_up[l] if out_up[l] is not None else empty_i)
            out["orders"].append(torch.zeros((0,), dtype=i32, device=dev))
        out["rows"] = [buffers.counts[l:l + 1] for l in range(L)]
        out["counts"], out["status"] = buffers.counts, buffers.status
        return out
    sizes = (C.c_int * L)()
    counts = buffers.counts if buffers is not None else None
    status = buffers.status if buffers is not None else None
    _lib.check(lib.d3f_pyramid_build(_lib.ptr(pts), _lib.ptr(lens), B, N0, C.byref(spec), bbp, _ptr_array(out_pts),
                                     _ptr_array(out_len), _ptr_array(out_nb), _ptr_array(out_pool),
                                     _ptr_array(out_up), cap_arr, sizes, _lib.ptr(ws), ws.numel(), _lib.stream(),
                                     _lib.ptr(counts), _lib.ptr(status), None),
               "d3f_pyramid_build")
    n = [int(sizes[l]) for l in range(L)]
    for l in range(L):
        out["points"].append(pts if l == 0 else out_pts[l][:n[l]])
        out["lengths"].append(lens if l == 0 else out_len[l])
        out["neighbors"].append(out_nb[l][:n[l]] if out_nb[l] is not None else empty_i)
        if levels[l]["dl"] is not None and l + 1 < L:
            out["pools"].append(out_pool[l][:n[l + 1]])
            out["upsamples"].append(out_up[l][:n[l]])
        else:
            out["pools"].append(empty_i)
            out["upsamples"].append(empty_i)
        out["orders"].append(torch.zeros((0,), dtype=i32, device=dev))
    # D3F_QUERY_ORDER=1: hand the level-0 gather kernels the hash grid's cell order as query visiting order
    if os.environ.get("D3F_QUERY_ORDER", "0") == "1" and levels[0]["conv_r"] is not None:
        out["orders"][0] = ops.NeighborGrid(pts, lens, levels[0]["conv_r"], bb).order()
    return out


def flat_inputs(inputs, stacked_features):
    """The positional list models/KPFCNN_model.py:86-121 unpacks: points + neighbors + pools + upsamples +
    [features] (the batch-weight / batch-index tensors are training-only)."""
    return inputs["points"] + inputs["neighbors"] + inputs["pools"] + inputs["upsamples"] + [stacked_features]


def calibrate_neighbors(config, clouds, keep_ratio=0.8, device="cuda"):
    """Column caps per level: the smallest count c such that at least keep_ratio of the neighbourhoods have
    <= c neighbours -- datasets/common.py:572-673 (histogram of conv-neighbour counts, cumulative sum,
    percentile). `clouds` is an iterable of float32[N,3] arrays (one cloud each)."""
    levels = _level_radii(config)
    hist_n = int(np.ceil(4 / 3 * np.pi * (config.density_parameter + 1) ** 3))
    hists = np.zeros((len(levels), hist_n), np.int64)
    for cloud in clouds:
        p = torch.as_tensor(np.ascontiguousarray(cloud, np.float32)).to(device)
        b = torch.tensor([p.shape[0]], dtype=torch.int32, device=device)
        bbox = ops.host_bbox(p)
        for li, lv in enumerate(levels):
            if lv["conv_r"] is not None:
                g = ops.NeighborGrid(p, b, lv["conv_r"], bbox)
                counts, _ = g.count(p, b)
                c = np.bincount(counts.cpu().numpy(), minlength=hist_n)[:hist_n]   # counts >= hist_n are dropped (:640)
                hists[li] += c
            if lv["dl"] is None:
                break
            p, b = ops.batch_grid_subsampling(p, b, lv["dl"], bbox=bbox)
    cumsum = np.cumsum(hists.T, axis=0)
    percentiles = np.sum(cumsum < (keep_ratio * cumsum[hist_n - 1, :]), axis=0)
    return [int(x) for x in percentiles]
