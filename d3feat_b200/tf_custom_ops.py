"""Host-side mirror of the reference's native ops (tf_custom_ops/), backed by the sm_90a hash-grid kernels.

Reference interface                                   -> here
  tf_batch_neighbors_module.batch_ordered_neighbors   -> batch_ordered_neighbors   (tf_batch_neighbors.cpp:8-30)
  tf_neighbors_module.ordered_neighbors               -> ordered_neighbors         (tf_neighbors.cpp:8-18)
  tf_batch_subsampling_module.batch_grid_subsampling  -> batch_grid_subsampling    (tf_batch_subsampling.cpp:8-20)
  tf_subsampling_module.grid_subsampling              -> grid_subsampling          (tf_subsampling.cpp:8-17)
  datasets/common.py:67-72 tf_batch_subsampling / tf_batch_neighbors wrappers -> same names

Tensors are contiguous CUDA torch tensors (float32 points, int32 lengths / indices). Like the TF ops these
return tensors whose shape is data dependent (max neighbour count, number of cells), so each call reads
one or two integers back from the device; the pyramid builder (pyramid.py) uses the capped single-phase
entry points instead and does not synchronise per op.

Canonical orders (see DESIGN.md): neighbours ascend in (d2, index); subsampled cells ascend in the
reference's cell key per cloud. Values are bit-identical to the reference's C++ cores.
"""
import ctypes as C

import numpy as np
import torch

from . import _lib


def host_bbox(points):
    """float32[6] numpy bbox of a CUDA point tensor via the d3f_bbox kernel (one device->host read)."""
    pts = _lib.tensor_arg(points, "host_bbox: points", torch.float32, (None, 3))
    out = torch.empty((6,), dtype=torch.float32, device=pts.device)
    _lib.check(_lib.lib().d3f_bbox(_lib.ptr(pts), pts.shape[0], _lib.ptr(out), _lib.stream()), "d3f_bbox")
    bb = out.cpu().numpy().astype(np.float32)
    if pts.shape[0] == 0:
        bb[:] = 0
    return bb


def merge_bbox(a, b):
    return np.concatenate([np.minimum(a[:3], b[:3]), np.maximum(a[3:], b[3:])]).astype(np.float32)


def _bbox_ptr(bb):
    bb = np.ascontiguousarray(bb, dtype=np.float32)
    return bb, bb.ctypes.data_as(C.c_void_p)


class NeighborGrid:
    """Hash grid over the supports (d3f_radius_neighbors_build); reusable for several query sets."""

    def __init__(self, supports, s_batches, radius, bbox=None):
        self.s = _lib.tensor_arg(supports, "NeighborGrid: supports", torch.float32, (None, 3))
        self.sb = _lib.tensor_arg(s_batches, "NeighborGrid: s_batches", torch.int32, (None,), self.s.device)
        supports, s_batches = self.s, self.sb
        self.radius = float(radius)
        self.B = int(s_batches.shape[0])
        self.Ns = int(supports.shape[0])
        self.bbox = host_bbox(supports) if bbox is None else np.asarray(bbox, np.float32)
        self._bb, self._bbp = _bbox_ptr(self.bbox)
        L = _lib.lib()
        nbytes = L.d3f_radius_neighbors_workspace_bytes(self.Ns, self.B, self.radius, self._bbp)
        if nbytes == 0:
            raise _lib.D3FError("radius_neighbors: grid too large for radius %g over bbox %s"
                                % (self.radius, self.bbox.tolist()))
        self.ws = _lib.workspace(nbytes, supports.device)
        _lib.check(L.d3f_radius_neighbors_build(_lib.ptr(self.s), _lib.ptr(self.sb), self.B, self.Ns, self.radius,
                                                self._bbp, _lib.ptr(self.ws), self.ws.numel(), _lib.stream()),
                   "d3f_radius_neighbors_build")

    def order(self):
        """int32[Ns]: support indices in cell order (spatially coherent visiting order)."""
        out = torch.empty((max(self.Ns, 1),), dtype=torch.int32, device=self.s.device)
        _lib.check(_lib.lib().d3f_radius_neighbors_order(_lib.ptr(self.ws), self.Ns, self.B, self.radius, self._bbp,
                                                         _lib.ptr(out), _lib.stream()), "d3f_radius_neighbors_order")
        return out[:self.Ns]

    def _queries(self, op, queries, q_batches):
        q = _lib.tensor_arg(queries, "NeighborGrid.%s: queries" % op, torch.float32, (None, 3), self.s.device)
        return q, _lib.tensor_arg(q_batches, "NeighborGrid.%s: q_batches" % op, torch.int32, (self.B,), self.s.device)

    def count(self, queries, q_batches):
        queries, q_batches = self._queries("count", queries, q_batches)
        Nq = int(queries.shape[0])
        counts = torch.empty((max(Nq, 1),), dtype=torch.int32, device=queries.device)
        mx = torch.zeros((1,), dtype=torch.int32, device=queries.device)
        _lib.check(_lib.lib().d3f_radius_neighbors_count(
            _lib.ptr(queries), _lib.ptr(q_batches), Nq, _lib.ptr(self.s), _lib.ptr(self.sb), self.B, self.Ns,
            self.radius, self._bbp, _lib.ptr(self.ws), _lib.ptr(counts), _lib.ptr(mx), _lib.stream()),
            "d3f_radius_neighbors_count")
        return counts[:Nq], mx

    def fill(self, queries, q_batches, cols, pad_value):
        queries, q_batches = self._queries("fill", queries, q_batches)
        Nq = int(queries.shape[0])
        out = torch.empty((Nq, int(cols)), dtype=torch.int32, device=queries.device)
        if Nq * int(cols) > 0:
            _lib.check(_lib.lib().d3f_radius_neighbors_fill(
                _lib.ptr(queries), _lib.ptr(q_batches), Nq, _lib.ptr(self.s), _lib.ptr(self.sb), self.B, self.Ns,
                self.radius, self._bbp, _lib.ptr(self.ws), int(cols), int(pad_value), _lib.ptr(out), _lib.stream()),
                "d3f_radius_neighbors_fill")
        return out


def _radius_scalar(radius):
    # the TF ops take a rank-0/1 float tensor and read element 0 (tf_batch_neighbors.cpp:75)
    if torch.is_tensor(radius):
        return float(radius.reshape(-1)[0].item())
    return float(np.asarray(radius, dtype=np.float32).reshape(-1)[0])


def batch_ordered_neighbors(queries, supports, q_batches, s_batches, radius, max_cols=None, bbox=None):
    """int32[Nq, max_count]: indices of the supports of the same cloud with d2 < radius^2, ascending in
    (d2, index), padded with Ns (neighbors.cpp:211-332). `max_cols` (extension): keep only the nearest
    max_cols columns and skip the count pass / host read (what big_neighborhood_filter does afterwards)."""
    dev = queries.device
    q, s = _lib.f32(queries, dev), _lib.f32(supports, dev)
    qb, sb = _lib.i32(q_batches, dev), _lib.i32(s_batches, dev)
    r = _radius_scalar(radius)
    grid = NeighborGrid(s, sb, r, bbox)
    if max_cols is None:
        _, mx = grid.count(q, qb)
        cols = int(mx.item())
    else:
        cols = int(max_cols)
    return grid.fill(q, qb, cols, s.shape[0])


def ordered_neighbors(queries, supports, radius):
    """Non-batch op (neighbors.cpp:58-123): one cloud, rows padded with -1."""
    dev = queries.device
    q, s = _lib.f32(queries, dev), _lib.f32(supports, dev)
    qb = torch.tensor([q.shape[0]], dtype=torch.int32, device=dev)
    sb = torch.tensor([s.shape[0]], dtype=torch.int32, device=dev)
    grid = NeighborGrid(s, sb, _radius_scalar(radius))
    _, mx = grid.count(q, qb)
    return grid.fill(q, qb, int(mx.item()), -1)


def _subsample(points, batches, dl, features=None, classes=None, bbox=None, sync=True):
    dev = points.device
    pts = _lib.f32(points, dev)
    b = _lib.i32(batches, dev)
    N, B = int(pts.shape[0]), int(b.shape[0])
    f = _lib.f32(features, dev) if features is not None else None
    c = _lib.i32(classes, dev).reshape(N, -1).contiguous() if classes is not None else None
    fdim = int(f.shape[1]) if f is not None else 0
    ldim = int(c.shape[1]) if c is not None else 0
    bb = host_bbox(pts) if bbox is None else np.asarray(bbox, np.float32)
    bb, bbp = _bbox_ptr(bb)
    L = _lib.lib()
    ws = _lib.workspace(L.d3f_grid_subsample_workspace_bytes(N, B), dev)
    out_p = torch.empty((max(N, 1), 3), dtype=torch.float32, device=dev)
    out_f = torch.empty((max(N, 1), fdim), dtype=torch.float32, device=dev) if fdim else None
    out_c = torch.empty((max(N, 1), ldim), dtype=torch.int32, device=dev) if ldim else None
    out_b = torch.empty((B,), dtype=torch.int32, device=dev)
    out_m = torch.empty((1,), dtype=torch.int32, device=dev)
    _lib.check(L.d3f_grid_subsample(_lib.ptr(pts), _lib.ptr(b), B, N, float(dl), _lib.ptr(f), fdim, _lib.ptr(c), ldim,
                                    bbp, _lib.ptr(out_p), _lib.ptr(out_f), _lib.ptr(out_c), _lib.ptr(out_b),
                                    _lib.ptr(out_m), _lib.ptr(ws), ws.numel(), _lib.stream()), "d3f_grid_subsample")
    M = int(out_m.item())
    if M < 0:
        raise _lib.D3FError("grid_subsample: a cloud is wider than the supplied bbox allows (sort-key overflow)")
    res = [out_p[:M], out_b]
    if fdim:
        res.append(out_f[:M])
    if ldim:
        res.append(out_c[:M])
    return res


def batch_grid_subsampling(points, batches, dl, bbox=None):
    """(float32[M,3], int32[B]): voxel barycenters per cloud and the new stack lengths
    (grid_subsampling.cpp:101-149, tf copy)."""
    p, b = _subsample(points, batches, _radius_scalar(dl), bbox=bbox)[:2]
    return p, b


def grid_subsampling(points, dl):
    """Non-batch op (tf_subsampling.cpp:8-17): one cloud."""
    nb = torch.tensor([points.shape[0]], dtype=torch.int32, device=points.device)
    return _subsample(points, nb, _radius_scalar(dl))[0]


# the wrappers of datasets/common.py:67-72
def tf_batch_subsampling(points, batches_len, sampleDl):
    return batch_grid_subsampling(points, batches_len, sampleDl)


def tf_batch_neighbors(queries, supports, q_batches, s_batches, radius):
    return batch_ordered_neighbors(queries, supports, q_batches, s_batches, radius)
