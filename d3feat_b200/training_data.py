"""Training pairs of D3Feat built on the GPU: ground-truth correspondences, keypoint sampling and the generators'
augmentation (csrc/correspond.cu; oracle/pairs_np.py is the contract, exact).

The reference builds these on the host in front of every step: KITTI's generator calls Open3D's KD-tree once per anchor
point (datasets/KITTI.py:35-48, 319-327) and draws 1024 matches without replacement (:184-189); 3DMatch's offline
cal_overlap.py runs cv2.BFMatcher over every fragment pair (:78-126) and the generator draws keypts_num matches with
replacement (datasets/ThreeDMatch.py:218-229); both add uniform noise and rotate each cloud about a random axis, KITTI
also scales each pair and shifts each cloud (ThreeDMatch.py:24-45, 266-273; KITTI.py:191-206).

    pairs = training_pairs(points, lengths, pairs, trans, config, "kitti", seed=step)
    pts, lens, anc, pos, backup = pairs.pair(0)
    inputs = enc.build_inputs(pts, lens)
    desc, scores = training.forward(inputs, config)
    loss, *stats = training.d3feat_loss(desc, scores, anc, pos, backup, config)

Random draws come from counter-based splitmix64 of (seed, pair, index, purpose), so the result does not depend on how
the work is spread over the GPU; numpy's random stream is not reproduced. Clouds are stacked as for icp_pairs: points
[N,3] float32 and lengths [B] int32 on the GPU, pairs [P,2] int32 (anchor cloud, positive cloud), trans [P,4,4] float64
mapping anchor points onto the positive (GroundTruth.pose). A pair naming a cloud outside [0, B) has no rows.
"""
import math
from collections import namedtuple

import numpy as np
import torch

from . import _lib

MODES = {"radius": 0, "nearest": 1}
MAX_ROWS = (1 << 31) - 1

# training_3DMatch.py:124-131 and training_KITTI.py:124-132 (augment_occlusion 'none' in both: not applied)
AUGMENT_3DMATCH = dict(augment_rotation=1, augment_scale_min=0.9, augment_scale_max=1.1, augment_noise=0.005,
                       augment_occlusion="none")
AUGMENT_KITTI = dict(augment_rotation=1, augment_scale_min=0.8, augment_scale_max=1.2, augment_noise=0.01,
                     augment_occlusion="none", augment_shift_range=2.0)

Correspondences = namedtuple("Correspondences", "offset rows count overlap")
Correspondences.__doc__ = """Ground-truth correspondences of P cloud pairs. offset [P+1] int64: pair p owns rows
    [offset[p], offset[p+1]); rows [M,2] int32 cloud-local (anchor row, positive row), ascending; count [P] int32;
    overlap [P] float64 = count / anchor rows (0 for an empty anchor), cal_overlap.py's ratio."""

Sample = namedtuple("Sample", "anc pos valid")
Sample.__doc__ = """k sampled correspondences per pair: anc [P,k] int32 anchor rows, pos [P,k] int32 positive rows plus
    the anchor's length (indices into the pair's [anchor || positive] stack), -1 for an invalid pair; valid [P] bool."""

Augmented = namedtuple("Augmented", "points lengths row_offset backup_points R scale shift")
Augmented.__doc__ = """Augmented clouds of P pairs. points [T,3] float32: pair p's anchor then positive rows from
    row_offset[p] (row_offset [P+1] int64); lengths [P,2] int32; backup_points [T,3] float32: trans applied to the
    anchor, the positive as it is (what d3feat_loss measures safe_radius on); R [2P,num_axis,3,3] float32 (cloud
    2p + side), scale [P] float64 (1 without scaling), shift [2P,3] float64 (0 without shifting)."""

TrainingPairs = namedtuple("TrainingPairs", "points lengths row_offset anc_inds pos_inds backup_points valid count")


class TrainingPairs(TrainingPairs):
    """A batch of P training pairs: points [T,3], lengths [P,2], row_offset [P+1] (int64), anc_inds / pos_inds [P,k]
    int32, backup_points [T,3], valid [P] bool (enough correspondences; an invalid pair holds -1 indices and is skipped
    by the reference's generators), count [P] int32 correspondences."""
    __slots__ = ()

    def pair(self, p):
        """(points [n,3], lengths [2], anc_inds [k], pos_inds [k], backup_points [n,3]) of pair p: one step of
        enc.build_inputs / training.forward / training.d3feat_loss (batch_num = 1)."""
        lo, hi = (int(v) for v in self.row_offset[p:p + 2].tolist())
        return (self.points[lo:hi], self.lengths[p], self.anc_inds[p], self.pos_inds[p],
                self.backup_points[lo:hi])


def _stack_args(points, lengths, pairs, trans, who):
    points = _lib.tensor_arg(points, "%s: points" % who, torch.float32, (None, 3))
    dev = points.device
    lengths = _lib.tensor_arg(lengths, "%s: lengths" % who, torch.int32, (None,), dev)
    pairs = _lib.tensor_arg(pairs, "%s: pairs" % who, torch.int32, (None, 2), dev)
    P = int(pairs.shape[0])
    trans = _lib.tensor_arg(trans, "%s: trans" % who, torch.float64, (P, 4, 4), dev)
    B = int(lengths.shape[0])
    if not 1 <= B <= 1024 or P < 1:
        raise ValueError("%s: %d clouds and %d pairs: need 1 to 1024 clouds and at least one pair" % (who, B, P))
    return points, lengths, pairs, trans, dev


def _number(v, name, who, lo=0.0, strict=False):
    try:
        x = float(v)
    except (TypeError, ValueError):
        raise ValueError("%s: %s=%r must be a number" % (who, name, v))
    if not math.isfinite(x) or x < lo or (strict and x <= lo):
        raise ValueError("%s: %s=%r must be finite and %s %g" % (who, name, v, ">" if strict else ">=", lo))
    return x


def _integer(v, name, who, lo, hi):
    if isinstance(v, bool) or not isinstance(v, (int, np.integer)) or not lo <= int(v) <= hi:
        raise ValueError("%s: %s=%r must be an integer in [%d, %d]" % (who, name, v, lo, hi))
    return int(v)


def correspondences(points, lengths, pairs, trans, distance, mode, *, bbox=None):
    """Every (anchor row, positive row) of each pair within `distance` after trans (mode "radius": all rows with
    d^2 < distance^2, KITTI's get_matching_indices) or the nearest such row (mode "nearest": cal_overlap.py's
    BFMatcher filtered by distance). bbox: 6 floats bounding the clouds, the bounds of all N rows when None (one
    device->host read); every coordinate must lie within 1024 cells (distance * 1.001) of the origin. The total number
    of rows is read back once to size `rows`. Returns Correspondences."""
    who = "correspondences"
    points, lengths, pairs, trans, dev = _stack_args(points, lengths, pairs, trans, who)
    tau = _number(distance, "distance", who, strict=True)
    if mode not in MODES:
        raise ValueError("%s: mode=%r must be one of %s" % (who, mode, sorted(MODES)))
    N, B, P = int(points.shape[0]), int(lengths.shape[0]), int(pairs.shape[0])
    if bbox is None:
        from .tf_custom_ops import host_bbox
        bbox = host_bbox(points)
    bbox = np.ascontiguousarray(bbox, np.float32).reshape(6)
    bb = bbox.ctypes.data_as(_lib.C.c_void_p)
    lib = _lib.lib()
    nbytes = lib.d3f_pair_correspondences_workspace_bytes(N, B, P, tau, bb)
    if nbytes == 0:
        raise ValueError("%s: no workspace for N=%d B=%d P=%d distance=%g bbox=%s: the grid exceeds its cell cap, a "
                         "bbox coordinate lies beyond 1024 cells of the origin, or P*ceil(N/256)*256 exceeds int32" % (
                             who, N, B, P, tau, bbox.tolist()))
    ws = _lib.workspace(nbytes, dev)
    offset = torch.empty((P + 1,), dtype=torch.int64, device=dev)
    count = torch.empty((P,), dtype=torch.int32, device=dev)
    overlap = torch.empty((P,), dtype=torch.float64, device=dev)
    m = MODES[mode]
    _lib.check(lib.d3f_pair_correspondences_count(_lib.ptr(points), _lib.ptr(lengths), B, N, bb, _lib.ptr(pairs), P,
                                                  _lib.ptr(trans), tau, m, _lib.ptr(offset), _lib.ptr(count),
                                                  _lib.ptr(overlap), _lib.ptr(ws), ws.numel(), _lib.stream()),
               "d3f_pair_correspondences_count")
    M = int(offset[P].item())
    if M > MAX_ROWS:
        raise ValueError("%s: %d correspondences exceed %d rows" % (who, M, MAX_ROWS))
    rows = torch.empty((M, 2), dtype=torch.int32, device=dev)
    _lib.check(lib.d3f_pair_correspondences_fill(_lib.ptr(points), B, N, bb, _lib.ptr(pairs), P, _lib.ptr(trans), tau,
                                                 m, M, _lib.ptr(rows), _lib.ptr(ws), ws.numel(), _lib.stream()),
               "d3f_pair_correspondences_fill")
    return Correspondences(offset, rows, count, overlap)


def sample_correspondences(corr, k, replace, min_count, seed, anchor_lengths):
    """k correspondences of every pair from corr (a Correspondences, or any table with offset [P+1] int64,
    nondecreasing within [0, M], and rows [M,2] int32, such as 3DMatch's keypts.pkl converted). offset may start above
    0 and end below M, as offset[a:b+1] of a larger table over its full rows does: rows outside [offset[0], offset[P])
    belong to no pair. replace=True: k draws with
    replacement (ThreeDMatch.py:218-229); False: a uniform random k-subset in random order (KITTI.py:184-189).
    valid = at least max(min_count, 1) candidates and, without replacement, at least k. anchor_lengths [P] int32 (the
    anchor's rows) offsets pos into the pair's [anchor || positive] stack. Never synchronises. Returns Sample."""
    who = "sample_correspondences"
    offset = _lib.tensor_arg(getattr(corr, "offset", None), "%s: offset" % who, torch.int64, (None,))
    dev = offset.device
    rows = _lib.tensor_arg(getattr(corr, "rows", None), "%s: rows" % who, torch.int32, (None, 2), dev)
    P = int(offset.shape[0]) - 1
    if P < 1:
        raise ValueError("%s: offset must hold P + 1 >= 2 entries" % who)
    anchor_lengths = _lib.tensor_arg(anchor_lengths, "%s: anchor_lengths" % who, torch.int32, (P,), dev)
    k = _integer(k, "k", who, 1, MAX_ROWS // P)
    min_count = _integer(min_count, "min_count", who, 0, MAX_ROWS)
    seed = _integer(seed, "seed", who, 0, (1 << 64) - 1)
    if not isinstance(replace, bool):
        raise ValueError("%s: replace=%r must be a bool" % (who, replace))
    M = int(rows.shape[0])
    if M > MAX_ROWS:
        raise ValueError("%s: %d rows exceed %d" % (who, M, MAX_ROWS))
    lib = _lib.lib()
    ws = _lib.workspace(lib.d3f_sample_correspondences_workspace_bytes(M, P), dev)
    anc, pos = (torch.empty((P, k), dtype=torch.int32, device=dev) for _ in range(2))
    valid = torch.empty((P,), dtype=torch.int32, device=dev)
    _lib.check(lib.d3f_sample_correspondences(_lib.ptr(offset), _lib.ptr(rows), M, P, _lib.ptr(anchor_lengths), k,
                                              int(replace), min_count, seed, _lib.ptr(anc), _lib.ptr(pos),
                                              _lib.ptr(valid), _lib.ptr(ws), ws.numel(), _lib.stream()),
               "d3f_sample_correspondences")
    return Sample(anc, pos, valid != 0)


def augment(points, lengths, pairs, trans, *, seed, noise, num_axis=1, scale=None, shift_range=None, capacity=None):
    """The generators' augmentation of both clouds of every pair: uniform noise, num_axis (1 or 3) random rotations,
    and with scale=(lo, hi) and shift_range (KITTI) one scale per pair and a shift per cloud. capacity: rows of the
    output buffers; None reads the total back (one synchronisation), an int never synchronises (rows past it are not
    written). Returns Augmented."""
    who = "augment"
    points, lengths, pairs, trans, dev = _stack_args(points, lengths, pairs, trans, who)
    seed = _integer(seed, "seed", who, 0, (1 << 64) - 1)
    noise = _number(noise, "noise", who)
    num_axis = _integer(num_axis, "num_axis", who, 1, 3)
    if num_axis == 2:
        raise ValueError("%s: num_axis=2 must be 1 or 3" % who)
    if (scale is None) != (shift_range is None):
        raise ValueError("%s: scale and shift_range go together (KITTI) or not at all (3DMatch)" % who)
    lo = hi = r = 0.0
    if scale is not None:
        try:
            lo, hi = (_number(v, "scale", who, lo=-math.inf) for v in scale)
        except TypeError:
            raise ValueError("%s: scale=%r must be a (min, max) pair" % (who, scale))
        if lo > hi:
            raise ValueError("%s: scale=%r must be ordered" % (who, scale))
        r = _number(shift_range, "shift_range", who)
    if capacity is not None:
        capacity = _integer(capacity, "capacity", who, 0, MAX_ROWS)
    N, B, P = int(points.shape[0]), int(lengths.shape[0]), int(pairs.shape[0])
    lib = _lib.lib()
    ws = _lib.workspace(lib.d3f_augment_pairs_workspace_bytes(B, P), dev)
    out_lengths = torch.empty((P, 2), dtype=torch.int32, device=dev)
    row_offset = torch.empty((P + 1,), dtype=torch.int64, device=dev)
    R = torch.empty((2 * P, num_axis, 3, 3), dtype=torch.float32, device=dev)
    sc = torch.empty((P,), dtype=torch.float64, device=dev)
    sh = torch.empty((2 * P, 3), dtype=torch.float64, device=dev)

    def run(cap, out, backup):
        _lib.check(lib.d3f_augment_pairs(_lib.ptr(points), _lib.ptr(lengths), B, N, _lib.ptr(pairs), P,
                                         _lib.ptr(trans), seed, noise, num_axis, int(scale is not None), lo, hi, r,
                                         cap, _lib.ptr(out), _lib.ptr(backup), _lib.ptr(out_lengths),
                                         _lib.ptr(row_offset), _lib.ptr(R), _lib.ptr(sc), _lib.ptr(sh), _lib.ptr(ws),
                                         ws.numel(), _lib.stream()),
                   "d3f_augment_pairs")

    if capacity is None:
        run(0, None, None)                     # the parameters and row_offset only
        capacity = int(row_offset[P].item())
        if capacity > MAX_ROWS:
            raise ValueError("%s: %d output rows exceed %d" % (who, capacity, MAX_ROWS))
    out = torch.empty((capacity, 3), dtype=torch.float32, device=dev)
    backup = torch.empty((capacity, 3), dtype=torch.float32, device=dev)
    run(capacity, out, backup)
    return Augmented(out, out_lengths, row_offset, backup, R, sc, sh)


DATASETS = ("3dmatch", "kitti")


def training_pairs(points, lengths, pairs, trans, config, dataset, seed, *, bbox=None):
    """One training batch of P pairs from stacked clouds and their ground truth, as the dataset's generator builds it:
      "3dmatch": nearest correspondences within config.first_subsampling_dl, config.keypts_num draws with replacement,
                 AUGMENT_3DMATCH's noise and rotation;
      "kitti":   every correspondence within 1.5 * first_subsampling_dl, keypts_num drawn without replacement (pairs
                 with fewer than 1024 are invalid), AUGMENT_KITTI's noise, rotation, scale and shift.
    Augmentation settings are read from config (augment_noise, augment_rotation, augment_scale_min / _max,
    augment_shift_range) where it has them. Two device->host reads: the number of correspondences and of output rows
    (three without bbox). Returns TrainingPairs; TrainingPairs.pair(p) is one step's input."""
    who = "training_pairs"
    if dataset not in DATASETS:
        raise ValueError("%s: dataset=%r must be one of %s" % (who, dataset, DATASETS))
    kitti = dataset == "kitti"
    aug = AUGMENT_KITTI if kitti else AUGMENT_3DMATCH
    opt = {key: getattr(config, key, v) for key, v in aug.items()}
    dl = _number(getattr(config, "first_subsampling_dl", None), "first_subsampling_dl", who, strict=True)
    corr = correspondences(points, lengths, pairs, trans, 1.5 * dl if kitti else dl,
                           "radius" if kitti else "nearest", bbox=bbox)
    a = augment(points, lengths, pairs, trans, seed=seed, noise=opt["augment_noise"],
                num_axis=opt["augment_rotation"],
                scale=(opt["augment_scale_min"], opt["augment_scale_max"]) if kitti else None,
                shift_range=opt["augment_shift_range"] if kitti else None)
    s = sample_correspondences(corr, config.keypts_num, not kitti, 1024 if kitti else 0, seed,
                               a.lengths[:, 0].contiguous())
    return TrainingPairs(a.points, a.lengths, a.row_offset, s.anc, s.pos, a.backup_points, s.valid, corr.count)
