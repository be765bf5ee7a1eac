"""Ground-truth metrics of matched and registered cloud pairs on the GPU (d3f_evaluate_pairs).

The last stage of every reference test script scores its keypoints, matches and poses against ground truth, per pair
on the host: feature-match recall (geometric_registration/evaluate.py:67-82, :207), keypoint repeatability
(repeatability/evaluate_3dmatch_our.py:30-41, evaluate_kitti_our.py:12-23), KITTI's RTE / RRE / success
(utils/tester.py:326-342) and 3DMatch registration recall (3dmatch/evaluate.m, mrEvaluateRegistration.m). Here all
pairs of a batch are scored in one device call that can run inside a captured CUDA graph
(encoder.GraphPipeline(..., evaluate={...})), and a whole benchmark run reads its totals once at the end.

Conventions. GroundTruth.pose maps source points onto the target (t ~ R s + t), the convention of
Registration.pose. A 3DMatch gt.log holds the inverse, target to source: io_utils.truth_for_pairs takes
G = inv(T_log) on the host. KITTI's `trans` is already source to target. Every distance test is d^2 < tau^2 with
tau^2 computed in fp64 (the reference compares sqrt(d^2) < tau: the two differ only at rounding ties); the cosine of
the rotation error is clamped to [-1, 1] (unclamped, a pose equal to G can give 1 + eps and a NaN in the reference).

The result is exact: oracle/evaluate_np.py is the contract, restated op for op in fp64 without FMA. Only rre_deg and
its sum go through acos, which is not correctly rounded on the GPU; they agree with the oracle within a few ulp.

Defaults are the 3DMatch evaluation's. For KITTI pass repeat_distance=0.5; its repeatability script scores the
keypoints against the saved RANSAC pose (utils/tester.py:316-317, evaluate_kitti_our.py:41-43), so pass that pose as
the truth to reproduce it.
"""
import math
from collections import namedtuple

import numpy as np
import torch

from . import _lib
from .keypoints import KeypointSet
from .matching import Matches, host_pairs

GroundTruth = namedtuple("GroundTruth", "pose info flags")
GroundTruth.__doc__ = """Truth of P cloud pairs. pose [P,4,4] float64 source-to-target (t ~ R s + t); info [P,6,6]
    float64 Choi information matrices or None; flags [P] int32: bit 0 = the pair has truth (it is evaluated), bit 1 =
    it counts for registration recall (3DMatch: j - i > 1; needs info). Host (numpy / CPU) or CUDA tensors. A
    non-finite pose of a flagged pair is a ValueError from the host; on the device it makes the pair a miss in every
    test."""

Evaluation = namedtuple("Evaluation", "valid n_match_inliers inlier_ratio fmr_hit n_repeated repeatability rte "
                                      "rre_deg rmse2 success recall_hit totals")
Evaluation.__doc__ = """Metrics of P pairs, R repeatability levels and S pose sets (the RANSAC poses, then the ICP
    poses). valid [P] int32 (1: evaluated); n_match_inliers [P] int32, inlier_ratio [P] float64, fmr_hit [P] int32;
    n_repeated [P,R] int32, repeatability [P,R] float64; rte, rre_deg, rmse2 (Choi's error) [S,P] float64, success
    (KITTI), recall_hit (3DMatch) [S,P] int32. A pair that is not evaluated has zeros and NaN rte / rre_deg / rmse2.
    totals [4 + R + 7 S] float64, summed in pair order: see summary()."""

OPTIONS = ("fmr_distance", "fmr_ratio", "repeat_distance", "repeat_levels", "err2", "rte_max", "rre_max_deg")
DEFAULT_LEVELS = (4, 8, 16, 32, 64, 128, 256, 512)
MAX_LEVELS = 14


def check_evaluate_options(k, fmr_distance=0.10, fmr_ratio=0.05, repeat_distance=0.10, repeat_levels=None, err2=0.04,
                           rte_max=2.0, rre_max_deg=5.0, who="evaluate_pairs"):
    """The options as (levels tuple, fmr_distance, fmr_ratio, repeat_distance, err2, rte_max, rre_max_deg), each
    checked against the limits of d3f_evaluate_pairs (ValueError). repeat_levels=None: 4, 8, ..., 512 clipped to k."""
    if repeat_levels is None:
        levels = tuple(n for n in DEFAULT_LEVELS if n <= k)
    else:
        try:
            levels = tuple(repeat_levels)
        except TypeError:
            raise ValueError("%s: repeat_levels=%r must be a sequence of integers" % (who, repeat_levels))
        if len(levels) > MAX_LEVELS or any(isinstance(n, bool) or not isinstance(n, (int, np.integer))
                                           for n in levels):
            raise ValueError("%s: repeat_levels=%r must be at most %d integers" % (who, repeat_levels, MAX_LEVELS))
        levels = tuple(int(n) for n in levels)
        if any(not 1 <= n <= k for n in levels) or any(b <= a for a, b in zip(levels, levels[1:])):
            raise ValueError("%s: repeat_levels=%r must ascend strictly within [1, k=%d]" % (who, repeat_levels, k))
    try:
        vals = [float(x) for x in (fmr_distance, fmr_ratio, repeat_distance, err2, rte_max, rre_max_deg)]
    except (TypeError, ValueError):
        raise ValueError("%s: the thresholds must be numbers" % who)
    fd, fr, rd, e2, rm, rr = vals
    for name, v in (("fmr_distance", fd), ("repeat_distance", rd), ("err2", e2), ("rte_max", rm)):
        if not (math.isfinite(v) and v > 0):
            raise ValueError("%s: %s=%r must be finite and > 0" % (who, name, v))
    if not (math.isfinite(fr) and 0 <= fr < 1):
        raise ValueError("%s: fmr_ratio=%r must be in [0, 1)" % (who, fr))
    if not (math.isfinite(rr) and 0 < rr <= 180):
        raise ValueError("%s: rre_max_deg=%r must be in (0, 180]" % (who, rr))
    return levels, fd, fr, rd, e2, rm, rr


def _on_device(x):
    return torch.is_tensor(x) and x.is_cuda


def _host(x, dtype):
    return np.asarray(x.cpu() if torch.is_tensor(x) else x, dtype)


def check_truth(truth, P, who="evaluate_pairs"):
    """ValueError unless `truth` is a GroundTruth of P pairs. A host pose is also checked: a pair with flags bit 0 and
    a non-finite entry in rows 0-2 of its pose is an error (a device pose is read as it is)."""
    if not isinstance(truth, GroundTruth):
        raise ValueError("%s: truth must be a GroundTruth" % who)
    for name, x, shape in (("pose", truth.pose, (P, 4, 4)), ("flags", truth.flags, (P,)),
                           ("info", truth.info, (P, 6, 6))):
        if x is None and name == "info":
            continue
        if tuple(np.shape(x)) != shape:
            raise ValueError("%s: truth %s must be %s, got %s" % (who, name, shape, tuple(np.shape(x))))
    if not _on_device(truth.pose):
        fl = _host(truth.flags, np.int64)
        bad = ((fl & 1) != 0) & ~np.isfinite(_host(truth.pose, np.float64)[:, :3, :]).all(axis=(1, 2))
        if bad.any():
            raise ValueError("%s: pair %d has truth with a non-finite pose" % (who, int(np.nonzero(bad)[0][0])))


def device_truth(truth, P, dev):
    """(pose, info or None, flags) of a checked GroundTruth as contiguous CUDA tensors."""
    check_truth(truth, P)

    def dev_t(x, dtype):
        t = x if torch.is_tensor(x) else torch.from_numpy(np.ascontiguousarray(x, _NP[dtype]))
        return t.to(device=dev, dtype=dtype).contiguous()
    info = None if truth.info is None else dev_t(truth.info, torch.float64)
    return dev_t(truth.pose, torch.float64), info, dev_t(truth.flags, torch.int32)


_NP = {torch.float64: np.float64, torch.int32: np.int32}


def evaluate_pairs(kp, matches, pairs, truth, registration=None, refinement=None, **options):
    """Ground-truth metrics of every pair.

    kp: the KeypointSet the matches were computed on (its points and count). matches: matching.Matches of `pairs`.
    pairs: [P,2] (src cloud, tgt cloud); a host list or array is range-checked against B (ValueError), a CUDA tensor
    is passed as it is, and a pair naming a cloud outside [0, B) is then not evaluated. truth: GroundTruth.
    registration / refinement: the Registration / Refinement whose poses are scored (either may be None).
    options: check_evaluate_options. Returns Evaluation."""
    if not isinstance(kp, KeypointSet) or not isinstance(matches, Matches):
        raise ValueError("evaluate_pairs: expects a KeypointSet and the Matches computed on it")
    points = kp.points
    if not torch.is_tensor(points) or not points.is_cuda or points.dtype != torch.float32 or points.dim() != 3 \
            or int(points.shape[2]) != 3:
        raise ValueError("evaluate_pairs: the KeypointSet's points must be a CUDA float32 tensor [B,k,3]")
    points = points.contiguous()
    dev = points.device
    B, k = int(points.shape[0]), int(points.shape[1])
    levels, fd, fr, rd, e2, rm, rr = check_evaluate_options(k, **options)
    cnt = _lib.i32(kp.count, dev)
    if torch.is_tensor(pairs) and pairs.is_cuda:
        if pairs.dim() != 2 or int(pairs.shape[1]) != 2:
            raise ValueError("evaluate_pairs: pairs must be [P, 2], got %s" % (tuple(pairs.shape),))
        pr = pairs.to(dtype=torch.int32).contiguous()
    else:
        pairs = pairs.numpy() if torch.is_tensor(pairs) else pairs
        pr = torch.from_numpy(host_pairs(pairs, B, "evaluate_pairs")).to(dev)
    P = int(pr.shape[0])
    mt, nm = matches.matches, matches.n_matches
    if mt.dim() != 3 or int(mt.shape[0]) != P or int(mt.shape[2]) != 2 or tuple(nm.shape) != (P,):
        raise ValueError("evaluate_pairs: matches of %s for %d pairs" % (tuple(mt.shape), P))
    mt, nm = mt.to(torch.int32).contiguous(), nm.to(torch.int32).contiguous()
    L = int(mt.shape[1])
    pose_gt, info, flags = device_truth(truth, P, dev)
    poses = []
    for what in (registration, refinement):
        if what is not None:
            T = what.pose
            if not torch.is_tensor(T) or not T.is_cuda or T.dtype != torch.float64 or tuple(T.shape) != (P, 4, 4):
                raise ValueError("evaluate_pairs: poses must be CUDA float64 [%d, 4, 4]" % P)
            poses.append(T.contiguous())
    R, S = len(levels), len(poses)
    lib = _lib.lib()
    ws = _lib.workspace(lib.d3f_evaluate_pairs_workspace_bytes(P, S), dev)
    i32, f64 = torch.int32, torch.float64
    valid, n_inl, fmr_hit = (torch.empty((P,), dtype=i32, device=dev) for _ in range(3))
    ratio = torch.empty((P,), dtype=f64, device=dev)
    n_rep = torch.empty((P, R), dtype=i32, device=dev)
    rep = torch.empty((P, R), dtype=f64, device=dev)
    rte, rre, rmse2 = (torch.empty((S, P), dtype=f64, device=dev) for _ in range(3))
    success, recall_hit = (torch.empty((S, P), dtype=i32, device=dev) for _ in range(2))
    totals = torch.empty((4 + R + 7 * S,), dtype=f64, device=dev)
    pose_ptrs = (_lib.C.c_void_p * 2)(*[T.data_ptr() for T in poses])
    lv = (_lib.C.c_int * MAX_LEVELS)(*levels)
    o = lambda t: _lib.ptr(t) if t.numel() else None     # noqa: E731 -- empty outputs (R = 0 or S = 0) are NULL
    _lib.check(lib.d3f_evaluate_pairs(_lib.ptr(points), _lib.ptr(cnt), B, k, _lib.ptr(mt), _lib.ptr(nm), L,
                                      _lib.ptr(pr), P, _lib.ptr(pose_gt), _lib.ptr(info), _lib.ptr(flags),
                                      pose_ptrs, S, lv, R, fd, fr, rd, e2, rm, rr, _lib.ptr(valid), _lib.ptr(n_inl),
                                      _lib.ptr(ratio), _lib.ptr(fmr_hit), o(n_rep), o(rep), o(rte), o(rre), o(rmse2),
                                      o(success), o(recall_hit), _lib.ptr(totals), _lib.ptr(ws), ws.numel(),
                                      _lib.stream()),
               "d3f_evaluate_pairs")
    return Evaluation(valid, n_inl, ratio, fmr_hit, n_rep, rep, rte, rre, rmse2, success, recall_hit, totals)


def summary(totals, levels, pose_sets=("ransac",)):
    """The reference's printed numbers from a totals vector (one device->host read if it is a CUDA tensor).

    levels: the repeatability levels of the run; pose_sets: names of its pose sets in order (("ransac",) with
    register, ("ransac", "icp") with ICP, () without poses). Ratios over an empty count are NaN. fmr is
    evaluate.py's recall (hits / pairs with truth); avg_inliers and avg_inlier_ratio keep its divisor, the hits."""
    t = np.asarray(totals.cpu() if torch.is_tensor(totals) else totals, np.float64).reshape(-1)
    R, S = len(levels), len(pose_sets)
    if t.shape[0] != 4 + R + 7 * S:
        raise ValueError("summary: %d totals for %d levels and %d pose sets" % (t.shape[0], R, S))

    def div(a, b):
        return float(a) / float(b) if b else float("nan")
    n, hits = t[0], t[1]
    out = dict(n_pairs=int(n), fmr_hits=int(hits), fmr=div(hits, n), avg_inliers=div(t[3], hits),
               avg_inlier_ratio=div(t[2], hits),
               repeatability={int(lv): div(t[4 + r], n) for r, lv in enumerate(levels)})
    for s, name in enumerate(pose_sets):
        b = t[4 + R + 7 * s: 4 + R + 7 * s + 7]
        out[name] = dict(successes=int(b[0]), success_rate=div(b[0], n), rte=div(b[1], b[2]), rre_deg=div(b[3], b[4]),
                         recall_hits=int(b[5]), recall_pairs=int(b[6]), registration_recall=div(b[5], b[6]))
    return out


def sweep_summary(totals, arms, counts, levels, pose_sets=("ransac",)):
    """The keypoint-count table of a GraphPipeline(..., sweep=...) run: one row per (arm, count), arms outer, each the
    summary() of that row's totals plus its "arm" and "count" -- inlier ratio, FMR, repeatability, and per pose set the
    success rate, RTE, RRE and registration recall. totals [len(arms), len(counts), 4 + R + 7 S] (evaluation_totals())."""
    t = np.asarray(totals.cpu() if torch.is_tensor(totals) else totals, np.float64)
    arms, counts = tuple(arms), tuple(int(c) for c in counts)
    if t.ndim != 3 or t.shape[:2] != (len(arms), len(counts)):
        raise ValueError("sweep_summary: totals of shape %s for %d arms and %d counts" % (t.shape, len(arms),
                                                                                         len(counts)))
    return [dict(arm=a, count=c, **summary(t[i, j], levels, pose_sets))
            for i, a in enumerate(arms) for j, c in enumerate(counts)]
