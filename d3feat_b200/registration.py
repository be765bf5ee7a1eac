"""Rigid registration of cloud pairs on the GPU: deterministic RANSAC over keypoint matches (d3f_register_pairs).

Every consumer of the matches estimates a pose next, with Open3D's RANSAC on the host, one pair at a time: the 3DMatch
evaluation (geometric_registration/evaluate.py:84-99: ransac_n 3, distance 0.05, edge ratio 0.9, (50000, 1000)), the
KITTI tester (utils/tester.py:305-316: ransac_n 4, distance = voxel size) and the demo (demo_registration.py:184-192:
ransac_n 4, (4000000, 500)). Here all pairs of a batch register in one device call that can run inside a captured
CUDA graph (encoder.GraphPipeline(..., match_pairs=pairs, register={...})).

The result is exact and deterministic: oracle/register_np.py is the contract, restated op for op in fp64 without FMA.
Hypothesis h of pair p draws its sample from a counter-based splitmix64 of (seed, p, h), so the result does not depend
on how the work is spread over the GPU. The parameters and checkers mean what Open3D's do; Open3D's own random
sequence cannot be reproduced, so its poses are not reproduced bit for bit. The reference writes inv(pose) to its log
(geometric_registration/evaluate.py:103-104); `pose` here maps source points onto the target, t' ~ R s + t.

icp_pairs refines poses by point-to-point ICP over the dense clouds (d3f_icp_pairs), as the KITTI loader does with
Open3D's registration_icp (datasets/KITTI.py:284-301); oracle/icp_np.py is its contract, exact in the same way.
"""
import math
from collections import namedtuple

import numpy as np
import torch

from . import _lib
from .keypoints import KeypointSet
from .matching import Matches, host_pairs

Registration = namedtuple("Registration", "pose n_inliers n_correspondences hypothesis n_validated")
Registration.__doc__ = """Registration of P cloud pairs. pose [P,4,4] float64 (t' ~ R s + t), n_inliers [P] int32 (of
    the best hypothesis, after which the pose is refit over them), n_correspondences [P] int32 (the rows RANSAC drew
    from), hypothesis [P] int32 (the best h, -1 when the pair registered nothing: identity pose), n_validated [P] int32
    (validated hypotheses scored, at most max_validation)."""

OPTIONS = ("distance", "ransac_n", "edge_ratio", "max_iterations", "max_validation", "seed", "mutual")

Refinement = namedtuple("Refinement", "pose fitness inlier_rmse n_correspondences iterations")
Refinement.__doc__ = """ICP refinement of P cloud pairs, all for the final pose. pose [P,4,4] float64 (t' ~ R s + t; row 3
    copied from init), fitness [P] float64 (corresponding source rows / source rows), inlier_rmse [P] float64 (root mean
    square distance of the correspondences, 0 without any), n_correspondences [P] int32, iterations [P] int32 (pose
    updates made). A pair naming a cloud outside [0, B) or with an empty cloud keeps init with 0 everywhere."""

ICP_OPTIONS = ("distance", "max_iterations", "relative_fitness", "relative_rmse")


def check_options(distance=0.05, ransac_n=3, edge_ratio=0.9, max_iterations=50000, max_validation=1000, seed=0,
                  mutual=False, who="register_pairs"):
    """The RANSAC options as (distance, ransac_n, edge_ratio, max_iterations, max_validation, seed, mutual), each
    checked against the limits of d3f_register_pairs (ValueError)."""
    def integer(name, v, lo, hi):
        if isinstance(v, bool) or not isinstance(v, int) or not lo <= v <= hi:
            raise ValueError("%s: %s=%r must be an integer in [%d, %d]" % (who, name, v, lo, hi))
        return v
    n = integer("ransac_n", ransac_n, 3, 8)
    T = integer("max_iterations", max_iterations, 1, 1 << 24)
    V = integer("max_validation", max_validation, 1, T)
    seed = integer("seed", seed, 0, (1 << 64) - 1)
    try:
        tau, ratio = float(distance), float(edge_ratio)
    except (TypeError, ValueError):
        raise ValueError("%s: distance=%r and edge_ratio=%r must be numbers" % (who, distance, edge_ratio))
    if not (math.isfinite(tau) and tau > 0):
        raise ValueError("%s: distance=%r must be finite and > 0" % (who, distance))
    if not 0 < ratio <= 1:
        raise ValueError("%s: edge_ratio=%r must be in (0, 1]" % (who, edge_ratio))
    if not isinstance(mutual, bool):
        raise ValueError("%s: mutual=%r must be a bool" % (who, mutual))
    return tau, n, ratio, T, V, seed, mutual


def correspondences(matches, mutual=False):
    """(corr [P,L,2] int32, n_corr [P] int32) from a Matches, with torch ops on the device (no synchronisation).
    mutual=False: (i, nn_st[i]) for every real source slot i, Open3D's feature matching; mutual=True: the mutual
    matches, build_correspondence's list."""
    if mutual:
        return matches.matches.contiguous(), matches.n_matches.contiguous()
    P, k = matches.nn_st.shape
    src = torch.arange(k, dtype=torch.int32, device=matches.nn_st.device).expand(P, k)
    corr = torch.stack([src, matches.nn_st], dim=2).contiguous()
    return corr, (matches.nn_st >= 0).sum(dim=1, dtype=torch.int32)


def register_pairs(kp, matches, pairs, *, distance=0.05, ransac_n=3, edge_ratio=0.9, max_iterations=50000,
                   max_validation=1000, seed=0, mutual=False):
    """RANSAC pose of every pair from its keypoint matches.

    kp: the KeypointSet the matches were computed on (its points and count). matches: matching.Matches of `pairs`.
    pairs: [P,2] (src cloud, tgt cloud); a host list or array is range-checked against B (ValueError), a CUDA tensor is
    passed as it is, and a pair naming a cloud outside [0, B) then registers nothing. The defaults are the 3DMatch
    evaluation's. Returns Registration(pose, n_inliers, n_correspondences, hypothesis, n_validated)."""
    tau, n, ratio, T, V, seed, mutual = check_options(distance, ransac_n, edge_ratio, max_iterations, max_validation,
                                                      seed, mutual)
    if not isinstance(kp, KeypointSet) or not isinstance(matches, Matches):
        raise ValueError("register_pairs: expects a KeypointSet and the Matches computed on it")
    points = kp.points
    if not torch.is_tensor(points) or not points.is_cuda or points.dtype != torch.float32 or points.dim() != 3 \
            or int(points.shape[2]) != 3:
        raise ValueError("register_pairs: the KeypointSet's points must be a CUDA float32 tensor [B,k,3]")
    points = points.contiguous()
    dev = points.device
    B, k = int(points.shape[0]), int(points.shape[1])
    cnt = _lib.i32(kp.count, dev)
    if torch.is_tensor(pairs) and pairs.is_cuda:
        if pairs.dim() != 2 or int(pairs.shape[1]) != 2:
            raise ValueError("register_pairs: pairs must be [P, 2], got %s" % (tuple(pairs.shape),))
        pr = pairs.to(dtype=torch.int32).contiguous()
    else:
        pairs = pairs.numpy() if torch.is_tensor(pairs) else pairs
        pr = torch.from_numpy(host_pairs(pairs, B, "register_pairs")).to(dev)
    P = int(pr.shape[0])
    corr, n_corr = correspondences(matches, mutual)
    if int(corr.shape[0]) != P or corr.dim() != 3 or int(corr.shape[2]) != 2:
        raise ValueError("register_pairs: matches of %d pairs for %d pairs" % (int(corr.shape[0]), P))
    corr, n_corr = corr.to(torch.int32).contiguous(), n_corr.to(torch.int32).contiguous()
    L = int(corr.shape[1])
    lib = _lib.lib()
    ws = _lib.workspace(lib.d3f_register_pairs_workspace_bytes(L, P, T, V), dev)
    pose = torch.empty((P, 4, 4), dtype=torch.float64, device=dev)
    n_inliers, hypothesis, n_validated = (torch.empty((P,), dtype=torch.int32, device=dev) for _ in range(3))
    _lib.check(lib.d3f_register_pairs(_lib.ptr(points), _lib.ptr(cnt), B, k, _lib.ptr(corr), _lib.ptr(n_corr), L,
                                      _lib.ptr(pr), P, n, T, V, tau, ratio, seed, _lib.ptr(pose), _lib.ptr(n_inliers),
                                      _lib.ptr(hypothesis), _lib.ptr(n_validated), _lib.ptr(ws), ws.numel(),
                                      _lib.stream()),
               "d3f_register_pairs")
    return Registration(pose, n_inliers, n_corr, hypothesis, n_validated)


def check_icp_options(distance=None, max_iterations=30, relative_fitness=1e-6, relative_rmse=1e-6, who="icp_pairs"):
    """The ICP options as (distance, max_iterations, relative_fitness, relative_rmse), each checked against the limits
    of d3f_icp_pairs (ValueError). The defaults are Open3D's ICPConvergenceCriteria; distance has none."""
    if isinstance(max_iterations, bool) or not isinstance(max_iterations, int) or not 0 <= max_iterations <= 1024:
        raise ValueError("%s: max_iterations=%r must be an integer in [0, 1024]" % (who, max_iterations))
    try:
        tau, rf, rr = float(distance), float(relative_fitness), float(relative_rmse)
    except (TypeError, ValueError):
        raise ValueError("%s: distance=%r, relative_fitness=%r and relative_rmse=%r must be numbers" % (
            who, distance, relative_fitness, relative_rmse))
    if not (math.isfinite(tau) and tau > 0):
        raise ValueError("%s: distance=%r must be finite and > 0" % (who, distance))
    for name, v in (("relative_fitness", rf), ("relative_rmse", rr)):
        if not (math.isfinite(v) and v >= 0):
            raise ValueError("%s: %s=%r must be finite and >= 0" % (who, name, v))
    return tau, max_iterations, rf, rr


def icp_pairs(points, lengths, pairs, init=None, *, distance, max_iterations=30, relative_fitness=1e-6,
              relative_rmse=1e-6, rows=None, bbox=None):
    """Point-to-point ICP of every pair over stacked clouds, from `init`.

    points: CUDA float32 [N,3], lengths [B] (cloud b holds rows [start[b], start[b+1]) of their exclusive scan; rows
    past the last cloud belong to none). pairs: [P,2] (source cloud, target cloud); a host list or array is
    range-checked against B (ValueError), a CUDA tensor is passed as it is, and a pair naming a cloud outside [0, B)
    then keeps init. init: [P,4,4] float64 source-to-target poses (host or CUDA), the identity when None. rows: a
    device int32 row count (N is then a capacity) or None. bbox: 6 floats bounding the clouds, the bounds of all N
    rows when None (one device->host read); it only sizes the target grid (cell distance * 1.001), whose every
    coordinate must lie within 1024 cells of the origin. The defaults are Open3D's ICPConvergenceCriteria; the KITTI
    ground-truth refinement is icp_pairs(scans, lens, [(0, 1)], M, distance=0.2, max_iterations=200).
    Returns Refinement(pose, fitness, inlier_rmse, n_correspondences, iterations)."""
    tau, I, rf, rr = check_icp_options(distance, max_iterations, relative_fitness, relative_rmse)
    if not torch.is_tensor(points) or not points.is_cuda or points.dtype != torch.float32 or points.dim() != 2 \
            or int(points.shape[1]) != 3:
        raise ValueError("icp_pairs: points must be a CUDA float32 tensor [N,3]")
    points = points.contiguous()
    dev = points.device
    N = int(points.shape[0])
    lens = _lib.i32(lengths, dev)
    B = int(lens.numel())
    if torch.is_tensor(pairs) and pairs.is_cuda:
        if pairs.dim() != 2 or int(pairs.shape[1]) != 2:
            raise ValueError("icp_pairs: pairs must be [P, 2], got %s" % (tuple(pairs.shape),))
        pr = pairs.to(dtype=torch.int32).contiguous()
    else:
        pairs = pairs.numpy() if torch.is_tensor(pairs) else pairs
        pr = torch.from_numpy(host_pairs(pairs, B, "icp_pairs")).to(dev)
    P = int(pr.shape[0])
    if init is None:
        init = torch.eye(4, dtype=torch.float64, device=dev).expand(P, 4, 4)
    init = torch.as_tensor(init).to(device=dev, dtype=torch.float64).contiguous()
    if tuple(init.shape) != (P, 4, 4):
        raise ValueError("icp_pairs: init must be [%d, 4, 4], got %s" % (P, tuple(init.shape)))
    if rows is not None:
        rows = _lib.i32(rows, dev).reshape(-1)[:1]
    if bbox is None:
        from .tf_custom_ops import host_bbox
        bbox = host_bbox(points)
    bbox = np.ascontiguousarray(bbox, np.float32).reshape(6)
    lib = _lib.lib()
    bb = bbox.ctypes.data_as(_lib.C.c_void_p)
    nbytes = lib.d3f_icp_pairs_workspace_bytes(N, B, P, tau, bb)
    if nbytes == 0:
        raise ValueError("icp_pairs: no workspace for N=%d B=%d P=%d distance=%g bbox=%s: the grid exceeds its cell cap, "
                         "a bbox coordinate lies beyond 1024 cells of the origin, or B is outside [1, 1024]" % (
                             N, B, P, tau, bbox.tolist()))
    ws = _lib.workspace(nbytes, dev)
    pose = torch.empty((P, 4, 4), dtype=torch.float64, device=dev)
    fitness, inlier_rmse = (torch.empty((P,), dtype=torch.float64, device=dev) for _ in range(2))
    n_corr, iterations = (torch.empty((P,), dtype=torch.int32, device=dev) for _ in range(2))
    _lib.check(lib.d3f_icp_pairs(_lib.ptr(points), _lib.ptr(lens), B, N, _lib.ptr(rows), bb, _lib.ptr(pr), P,
                                 _lib.ptr(init), tau, I, rf, rr, _lib.ptr(pose), _lib.ptr(fitness),
                                 _lib.ptr(inlier_rmse), _lib.ptr(n_corr), _lib.ptr(iterations), _lib.ptr(ws),
                                 ws.numel(), _lib.stream()),
               "d3f_icp_pairs")
    return Refinement(pose, fitness, inlier_rmse, n_corr, iterations)
