"""Descriptor matching between keypoint sets on the GPU (d3f_match_descriptors).

Every consumer of the keypoints matches descriptors between two fragments next, on the host: the 3DMatch evaluation
keeps the mutual nearest neighbours of `sqrt(2 - 2 * src @ tgt.T)` in ascending source order
(geometric_registration/evaluate.py:11-27); the KITTI tester and the registration demo hand the keypoints to Open3D,
which matches each source keypoint to its nearest target descriptor (utils/tester.py:281-314,
demo_registration.py:184-192). Here all pairs of a batch are matched in one device call that can run inside a captured
CUDA graph (encoder.GraphPipeline(..., keypoints=k, match_pairs=pairs)).

Contract, exact: s_ij = 0.0f, then for c = 0 .. D-1 in ascending order s_ij = s_ij + a_ic * b_jc in fp32, each product
and sum rounded on its own (no FMA). nn_st[p, i] = np.argmax(s[i, :]) and nn_ts[p, j] = np.argmax(s[:, j]) -- NaN
above everything, -0.0 equal to +0.0, ties to the smallest slot -- and sim_* the similarity there (a NaN is reported as
the positive quiet NaN). The mutual matches are (i, nn_st[i]) for every real i with nn_ts[nn_st[i]] == i, in
ascending i: build_correspondence's list. On unit descriptors argmax s is the reference's argmin sqrt(2 - 2s), except
where the rounding of 2 - 2s merges distinct similarities.

A dense match of every point is select_keypoints(..., k=max_len) followed by match_keypoints.
"""
from collections import namedtuple

import numpy as np
import torch

from . import _lib
from .keypoints import KeypointSet

Matches = namedtuple("Matches", "nn_st sim_st nn_ts sim_ts matches n_matches")
Matches.__doc__ = """Matches of P cloud pairs with k keypoint slots per cloud. nn_st [P,k] int32 / sim_st [P,k] float32:
    each source slot's nearest target slot and its similarity; nn_ts / sim_ts the same from the target side (-1 and 0
    for slots past the count, and for every slot when the other cloud is empty). matches [P,k,2] int32: the mutual
    (source slot, target slot) pairs in ascending source slot, rows past n_matches [P] int32 hold -1."""


def host_pairs(pairs, n_clouds, who="match_keypoints"):
    """A host list / array of (src, tgt) cloud pairs as int32 [P,2], every id checked against [0, n_clouds)."""
    arr = np.asarray(pairs)
    if arr.ndim != 2 or arr.shape[1] != 2 or arr.shape[0] < 1 or not np.issubdtype(arr.dtype, np.integer):
        raise ValueError("%s: pairs must be a non-empty [P, 2] list of integer cloud ids, got shape %s" % (
            who, arr.shape))
    bad = (arr < 0) | (arr >= n_clouds)
    if bad.any():
        p = int(np.nonzero(bad.any(axis=1))[0][0])
        raise ValueError("%s: pair %d %s names a cloud outside [0, %d)" % (who, p, tuple(arr[p].tolist()), n_clouds))
    return np.ascontiguousarray(arr, np.int32)


def match_keypoints(kp_or_desc, pairs, count=None):
    """Mutual nearest-neighbour matching of descriptors between cloud pairs.

    kp_or_desc: a KeypointSet (its descriptors and count), or desc [B,k,D] CUDA float32 with `count` [B] (slot j of
    cloud b is real iff j < clamp(count[b], 0, k)).
    pairs: [P,2] (src cloud, tgt cloud). A host list or array is range-checked against B (ValueError); a CUDA tensor
    is passed as it is, and a pair naming a cloud outside [0, B) then matches nothing.
    Returns Matches(nn_st, sim_st, nn_ts, sim_ts, matches, n_matches)."""
    if isinstance(kp_or_desc, KeypointSet):
        if count is not None:
            raise ValueError("match_keypoints: count comes from the KeypointSet")
        desc, count = kp_or_desc.descriptors, kp_or_desc.count
        if desc is None:
            raise ValueError("match_keypoints: the KeypointSet holds no descriptors")
    else:
        desc = kp_or_desc
        if count is None:
            raise ValueError("match_keypoints: descriptors [B,k,D] need `count`")
    if not torch.is_tensor(desc) or not desc.is_cuda or desc.dtype != torch.float32 or desc.dim() != 3:
        raise ValueError("match_keypoints: descriptors must be a CUDA float32 tensor [B,k,D]")
    desc = desc.contiguous()
    dev = desc.device
    B, k, D = (int(x) for x in desc.shape)
    cnt = _lib.i32(count, dev)
    if tuple(cnt.shape) != (B,):
        raise ValueError("match_keypoints: count %s does not match %d clouds" % (tuple(cnt.shape), B))
    if torch.is_tensor(pairs) and pairs.is_cuda:
        if pairs.dim() != 2 or int(pairs.shape[1]) != 2:
            raise ValueError("match_keypoints: pairs must be [P, 2], got %s" % (tuple(pairs.shape),))
        pr = pairs.to(dtype=torch.int32).contiguous()
    else:
        pairs = pairs.numpy() if torch.is_tensor(pairs) else pairs
        pr = torch.from_numpy(host_pairs(pairs, B)).to(dev)
    P = int(pr.shape[0])
    lib = _lib.lib()
    ws = _lib.workspace(lib.d3f_match_descriptors_workspace_bytes(k, P), dev)
    i32, f32 = torch.int32, torch.float32
    nn_st = torch.empty((P, k), dtype=i32, device=dev)
    sim_st = torch.empty((P, k), dtype=f32, device=dev)
    nn_ts = torch.empty((P, k), dtype=i32, device=dev)
    sim_ts = torch.empty((P, k), dtype=f32, device=dev)
    matches = torch.empty((P, k, 2), dtype=i32, device=dev)
    n_matches = torch.empty((P,), dtype=i32, device=dev)
    _lib.check(lib.d3f_match_descriptors(_lib.ptr(desc), _lib.ptr(cnt), B, k, D, _lib.ptr(pr), P, _lib.ptr(nn_st),
                                         _lib.ptr(sim_st), _lib.ptr(nn_ts), _lib.ptr(sim_ts), _lib.ptr(matches),
                                         _lib.ptr(n_matches), _lib.ptr(ws), ws.numel(), _lib.stream()),
               "d3f_match_descriptors")
    return Matches(nn_st, sim_st, nn_ts, sim_ts, matches, n_matches)
