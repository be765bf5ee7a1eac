"""Training pairs on the GPU against the reference's host searches, on the same data.

    python scripts/train_pairs_bench.py --out DIR [--steps 20] [--warmup 3]

GPU (medians over --steps calls after --warmup, host clock around a device synchronise):
  * training_pairs on a KITTI-like pair: a 16 000-point synth.lidar_scan (voxel 0.30) and its rigidly moved copy,
    "kitti" (radius correspondences at tau = 0.45, 1024 keypoints without replacement, noise, rotation, scale and
    shift);
  * the all-pairs "nearest" overlap table over 16 synth.room_fragment scenes of 10 000 points at tau = 0.03
    (120 pairs, one correspondences call).
Host (labelled as host timings; not the reference's own code): scipy's cKDTree query_ball_point for the KITTI pair,
standing in for Open3D's per-point KD-tree loop, and, for the table, cKDTree nearest queries over all 120 pairs and
cv2.BFMatcher(NORM_L2).match on the first BF_PAIRS pairs (reported per pair). Writes DIR/train_pairs_bench.json with
the card's name and power limit.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

BF_PAIRS = 8


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def timed(fn, steps, warmup, sync):
    for _ in range(warmup):
        fn()
    sync()
    ts = []
    for _ in range(steps):
        t0 = time.perf_counter()
        fn()
        sync()
        ts.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    import torch
    from scipy.spatial import cKDTree
    from d3feat_b200 import synth, training as T, training_data as td
    if not torch.cuda.is_available():
        raise SystemExit("train_pairs_bench: no CUDA device")
    dev = torch.device("cuda", 0)
    sync = torch.cuda.synchronize
    res = dict(card=card())

    # KITTI-like pair
    a = synth.lidar_scan(0, 16000)
    th = 0.1
    M = np.eye(4)
    M[:3, :3] = [[np.cos(th), -np.sin(th), 0], [np.sin(th), np.cos(th), 0], [0, 0, 1]]
    M[:3, 3] = [2.0, 0.5, 0.0]
    b = (a.astype(np.float64) @ M[:3, :3].T + M[:3, 3]).astype(np.float32)
    pts = torch.as_tensor(np.concatenate([a, b])).to(dev)
    lens = torch.tensor([len(a), len(b)], dtype=torch.int32, device=dev)
    pairs = torch.tensor([[0, 1]], dtype=torch.int32, device=dev)
    trans = torch.as_tensor(M[None]).to(dev)
    cfg = synth.Config(**T.TRAINING_KITTI)
    bbox = np.concatenate([np.minimum(a.min(0), b.min(0)), np.maximum(a.max(0), b.max(0))]).astype(np.float32)
    tp = td.training_pairs(pts, lens, pairs, trans, cfg, "kitti", 0, bbox=bbox)
    res["kitti_pair"] = dict(points=[len(a), len(b)], correspondences=int(tp.count[0]), valid=bool(tp.valid[0]),
                             gpu_training_pairs_ms=timed(
                                 lambda: td.training_pairs(pts, lens, pairs, trans, cfg, "kitti", 0, bbox=bbox),
                                 args.steps, args.warmup, sync))
    q = a.astype(np.float64) @ M[:3, :3].T + M[:3, 3]
    t0 = time.perf_counter()
    cKDTree(b.astype(np.float64)).query_ball_point(q, 0.45)
    res["kitti_pair"]["host_ckdtree_ms"] = (time.perf_counter() - t0) * 1e3

    # all-pairs overlap table
    frags = [synth.room_fragment(s, 10000) for s in range(16)]
    P = [[i, j] for i in range(16) for j in range(i + 1, 16)]
    fp = torch.as_tensor(np.concatenate(frags)).to(dev)
    fl = torch.tensor([len(f) for f in frags], dtype=torch.int32, device=dev)
    fpairs = torch.tensor(P, dtype=torch.int32, device=dev)
    ftrans = torch.eye(4, dtype=torch.float64, device=dev).repeat(len(P), 1, 1)
    cat = np.concatenate(frags)
    fbox = np.concatenate([cat.min(0), cat.max(0)]).astype(np.float32)
    c = td.correspondences(fp, fl, fpairs, ftrans, 0.03, "nearest", bbox=fbox)
    res["overlap_table"] = dict(fragments=16, points=10000, pairs=len(P), correspondences=int(c.offset[-1]),
                                gpu_ms=timed(lambda: td.correspondences(fp, fl, fpairs, ftrans, 0.03, "nearest",
                                                                        bbox=fbox),
                                             args.steps, args.warmup, sync))
    t0 = time.perf_counter()
    trees = [cKDTree(f.astype(np.float64)) for f in frags]
    for i, j in P:
        trees[j].query(frags[i].astype(np.float64), k=1, distance_upper_bound=0.03)
    res["overlap_table"]["host_ckdtree_ms"] = (time.perf_counter() - t0) * 1e3
    try:
        import cv2
        bf = cv2.BFMatcher(cv2.NORM_L2)
        t0 = time.perf_counter()
        for i, j in P[:BF_PAIRS]:
            bf.match(frags[i], frags[j])
        res["overlap_table"]["host_bfmatcher_ms_per_pair"] = (time.perf_counter() - t0) * 1e3 / BF_PAIRS
    except ImportError:
        res["overlap_table"]["host_bfmatcher_ms_per_pair"] = "not measured (no cv2)"
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "train_pairs_bench.json"), "w") as fh:
        json.dump(res, fh, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
