"""GPU: what the keypoint sweep costs. Writes OUT_DIR/keypoint_sweep_bench.json (timings, the card, and the sweep's
summary table of the last timed run) and prints it.

Pipeline: GraphPipeline(decoder=True, keypoints=5000, match_pairs, register, evaluate) with and without
sweep=dict(counts=(5000, 2500, 1000, 500, 250), arms=("score", "random")), in alternating runs on the same batch,
median step over `steps` steps after `warmup` (the timing of scripts/eval_bench.py), for
  * 3DMatch-shaped: 16 synthetic rooms of 30 000 points, every i < j pair (120), register={}, evaluate={};
  * KITTI-shaped: one pair of 20 000-point clouds, RANSAC (ransac_n 4), ICP, evaluate with repeat_distance 0.5.
Op: d3f_sample_keypoints alone at k = 5000 on the 3DMatch batch's level 0 (points, 32-d descriptors and scores
gathered), a CUDA graph of `reps` calls timed with CUDA events. The card's name, power limit and max SM clock are read
in the same process.

    python scripts/keypoint_sweep_bench.py --out DIR [--rounds 3] [--steps 20] [--warmup 4]
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(ROOT))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(os.path.dirname(ROOT), "tests"))

import numpy as np
import torch

from eval_bench import run
from keypoint_bench import card_info

COUNTS = (5000, 2500, 1000, 500, 250)
ARMS = ("score", "random")


def workloads(dev):
    """(name, points, lengths, truth, pipeline keyword arguments) of both workloads."""
    from d3feat_b200.evaluation import GroundTruth
    from test_gpu_evaluation import info_matrices
    from test_gpu_keypoint_sweep import scene
    from d3feat_b200 import synth
    d = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)     # noqa: E731
    rooms = [synth.room_fragment(i, 30000) for i in range(16)]
    pairs = [(i, j) for i in range(16) for j in range(i + 1, 16)]
    truth = GroundTruth(d(np.tile(np.eye(4), (len(pairs), 1, 1))), d(info_matrices(len(pairs))),
                        d(np.full(len(pairs), 3, np.int32)))
    out = [("3dmatch_16x30000", d(np.concatenate(rooms, 0)), d(np.array([30000] * 16, np.int32)), truth,
            dict(match_pairs=pairs, register={}, evaluate={}))]
    P, L, kp_pairs, T = scene(900, 2, 20000, keep=0.9)
    T = GroundTruth(d(T.pose), None, d(T.flags))
    out.append(("kitti_pair_2x20000", d(P), d(L), T,
                dict(match_pairs=kp_pairs, register=dict(ransac_n=4, distance=0.3, max_iterations=50000),
                     icp=dict(distance=0.3), evaluate=dict(repeat_distance=0.5))))
    return out


def time_sampler(P, L, desc, scores, reps, iters):
    """Device µs per d3f_sample_keypoints call at k = COUNTS[0] (graph of `reps` calls, median over `iters`)."""
    from d3feat_b200.keypoints import sample_keypoints
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        sample_keypoints(L, COUNTS[0], 0, points=P, descriptors=desc, scores=scores)
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(reps):
            sample_keypoints(L, COUNTS[0], 0, points=P, descriptors=desc, scores=scores)
    g.replay()
    torch.cuda.synchronize()
    per_call = []
    for _ in range(iters):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        g.replay()
        e1.record()
        e1.synchronize()
        per_call.append(e0.elapsed_time(e1) * 1e3 / reps)
    return float(np.median(per_call))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="directory for keypoint_sweep_bench.json")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=4)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "keypoint_sweep_bench.py needs a GPU"
    assert args.steps >= 10, "--steps: the median of at least 10 steps"

    from d3feat_b200 import synth, _lib
    from d3feat_b200.encoder import KPFCNN, GraphPipeline
    from d3feat_b200.evaluation import sweep_summary

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    _lib.lib()
    card = card_info()
    print(json.dumps(card), flush=True)
    cfg = synth.Config(architecture=synth.ARCH_3DMATCH)
    enc = KPFCNN(cfg, synth.make_params(cfg, 0), [40, 40, 40, 40, 40], device=dev)
    res = dict(card=card, counts=list(COUNTS), arms=list(ARMS), steps=args.steps, warmup=args.warmup,
               rounds=args.rounds, workloads={})
    for name, P, L, truth, kw in workloads(dev):
        kw = dict(decoder=True, keypoints=COUNTS[0], **kw)
        pipes = {"single": GraphPipeline.for_batch(enc, P, L, **kw),
                 "sweep": GraphPipeline.for_batch(enc, P, L, sweep=dict(counts=COUNTS, arms=ARMS), **kw)}
        runs = {v: [] for v in pipes}
        for r in range(args.rounds):
            for v in (list(pipes) if r % 2 == 0 else list(pipes)[::-1]):     # alternate which variant goes first
                pipes[v].reset_evaluation()
                runs[v].append(run(pipes[v], P, L, truth, args.steps, args.warmup))
        med = {v: float(np.median(x)) for v, x in runs.items()}
        sw = pipes["sweep"]
        table = sweep_summary(sw.evaluation_totals(), sw.sweep_arms, sw.sweep_counts, sw.evaluate_levels,
                              sw.evaluate_pose_sets)
        row = dict(pairs=len(kw["match_pairs"]), clouds=int(L.shape[0]), points=int(P.shape[0]),
                   kernels_per_step={v: int(p.kernels_per_step) for v, p in pipes.items()}, runs_ms=runs,
                   median_ms=med, sweep_over_single=med["sweep"] / med["single"], summary=table)
        if name.startswith("3dmatch"):
            inputs, _, det = sw.out[0]                 # slot 0's level 0 and network outputs
            desc, scores = det.descriptors, det.scores
            row["sample_keypoints_us"] = time_sampler(inputs["points"][0], inputs["lengths"][0], desc, scores,
                                                      reps=20, iters=7)
        res["workloads"][name] = row
        print(json.dumps({name: {f: v for f, v in row.items() if f != "summary"}}), flush=True)
        for r in table:
            print("%-22s %-6s %5d  FMR %.3f  inlier ratio %.4f  repeat@%d %.3f" % (
                name, r["arm"], r["count"], r["fmr"], r["avg_inlier_ratio"], max(r["repeatability"]),
                r["repeatability"][max(r["repeatability"])]), flush=True)
        del pipes, sw
        torch.cuda.synchronize()
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "keypoint_sweep_bench.json"), "w") as fh:
        json.dump(res, fh, indent=1, default=float)
    print("wrote %s" % os.path.join(args.out, "keypoint_sweep_bench.json"))


if __name__ == "__main__":
    main()
