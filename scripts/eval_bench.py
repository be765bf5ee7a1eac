"""GPU: what the ground-truth metrics cost, as an op and inside a serving step. Writes OUT_DIR/eval_bench.json and
prints it.

Op: d3f_evaluate_pairs with both pose sets (RANSAC and ICP poses) and Choi information matrices, on
  * P = 28 (every i < j of 8 fragments), k = 250, levels 4 .. 128 and 250 (a 3DMatch scene batch);
  * P = 1770 (every i < j of one 60-fragment scene), k = 250, the same levels;
  * P = 28, k = 5000, levels 4 .. 4096 and 5000 (the repeatability sweep at its largest);
keypoints are noisy rigid copies of one set (tests/test_gpu_evaluation.py's make_case), every pair flagged for FMR and
recall. A CUDA graph of `reps` back-to-back calls is replayed after a warm-up replay and timed with CUDA events; the
host numpy restatement (oracle/evaluate_np.py) is timed on the same input and compared with the device result.

Pipeline: GraphPipeline(decoder=True, keypoints=250, match_pairs = every i < j of 8 x 30 000-point clouds,
register={}) with and without evaluate={}, in alternating runs, median step over `steps` steps after `warmup`, as
scripts/keypoint_bench.py times them. The card's name, power limit and max SM clock are read in the same process.

    python scripts/eval_bench.py --out DIR [--rounds 5] [--steps 24] [--warmup 6]
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(ROOT))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(os.path.dirname(ROOT), "tests"))

import numpy as np
import torch

from keypoint_bench import card_info

DEFAULT = (4, 8, 16, 32, 64, 128)


def make_op_case(n_frag, k, levels):
    from test_gpu_evaluation import info_matrices, make_case
    rng = np.random.default_rng(n_frag * 7 + k)
    pairs = [(i, j) for i in range(n_frag) for j in range(i + 1, n_frag)]
    pts, cnt, matches, n_m, G, poses = make_case(rng, k, [k] * n_frag, pairs)
    return dict(points=pts, count=cnt, matches=matches, n_matches=n_m, pairs=np.array(pairs), pose=G,
                info=info_matrices(len(pairs)), flags=np.full(len(pairs), 3), poses=poses, levels=levels)


def time_op(case, dev, reps, iters):
    """Device µs per d3f_evaluate_pairs call (graph of `reps` calls, median over `iters` replays), the kernels of one
    call and the outputs."""
    from d3feat_b200 import _lib
    from d3feat_b200.evaluation import Evaluation, GroundTruth, evaluate_pairs
    from d3feat_b200.keypoints import KeypointSet
    from d3feat_b200.matching import Matches
    from d3feat_b200.registration import Refinement, Registration
    d = lambda a, dt: torch.from_numpy(np.ascontiguousarray(a, dt)).to(dev)   # noqa: E731
    kp = KeypointSet(None, d(case["count"], np.int32), d(case["points"], np.float32), None, None)
    m = Matches(None, None, None, None, d(case["matches"], np.int32), d(case["n_matches"], np.int32))
    truth = GroundTruth(d(case["pose"], np.float64), d(case["info"], np.float64), d(case["flags"], np.int32))
    reg = Registration(d(case["poses"][0], np.float64), None, None, None, None)
    ref = Refinement(d(case["poses"][1], np.float64), None, None, None, None)
    pr = d(case["pairs"], np.int32)
    opts = dict(repeat_levels=case["levels"])
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        evaluate_pairs(kp, m, pr, truth, reg, ref, **opts)
    torch.cuda.current_stream().wait_stream(s)
    n0 = _lib.launch_count()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(reps):
            ev = evaluate_pairs(kp, m, pr, truth, reg, ref, **opts)
    kernels = (_lib.launch_count() - n0) // reps
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
    return float(np.median(per_call)), kernels, {f: getattr(ev, f).cpu().numpy() for f in Evaluation._fields}


def run(pipe, P, L, truth, steps, warmup):
    """Median per-step ms of `steps` pipelined steps after `warmup` untimed ones (keypoint_bench.run with truth)."""
    kw = {} if truth is None else dict(truth=truth)
    nkw = {} if truth is None else dict(next_truth=truth)
    pipe.prime(P, L, **kw)
    for _ in range(warmup):
        pipe.step(P, L, **nkw)
    pipe.drain()
    torch.cuda.synchronize()
    marks = [torch.cuda.Event(enable_timing=True) for _ in range(steps + 1)]
    marks[0].record()
    for i in range(steps):
        pipe.step(P, L, **nkw)
        marks[i + 1].record()
    pipe.drain()
    torch.cuda.synchronize()
    pipe.check()
    w = min(len(pipe.s_encs), steps)
    per_step = [marks[i].elapsed_time(marks[i + w]) / w for i in range(steps - w + 1)]
    return float(np.median(per_step))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="directory for eval_bench.json")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=24)
    ap.add_argument("--warmup", type=int, default=6)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "eval_bench.py needs a GPU"
    assert args.steps >= 20, "--steps: the median of at least 20 steps"

    from d3feat_b200 import synth, _lib
    from d3feat_b200.encoder import KPFCNN, GraphPipeline
    from d3feat_b200.evaluation import GroundTruth
    from oracle import evaluate_np
    from test_gpu_evaluation import OPTS, mismatches

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    _lib.lib()
    card = card_info()
    print(json.dumps(card), flush=True)
    op = []
    for n_frag, k, levels, reps in ((8, 250, DEFAULT + (250,), 20), (60, 250, DEFAULT + (250,), 5),
                                    (8, 5000, DEFAULT + (256, 512, 1024, 2048, 4096, 5000), 3)):
        case = make_op_case(n_frag, k, levels)
        us, kernels, got = time_op(case, dev, reps=reps, iters=7)
        t0 = time.perf_counter()
        want = evaluate_np.evaluate(case["points"], case["count"], case["matches"], case["n_matches"], case["pairs"],
                                    case["pose"], case["info"], case["flags"], case["poses"], levels=levels, **OPTS)
        host_ms = (time.perf_counter() - t0) * 1e3
        row = dict(P=len(case["pairs"]), k=k, levels=list(levels), device_us_per_call=us, kernels_per_call=kernels,
                   host_numpy_restatement_ms=host_ms,
                   equal_to_restatement=mismatches(got, want, len(levels), 2) == [],
                   fmr_hits=int(want["totals"][1]), successes=[int(want["totals"][4 + len(levels) + 7 * s])
                                                               for s in range(2)])
        op.append(row)
        print(json.dumps(row), flush=True)

    cfg = synth.Config(architecture=synth.ARCH_3DMATCH)
    clouds = [synth.room_fragment(i, 30000) for i in range(8)]
    P0 = torch.from_numpy(np.concatenate(clouds, 0)).to(dev)
    L0 = torch.from_numpy(np.array([c.shape[0] for c in clouds], np.int32)).to(dev)
    enc = KPFCNN(cfg, synth.make_params(cfg, 0), [40, 40, 40, 40, 40], device=dev)
    pairs = [(i, j) for i in range(8) for j in range(i + 1, 8)]
    truth = GroundTruth(torch.eye(4, dtype=torch.float64, device=dev).repeat(len(pairs), 1, 1),
                        torch.from_numpy(make_op_case(8, 250, DEFAULT)["info"]).to(dev),
                        torch.full((len(pairs),), 3, dtype=torch.int32, device=dev))
    kw = dict(decoder=True, keypoints=250, match_pairs=pairs, register={})
    pipes = {"register": (GraphPipeline.for_batch(enc, P0, L0, **kw), None),
             "register+evaluate": (GraphPipeline.for_batch(enc, P0, L0, evaluate={}, **kw), truth)}
    runs = {name: [] for name in pipes}
    for r in range(args.rounds):
        names = list(pipes) if r % 2 == 0 else list(pipes)[::-1]       # alternate which variant goes first
        for name in names:
            pipe, tr = pipes[name]
            runs[name].append(run(pipe, P0, L0, tr, args.steps, args.warmup))
    med = {name: float(np.median(v)) for name, v in runs.items()}
    res = dict(card=card, op=op,
               pipeline=dict(workload="8 x 30000-point synthetic fragments, ARCH_3DMATCH (encoder + decoder), limits 40",
                             k=250, pairs=len(pairs), steps=args.steps, warmup=args.warmup, rounds=args.rounds,
                             kernels_per_step={name: int(p.kernels_per_step) for name, (p, _) in pipes.items()},
                             runs_ms=runs, median_ms=med,
                             added_ms_per_step=med["register+evaluate"] - med["register"]))
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "eval_bench.json"), "w") as fh:
        json.dump(res, fh, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
