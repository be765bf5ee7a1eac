"""GPU: what descriptor matching costs, as an op and inside a serving step. Writes OUT_DIR/match_bench.json and prints it.

Op: d3f_match_descriptors on P cloud pairs of k unit descriptors (D = 32, every slot real) for P in {1, 28} and k in
{250, 1000, 5000}. A CUDA graph of --reps back-to-back calls is replayed --iters times after a warm-up replay and timed
with CUDA events, so the host's launch cost is not in the number. The lower bound is the 2 * P * k^2 * D fp32
instructions of the contract (a separate multiply and add per channel: no FMA) at the data-sheet rate of the H100 SXM,
67 TFLOP/s = 33.5 T FMA instructions/s; it is derived, not measured. The host numpy restatement (oracle/match_np.py),
the same arithmetic one pair at a time, is timed on the same sizes, except P = 28 at k = 5000.

Pipeline: GraphPipeline(decoder=True, keypoints=250) with and without match_pairs = every i < j of bench.py's
8 x 30 000-point workload (28 pairs), in alternating runs, timed as scripts/keypoint_bench.py does. The card's name,
power limit and max SM clock are read in the same process.

    python scripts/match_bench.py --out DIR [--rounds 5] [--steps 24] [--warmup 6]
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(ROOT))
sys.path.insert(0, ROOT)

import numpy as np
import torch

from keypoint_bench import card_info, run

FMA_INSTR_PER_S = 33.5e12      # H100 SXM data sheet: 67 TFLOP/s fp32 = 33.5 T FMA instructions/s


def time_op(k, P, D, dev, reps, iters):
    """Device µs per d3f_match_descriptors call (graph of `reps` calls, median over `iters` replays)."""
    from d3feat_b200 import _lib
    lib = _lib.lib()
    rng = np.random.default_rng(k + P)
    B = 8
    d = rng.normal(size=(B, k, D)).astype(np.float32)
    d /= np.linalg.norm(d, axis=-1, keepdims=True)
    desc = torch.from_numpy(d).to(dev)
    count = torch.full((B,), k, dtype=torch.int32, device=dev)
    all_pairs = [(i, j) for i in range(B) for j in range(i + 1, B)]
    pairs = torch.tensor(all_pairs[:P], dtype=torch.int32, device=dev)
    out = [torch.empty(s, dtype=dt, device=dev) for s, dt in (
        ((P, k), torch.int32), ((P, k), torch.float32), ((P, k), torch.int32), ((P, k), torch.float32),
        ((P, k, 2), torch.int32), ((P,), torch.int32))]
    ws = _lib.workspace(lib.d3f_match_descriptors_workspace_bytes(k, P), dev)

    def call():
        _lib.check(lib.d3f_match_descriptors(_lib.ptr(desc), _lib.ptr(count), B, k, D, _lib.ptr(pairs), P,
                                             *[_lib.ptr(o) for o in out], _lib.ptr(ws), ws.numel(), _lib.stream()),
                   "d3f_match_descriptors")

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        call()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(reps):
            call()
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
    return float(np.median(per_call)), d, all_pairs[:P]


def time_host(d, pairs, repeats):
    from oracle import match_np
    count = np.full(d.shape[0], d.shape[1], np.int32)
    best = float("inf")
    for _ in range(repeats):
        t0 = time.perf_counter()
        match_np.match(d, count, pairs)
        best = min(best, time.perf_counter() - t0)
    return best * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="directory for match_bench.json")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=24)
    ap.add_argument("--warmup", type=int, default=6)
    ap.add_argument("--k", type=int, default=250, help="keypoints per cloud in the pipeline")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "match_bench.py needs a GPU"
    assert args.steps >= 20, "--steps: the median of at least 20 steps"

    from d3feat_b200 import synth, _lib
    from d3feat_b200.encoder import KPFCNN, GraphPipeline

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    _lib.lib()
    card = card_info()
    D = 32
    op = []
    for k in (250, 1000, 5000):
        for P in (1, 28):
            reps = max(1, min(200, int(4e9 / (2 * P * k * k * D))))
            us, d, pairs = time_op(k, P, D, dev, reps, iters=20)
            bound_us = 2 * P * k * k * D / FMA_INSTR_PER_S * 1e6
            host_ms = time_host(d, pairs, 3 if k <= 1000 else 1) if (k < 5000 or P == 1) else None
            op.append(dict(k=k, P=P, D=D, reps_per_graph=reps, device_us_per_call=us, lower_bound_us=bound_us,
                           share_of_bound=bound_us / us, host_numpy_restatement_ms=host_ms))
            print(json.dumps(op[-1]), flush=True)

    cfg = synth.Config(architecture=synth.ARCH_3DMATCH)
    clouds = [synth.room_fragment(i, 30000) for i in range(8)]
    P0 = torch.from_numpy(np.concatenate(clouds, 0)).to(dev)
    L0 = torch.from_numpy(np.array([c.shape[0] for c in clouds], np.int32)).to(dev)
    enc = KPFCNN(cfg, synth.make_params(cfg, 0), [40, 40, 40, 40, 40], device=dev)
    pairs = [(i, j) for i in range(8) for j in range(i + 1, 8)]
    pipes = {"keypoints": GraphPipeline.for_batch(enc, P0, L0, decoder=True, keypoints=args.k),
             "keypoints+match": GraphPipeline.for_batch(enc, P0, L0, decoder=True, keypoints=args.k,
                                                        match_pairs=pairs)}
    runs = {name: [] for name in pipes}
    for r in range(args.rounds):
        names = list(pipes) if r % 2 == 0 else list(pipes)[::-1]       # alternate which variant goes first
        for name in names:
            runs[name].append(run(pipes[name], P0, L0, args.steps, args.warmup))
    med = {name: float(np.median(v)) for name, v in runs.items()}
    res = dict(card=card, op=op,
               pipeline=dict(workload="8 x 30000-point synthetic fragments, ARCH_3DMATCH (encoder + decoder), limits 40",
                             k=args.k, pairs=len(pairs), steps=args.steps, warmup=args.warmup, rounds=args.rounds,
                             kernels_per_step={name: int(p.kernels_per_step) for name, p in pipes.items()},
                             runs_ms=runs, median_ms=med,
                             added_ms_per_step=med["keypoints+match"] - med["keypoints"]))
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "match_bench.json"), "w") as fh:
        json.dump(res, fh, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
