"""GPU: what keypoint selection adds to a serving step. Builds bench.py's workload (8 stacked synthetic fragments x
30 000 points, 40 neighbour columns, the same seeds) with the synthetic 3DMatch decoder parameters and times
GraphPipeline(decoder=True) against GraphPipeline(decoder=True, keypoints=250) in alternating runs, each after its
own warm-up. A step's time is the interval between consecutive end-of-step events on the caller's stream, averaged
over a window of as many steps as there are encoder streams (consecutive encoders alternate between them); every run
reports the median of its steps. The card's name, power limit and max SM clock are read in the same process.
Writes OUT_DIR/keypoint_bench.json and prints it.

    python scripts/keypoint_bench.py --out DIR [--steps 24] [--warmup 6] [--rounds 3] [--k 250]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np
import torch


def card_info():
    q = "name,power.limit,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=" + q, "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, power, clock = [x.strip() for x in out.split(",")]
    except (OSError, ValueError, subprocess.SubprocessError):
        name, power, clock = torch.cuda.get_device_name(0), "unknown", "unknown"
    return dict(name=name, power_limit=power, max_sm_clock=clock)


def run(pipe, P, L, steps, warmup):
    """Median per-step ms of `steps` pipelined steps after `warmup` untimed ones."""
    pipe.prime(P, L)
    for _ in range(warmup):
        pipe.step(P, L)
    pipe.drain()
    torch.cuda.synchronize()
    marks = [torch.cuda.Event(enable_timing=True) for _ in range(steps + 1)]
    marks[0].record()
    for i in range(steps):
        pipe.step(P, L)                     # the caller's stream waits for this step's result
        marks[i + 1].record()
    pipe.drain()
    torch.cuda.synchronize()
    pipe.check()
    w = min(len(pipe.s_encs), steps)
    per_step = [marks[i].elapsed_time(marks[i + w]) / w for i in range(steps - w + 1)]
    return float(np.median(per_step))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="directory for keypoint_bench.json")
    ap.add_argument("--steps", type=int, default=24)
    ap.add_argument("--warmup", type=int, default=6)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--k", type=int, default=250)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "keypoint_bench.py needs a GPU"
    assert args.steps >= 20, "--steps: the median of at least 20 steps"

    from d3feat_b200 import synth, _lib
    from d3feat_b200.encoder import KPFCNN, GraphPipeline

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    _lib.lib()
    cfg = synth.Config(architecture=synth.ARCH_3DMATCH)
    limits = [40, 40, 40, 40, 40]
    clouds = [synth.room_fragment(i, 30000) for i in range(8)]
    P = torch.from_numpy(np.concatenate(clouds, 0)).to(dev)
    L = torch.from_numpy(np.array([c.shape[0] for c in clouds], np.int32)).to(dev)
    enc = KPFCNN(cfg, synth.make_params(cfg, 0), limits, device=dev)
    pipes = {"decoder": GraphPipeline.for_batch(enc, P, L, decoder=True),
             "decoder+keypoints": GraphPipeline.for_batch(enc, P, L, decoder=True, keypoints=args.k)}
    card = card_info()
    runs = {name: [] for name in pipes}
    for r in range(args.rounds):
        names = list(pipes) if r % 2 == 0 else list(pipes)[::-1]       # alternate which variant goes first
        for name in names:
            runs[name].append(run(pipes[name], P, L, args.steps, args.warmup))
    med = {name: float(np.median(v)) for name, v in runs.items()}
    res = dict(card=card, workload="8 x 30000-point synthetic fragments, ARCH_3DMATCH (encoder + decoder), limits 40",
               k=args.k, steps=args.steps, warmup=args.warmup, rounds=args.rounds,
               kernels_per_step={name: int(p.kernels_per_step) for name, p in pipes.items()},
               runs_ms=runs, median_ms=med, added_ms_per_step=med["decoder+keypoints"] - med["decoder"])
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "keypoint_bench.json"), "w") as fh:
        json.dump(res, fh, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
