"""Time the kernel-point optimiser: load_kernels' 100 tries of K points (K = 15, 32, 64) on the GPU, with CUDA events
after a warm-up, and the float64 numpy restatement (oracle/kernel_points_np.py) on the host, from the same seeded
initial points. Writes DIR/kernel_points_bench.json and prints it.

    python scripts/kernel_points_bench.py --out DIR [--ks 15,32,64] [--host-ks 15,32,64] [--reps 3]

The GPU part needs a CUDA device (it never falls back) and reads the card's name and power limit in the same run.
--host-ks '' skips the host timing, which takes minutes for K = 64.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import kernel_points_np as O  # noqa: E402

TRIES = 100


def initial(K, seed=0):
    from d3feat_b200 import kernel_points as kp
    return kp.initial_points(K, TRIES, seed, "center")


def gpu_card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def time_gpu(ks, reps):
    import torch
    from d3feat_b200 import kernel_points as kp
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: the GPU timing does not fall back")
    dev = torch.device("cuda", 0)
    out = {}
    for K in ks:
        x = torch.from_numpy(initial(K)).to(dev)
        _, _, n = kp.optimize(x, "center")                 # warm-up: module load, shared-memory attribute
        torch.cuda.synchronize()
        ms = []
        for _ in range(reps):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            _, _, n = kp.optimize(x, "center")
            b.record()
            b.synchronize()
            ms.append(a.elapsed_time(b))
        it = int(n)
        out[K] = {"iterations": it, "ms": ms, "ms_median": float(np.median(ms)),
                  "us_per_iteration": 1e3 * float(np.median(ms)) / it}
        print("gpu K=%d: %d iterations, %.1f ms (median of %d)" % (K, it, np.median(ms), reps), flush=True)
    return out


def time_host(ks):
    out = {}
    for K in ks:
        x = initial(K)
        t = time.perf_counter()
        _, _, n = O.optimize(x, "center")
        s = time.perf_counter() - t
        out[K] = {"iterations": int(n), "s": s}
        print("host K=%d: %d iterations, %.1f s" % (K, n, s), flush=True)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--ks", default="15,32,64")
    ap.add_argument("--host-ks", default="15,32,64")
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    ks = [int(k) for k in args.ks.split(",") if k]
    host_ks = [int(k) for k in args.host_ks.split(",") if k]
    res = {"tries": TRIES, "fixed": "center"}
    if ks:
        res["card"] = gpu_card()
        res["gpu"] = time_gpu(ks, args.reps)
    if host_ks:
        import platform
        res["host_cpu"] = platform.processor() or platform.machine()
        res["host"] = time_host(host_ks)
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "kernel_points_bench.json"), "w") as fh:
        json.dump(res, fh, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
