"""Forward and backward of every KPConv layer shape of the bench workload step (8 x 30 000-point fragments).

    python scripts/kpconv_grad_bench.py --out DIR [--reps 20]

For each rigid KPConv of the encoder (the layers bench.py runs, captured with their real pyramid inputs), times with
CUDA events, L2 flushed before every call:
  * the forward (KPConv_ops),
  * the weight gradient alone (kpconv_backward(features_grad=False)),
  * the feature gradient alone, which includes one read-back of the reverse-table width,
and reports the weight-gradient kernels (wgrad_partial_kernel + wgrad_reduce_kernel, from torch.profiler in a run of
their own) against their bound: the larger of (bytes of wf and G read) / 3.35 TB/s and their flops / 67 TFLOP/s (FP32,
the data-sheet rate of the compute type used). Writes DIR/kpconv_grad_bench.json with the card's name and power limit.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

HBM = 3.35e12
FP32 = 67e12


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def capture_layers(dev):
    """(q, s, idx, f, Kp, W, extent, influence, mode) of every distinct rigid KPConv shape of one encoder step."""
    import torch
    from d3feat_b200 import convolution_ops as co, synth
    from d3feat_b200.encoder import KPFCNN
    cfg = synth.Config(architecture=synth.ARCH_ENCODER)
    clouds = [synth.room_fragment(i, 30000) for i in range(8)]
    pts = np.concatenate(clouds, 0).astype(np.float32)
    lens = np.array([len(c) for c in clouds], np.int32)
    enc = KPFCNN(cfg, synth.make_params(cfg, seed=0), [40] * 5, device=dev)
    seen, layers = set(), []
    orig = co.KPConv_ops

    def hook(q, s, idx, f, Kp, W, extent, influence, mode, **kw):
        key = (q.shape[0], s.shape[0], idx.shape[1], tuple(W.shape))
        if key not in seen:
            seen.add(key)
            layers.append((q, s, idx, f.clone(), Kp, W, extent, influence, mode))
        return orig(q, s, idx, f, Kp, W, extent, influence, mode, **kw)
    co.KPConv_ops = hook
    try:
        with torch.no_grad():
            enc(pts, lens)
    finally:
        co.KPConv_ops = orig
    torch.cuda.synchronize()
    return layers


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--reps", type=int, default=20)
    a = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile
    from d3feat_b200 import convolution_ops as co
    assert torch.cuda.is_available(), "the benchmark measures the GPU; there is no CPU fallback"
    dev = torch.device("cuda", 0)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    rows = []
    for q, s, idx, f, Kp, W, extent, infl, mode in capture_layers(dev):
        Nq, Ns, H = q.shape[0], s.shape[0], idx.shape[1]
        K, Cin, Cout = W.shape
        g = torch.randn((Nq, Cout), device=dev)
        calls = {
            "forward": lambda: co.KPConv_ops(q, s, idx, f, Kp, W, extent, infl, mode),
            "weight_grad": lambda: co.kpconv_backward(q, s, idx, f, Kp, W, extent, infl, mode, g, features_grad=False),
            "feature_grad": lambda: co.kpconv_backward(q, s, idx, f, Kp, W, extent, infl, mode, g, weights_grad=False),
        }
        res = dict(Nq=Nq, Ns=Ns, H=H, K=K, Cin=Cin, Cout=Cout)
        for name, fn in calls.items():
            fn(); fn()
            ts = []
            for _ in range(a.reps):
                flush.zero_()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                fn()
                e1.record()
                torch.cuda.synchronize()
                ts.append(e0.elapsed_time(e1))
            res[name + "_ms"] = float(np.median(ts))
        # the weight-gradient kernels alone, from the profiler
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(5):
                flush.zero_()
                calls["weight_grad"]()
            torch.cuda.synchronize()
        us = {}
        for e in prof.events():
            if e.device_type == torch.autograd.DeviceType.CUDA and "wgrad_" in e.name:
                key = "partial" if "partial" in e.name else "reduce"
                us.setdefault(key, []).append(e.device_time)
        kern_ms = sum(np.median(v) for v in us.values()) / 1e3 if us else float("nan")
        byts = 4.0 * Nq * (K * Cin + Cout)                         # wf and G, each read once
        flops = 2.0 * Nq * K * Cin * Cout
        bound_ms = max(byts / HBM, flops / FP32) * 1e3
        res.update(wgrad_kernels_ms=kern_ms, wgrad_bound_ms=bound_ms,
                   wgrad_bound="HBM" if byts / HBM > flops / FP32 else "FP32",
                   wgrad_share_of_bound=bound_ms / kern_ms if kern_ms == kern_ms else None)
        rows.append(res)
        print(json.dumps(res))
    out = dict(card=card(), layers=rows, note="CUDA events, L2 flushed (256 MB written) before every call, median of "
               "%d; weight-gradient kernels from torch.profiler" % a.reps)
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, "kpconv_grad_bench.json"), "w") as fh:
        json.dump(out, fh, indent=1)
    print(json.dumps(dict(card=out["card"])))


if __name__ == "__main__":
    main()
