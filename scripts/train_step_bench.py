"""One D3Feat training step on the GPU: a pair of 30 000-point synth.room_fragment scenes (the second a rigidly moved
copy of the first), the 3DMatch architecture and training configuration, 256 keypoint correspondences.

    python scripts/train_step_bench.py --out DIR [--steps 20] [--warmup 3]

Run 1 (no profiler): forward, loss and backward of each step timed with CUDA events; medians over --steps steps after
--warmup steps. The step includes no optimiser update, so every step sees the same parameters (the moving statistics
still move). Run 2 (torch.profiler, 2 steps): the device time of each kernel of the new training ops, against its HBM
bound: the bytes each kernel must move (every input read once, every output written once, computed from the shapes of
the calls the step made) over 3.35 TB/s. The reverse-table kernels (sort and scan) are shared with the KPConv backward
and reported as one total. Writes DIR/train_step_bench.json with the card's name and power limit.
"""
import argparse
import collections
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

HBM = 3.35e12


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def workload(dev):
    import torch
    from d3feat_b200 import pyramid, synth, training as T
    from d3feat_b200.encoder import KPFCNN
    cfg = synth.Config(**T.TRAINING_3DMATCH)
    n = 30000
    a = synth.room_fragment(0, n)
    th = 0.3
    R = np.array([[np.cos(th), -np.sin(th), 0], [np.sin(th), np.cos(th), 0], [0, 0, 1]])
    b = (a @ R.T + np.array([0.5, -0.2, 0.1])).astype(np.float32)
    limits = pyramid.calibrate_neighbors(cfg, [a], device=dev)
    enc = KPFCNN(cfg, synth.make_params(cfg, seed=0), limits, device=dev)
    inputs = enc.build_inputs(np.concatenate([a, b]), np.array([n, n], np.int32))
    anc = np.random.default_rng(0).choice(n, cfg.keypts_num, replace=True).astype(np.int32)
    anc_t = torch.as_tensor(anc).to(dev)
    return cfg, enc.store, inputs, anc_t, anc_t + n, limits


def step(cfg, store, inputs, anc, pos, events=None):
    from d3feat_b200 import training as T
    from d3feat_b200.variables import use_params
    for t in store.t.values():
        t.grad = None
    ev = events or [None] * 4
    rec = lambda i: ev[i] is not None and ev[i].record()
    rec(0)
    with use_params(store):
        desc, scores = T.forward(inputs, cfg)
        rec(1)
        loss = T.d3feat_loss(desc, scores, anc, pos, inputs["points"][0], cfg)[0]
    rec(2)
    loss.backward()
    rec(3)
    return loss


# kernel name -> (op, bytes of one call from the call's shapes); b = 4 bytes per float / int
def kernel_bytes(op, s):
    f = 4
    if op == "batch_norm_forward":
        N, C, res = s
        return {"colsum_partial_kernel<0>": f * N * C, "colsum_partial_kernel<1>": f * N * C,
                "affine_leaky_kernel": f * N * C * (2 + res)}
    if op == "batch_norm_backward":
        N, C, res = s
        return {"colsum_partial_kernel<2>": 3 * f * N * C, "bn_dx_kernel": f * N * C * (4 + res)}
    if op == "ind_max_pool_backward":
        N1, N2, H, C = s
        return {"colmin_pass_kernel": 2 * f * N1 * C, "maxpool_share_kernel": f * (N2 * H + 3 * N2 * C + N1 * C),
                "maxpool_gather_kernel": f * (2 * N1 * C + 2 * N2 * C + N2 * H + 2 * N1)}
    if op == "gather_rows_backward":
        N1, N2, C = s
        return {"gather_rows_grad_kernel": f * (N2 * C + N1 * C + N2 + 2 * N1)}
    if op == "l2_normalize_backward":
        N, C = s
        return {"l2_normalize_grad_kernel": 3 * f * N * C}
    if op == "detection_scores_backward":
        N, H, Dm = s
        return {"det_rowmax_kernel": f * N * Dm, "det_row_grad_kernel": f * (N * Dm * 5 + N * H + N),
                "det_gather_kernel": f * (4 * N * Dm + N * H + 2 * N)}
    return {}


def record_calls(calls):
    """Wrap the training entry points to log the shapes of every call the step makes."""
    from d3feat_b200 import training as T
    shapes = {
        "batch_norm_forward": lambda x, *a, **k: (x.shape[0], x.shape[1], int((a[5] if len(a) > 5 else k.get("residual"))
                                                                             is not None)),
        "batch_norm_backward": lambda x, out, g, *a, **k: (x.shape[0], x.shape[1], int(k.get("residual_grad", False))),
        "ind_max_pool_backward": lambda x, inds, *a: (x.shape[0], inds.shape[0], inds.shape[1], x.shape[1]),
        "gather_rows_backward": lambda inds, g, n: (int(n), inds.shape[0], g.shape[1]),
        "l2_normalize_backward": lambda x, g: tuple(x.shape),
        "detection_scores_backward": lambda x, nb, *a: (x.shape[0], nb.shape[1], x.shape[1]),
    }
    for name, sh in shapes.items():
        fn = getattr(T, name)

        def wrapped(*a, _fn=fn, _name=name, _sh=sh, **k):
            calls.append((_name, _sh(*a, **k)))
            return _fn(*a, **k)
        setattr(T, name, wrapped)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("train_step_bench.py needs a GPU")
    dev = torch.device("cuda", 0)
    cfg, store, inputs, anc, pos, limits = workload(dev)
    from d3feat_b200 import training as T
    T.trainable(store)
    for _ in range(args.warmup):
        step(cfg, store, inputs, anc, pos)
    torch.cuda.synchronize()
    times = []
    for _ in range(args.steps):
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
        step(cfg, store, inputs, anc, pos, ev)
        torch.cuda.synchronize()
        times.append([ev[0].elapsed_time(ev[1]), ev[1].elapsed_time(ev[2]), ev[2].elapsed_time(ev[3]),
                      ev[0].elapsed_time(ev[3])])
    med = np.median(np.array(times), axis=0)

    calls = []
    record_calls(calls)
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(2):
            step(cfg, store, inputs, anc, pos)
        torch.cuda.synchronize()
    kt = collections.defaultdict(float)
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA:
            kt[e.name] += e.device_time / 1e3 / 2          # ms per step
    need = collections.defaultdict(float)
    for op, s in calls:
        for k, b in kernel_bytes(op, s).items():
            need[k] += b / 2                               # bytes per step
    rows = []
    for k, b in sorted(need.items()):
        t = sum(v for n, v in kt.items() if k in n)
        rows.append(dict(kernel=k, ms=t, bytes=b, hbm_bound_ms=b / HBM * 1e3,
                         share_of_hbm_bound=(b / HBM * 1e3) / t if t > 0 else None))
    shared = sum(v for n, v in kt.items() if any(s in n for s in ("reverse_keys", "radix", "scan", "sort")))
    total_ms = sum(kt.values())
    res = dict(card=card(), workload="2 x 30000-point room_fragment, 3DMatch config, %d correspondences" % cfg.keypts_num,
               neighborhood_limits=limits, level_sizes=[int(p.shape[0]) for p in inputs["points"]],
               step_ms=dict(forward=med[0], loss=med[1], backward=med[2], total=med[3]), steps=args.steps,
               kernels=rows, reverse_table_sort_scan_ms=shared, profiled_device_ms_per_step=total_ms)
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "train_step_bench.json"), "w") as fh:
        json.dump(res, fh, indent=1)
    print(json.dumps(res["step_ms"]), res["card"])
    for r in rows:
        print("%-28s %8.3f ms  bound %7.3f ms  share %s" % (r["kernel"], r["ms"], r["hbm_bound_ms"],
                                                           "%.2f" % r["share_of_hbm_bound"] if r["share_of_hbm_bound"]
                                                           else "-"))
    print("reverse-table sort + scan (shared with the KPConv backward): %.3f ms per step" % shared)


if __name__ == "__main__":
    main()
