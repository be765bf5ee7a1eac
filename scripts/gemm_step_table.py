"""GPU: every GEMM one step of bench.py's default workload (8 x 30k points, 5-level encoder) issues, timed alone and
set against the least time the hardware could take for its shape.

The shapes come from a hooked eager pass of the encoder (the same hooks as bench.py's roofline section): unary and
[A | A2] pair GEMMs as they are called, and for every KPConv its contraction [Nq, K*Cin] x [K*Cin, Cout] on a buffer
of the size of the real weighted-feature matrix. Each is timed through the Python entry points with CUDA events, warm,
an L2 flush before every launch, median of --reps launches.

Bound of a shape (derived from the data sheet of the H100 SXM, not measured): the larger of
  minimum bytes / 3.35 TB/s     (A once, the packed hi/lo weight once, C once, the residual once)
  3 * 2 M K N flops / 495 TFLOP/s (three TF32 products per fp32 product)

    python scripts/gemm_step_table.py --out DIR [--reps 50]
    python scripts/gemm_step_table.py --dry-run        # no GPU: nominal level sizes, shapes and bounds only
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np

HBM_BYTES_PER_S = 3.35e12     # H100 SXM data sheet
TF32_FLOPS = 495e12           # H100 SXM data sheet, dense TF32
NOMINAL_ROWS = [240000, 60336, 15200, 4177, 1204]   # level sizes of the 8 x 30k batch, for --dry-run


def gemm_bound(M, K, N, residual=False):
    """(bound in us, 'hbm' or 'tensor', minimum bytes, flops x 3) of C[M,N] = A[M,K] @ W[K,N] in 3xTF32."""
    nbytes = 4.0 * (M * K + 2 * K * N + M * N * (2 if residual else 1))
    flops3 = 3 * 2.0 * M * K * N
    t_mem, t_mma = nbytes / HBM_BYTES_PER_S * 1e6, flops3 / TF32_FLOPS * 1e6
    return max(t_mem, t_mma), ("hbm" if t_mem >= t_mma else "tensor"), nbytes, flops3


def shape_row(kind, M, K, N, K2=0, flags="", row_map=False, residual=False):
    bound, which, nbytes, flops3 = gemm_bound(M, K + K2, N, residual)
    return dict(kind=kind, M=M, K=K, K2=K2, N=N, flags=flags, row_map=row_map, min_bytes=nbytes, flops_x3=flops3,
                bound_us=bound, bound_by=which)


def nominal_shapes(cfg):
    """The GEMMs of the encoder walked the way assemble_CNN_blocks walks it, at NOMINAL_ROWS."""
    rows, layer, fdim, cin = [], 0, cfg.first_features_dim, cfg.in_features_dim
    kp = cfg.num_kernel_points
    for block in cfg.architecture:
        if "upsample" in block:
            break
        m = NOMINAL_ROWS[layer]
        strided = "strided" in block
        if block == "simple":
            if cin > 1:
                rows.append(shape_row("kpconv", m, kp * cin, fdim, flags="rowscale+bn+leaky", row_map=True))
            cin = fdim
        else:
            mo = NOMINAL_ROWS[layer + 1] if strided else m
            rows.append(shape_row("unary", m, cin, fdim // 2, flags="bn+leaky"))
            rows.append(shape_row("kpconv", mo, kp * (fdim // 2), fdim // 2, flags="rowscale+bn+leaky",
                                  row_map=not strided))
            if cin != 2 * fdim:
                rows.append(shape_row("pair", mo, fdim // 2, 2 * fdim, K2=cin, flags="bias+leaky"))
            else:
                rows.append(shape_row("unary", mo, fdim // 2, 2 * fdim, flags="bn+residual+leaky", residual=True))
            cin = 2 * fdim
        if strided:
            layer += 1
            fdim *= 2
    return rows


def print_table(rows, timed):
    head = "%-7s %7s %11s %5s  %-20s %3s %9s %9s %8s %-6s" % ("kind", "M", "K", "N", "epilogue", "map", "MB(min)",
                                                              "GF x3", "bound us", "by")
    if timed:
        head += " %9s %7s %9s" % ("us", "t/bound", "t-bound")
    print(head)
    for r in rows:
        k = "%d" % r["K"] if not r["K2"] else "%d|%d" % (r["K"], r["K2"])
        line = "%-7s %7d %11s %5d  %-20s %3s %9.1f %9.1f %8.1f %-6s" % (
            r["kind"], r["M"], k, r["N"], r["flags"], "yes" if r["row_map"] else "no", r["min_bytes"] / 1e6,
            r["flops_x3"] / 1e9, r["bound_us"], r["bound_by"])
        if timed:
            line += " %9.1f %7.2f %9.1f" % (r["us"], r["us"] / r["bound_us"], r["us"] - r["bound_us"])
        print(line)
    tot_b = sum(r["bound_us"] for r in rows)
    if timed:
        tot = sum(r["us"] for r in rows)
        print("sum: %.1f us measured against %.1f us of bound (%.2fx)" % (tot, tot_b, tot / tot_b))
    else:
        print("sum of bounds: %.1f us" % tot_b)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", help="directory for gemm_step_table.json")
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--dry-run", action="store_true", help="no GPU: shapes at nominal level sizes and their bounds")
    args = ap.parse_args()

    from d3feat_b200 import synth
    cfg = synth.Config(architecture=synth.ARCH_ENCODER)
    if args.dry_run:
        print_table(nominal_shapes(cfg), timed=False)
        return
    if not args.out:
        ap.error("--out is required without --dry-run")

    import torch
    assert torch.cuda.is_available(), "gemm_step_table.py needs a GPU"
    from d3feat_b200 import _lib
    from d3feat_b200 import convolution_ops as co
    from d3feat_b200.encoder import KPFCNN

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    _lib.lib()
    params = synth.make_params(cfg, seed=0)
    clouds = [synth.room_fragment(i, 30000) for i in range(8)]
    P = np.concatenate(clouds, 0)
    L = np.array([c.shape[0] for c in clouds], np.int32)
    P_dev, L_dev = torch.from_numpy(P).to(dev), torch.from_numpy(L).to(dev)
    enc = KPFCNN(cfg, params, [40] * 5, device=dev)
    bbox = np.concatenate([P.min(0), P.max(0)]).astype(np.float32)

    calls = []
    orig_kp, orig_un, orig_up = co.KPConv_ops, co.unary_convolution, co.unary_pair_convolution

    def hook_kp(q, s, idx, f, Kp, W, *a, **k):
        calls.append(("kpconv", (idx, W), k))
        return orig_kp(q, s, idx, f, Kp, W, *a, **k)

    def hook_un(x, w, **k):
        calls.append(("unary", (x, w), k))
        return orig_un(x, w, **k)

    def hook_up(x1, w1, a1, x2, w2, a2, alpha, **k):
        calls.append(("pair", (x1, w1, a1, x2, w2, a2, alpha), k))
        return orig_up(x1, w1, a1, x2, w2, a2, alpha, **k)

    co.KPConv_ops, co.unary_convolution, co.unary_pair_convolution = hook_kp, hook_un, hook_up
    try:
        enc(P_dev, L_dev, bbox=bbox, decoder=False)
    finally:
        co.KPConv_ops, co.unary_convolution, co.unary_pair_convolution = orig_kp, orig_un, orig_up
    torch.cuda.synchronize()

    flush = torch.empty((256 << 20,), dtype=torch.uint8, device=dev)     # > 50 MB L2

    def time_us(fn):
        for _ in range(5):
            fn()
        evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(args.reps)]
        for a, b in evs:
            flush.fill_(1)
            a.record()
            fn()
            b.record()
        torch.cuda.synchronize()
        return float(np.median([a.elapsed_time(b) for a, b in evs])) * 1e3

    def ep_flags(k, extra=""):
        f = extra
        if k.get("epilogue") is not None:
            f += "bn+" + ("leaky+" if k["epilogue"][2] is not None else "")
        if k.get("bias") is not None:
            f += "bias+"
        if k.get("residual") is not None:
            f += "residual+"
        return f.rstrip("+")

    rows = []
    for kind, a, k in calls:
        if kind == "kpconv":
            idx, W = a
            Kp, Cin, Cout = (int(v) for v in W.shape)
            if Cin == 1:
                continue                      # the Cin = 1 layer has its own kernel and no GEMM
            M = int(idx.shape[0])
            # the contraction alone, on a weighted-feature matrix of the real size; inside the KPConv it also scales
            # the rows and, for cell-ordered queries, scatters them through a row map
            wf = torch.randn(M, Kp * Cin, device=dev)
            w2 = W.reshape(Kp * Cin, Cout)
            r = shape_row("kpconv", M, Kp * Cin, Cout, flags=ep_flags(k, "rowscale+"),
                          row_map=k.get("query_order") is not None)
            r["us"] = time_us(lambda: orig_un(wf, w2, epilogue=k.get("epilogue"), rows=k.get("rows_q")))
            del wf
        elif kind == "unary":
            x, w = a
            r = shape_row("unary", int(x.shape[0]), int(w.shape[0]), int(w.shape[1]), flags=ep_flags(k),
                          residual=k.get("residual") is not None)
            r["us"] = time_us(lambda: orig_un(x, w, **k))
        else:
            x1, w1, a1, x2, w2, a2, alpha = a
            r = shape_row("pair", int(x1.shape[0]), int(w1.shape[0]), int(w1.shape[1]), K2=int(w2.shape[0]),
                          flags="bias+leaky")
            r["us"] = time_us(lambda: orig_up(x1, w1, a1, x2, w2, a2, alpha, **k))
        rows.append(r)

    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader",
                        "-i", str(torch.cuda.current_device())], capture_output=True, text=True).stdout.strip()
    print("card: %s" % q)
    print_table(rows, timed=True)
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "gemm_step_table.json"), "w") as fh:
        json.dump(dict(gpu=torch.cuda.get_device_name(dev), nvidia_smi=q, reps=args.reps,
                       bounds="derived from the data sheet: 3.35 TB/s HBM3, 495 TFLOP/s dense TF32",
                       total_us=sum(r["us"] for r in rows), total_bound_us=sum(r["bound_us"] for r in rows),
                       gemms=rows), fh, indent=1)


if __name__ == "__main__":
    main()
