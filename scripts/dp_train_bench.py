"""The data-parallel training step and its new kernels on the GPU: the 3DMatch architecture and training configuration,
each rank on its own pair of 30 000-point synth.room_fragment scenes (the second a rigidly moved copy of the first),
256 keypoint correspondences.

    python scripts/dp_train_bench.py --out DIR [--steps 10] [--warmup 3]

1. P, the number of trainable parameters of the 3DMatch architecture.
2. The step (forward, loss, backward, reduce_gradients, MomentumClip.step, reduce_moving_statistics) at world size 1,
   timed with CUDA events, median over --steps after --warmup; the reduction and update part is reported on its own.
   With more than one GPU, the same at world size N (one process per GPU, NCCL), rank 0's median.
3. The device time of d3f_rank_mean at R = 1, 2, 8 over P and of the two update kernels over the whole store
   (torch.profiler, 20 calls each), against their HBM bound at 3.35 TB/s: rank_mean reads R*P and writes P floats; the
   update reads g twice (partials, then the update), accum and var once, writes accum and var, and writes and reads
   one fp64 partial per 2048-element block.

Writes DIR/dp_train_bench.json with the card's name and power limit.
"""
import argparse
import collections
import datetime
import json
import os
import socket
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

HBM = 3.35e12
N_POINTS = 30000


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def replica(dev, seed):
    """(config, store, encoder inputs, anc, pos, params, optimiser) of one rank: its own pair of scenes."""
    import torch
    from d3feat_b200 import pyramid, synth, training as T
    from d3feat_b200.encoder import KPFCNN
    cfg = synth.Config(**T.TRAINING_3DMATCH)
    a = synth.room_fragment(seed, N_POINTS)
    th = 0.3
    R = np.array([[np.cos(th), -np.sin(th), 0], [np.sin(th), np.cos(th), 0], [0, 0, 1]])
    b = (a @ R.T + np.array([0.5, -0.2, 0.1])).astype(np.float32)
    limits = pyramid.calibrate_neighbors(cfg, [synth.room_fragment(0, N_POINTS)], device=dev)
    enc = KPFCNN(cfg, synth.make_params(cfg, seed=0), limits, device=dev)
    inputs = enc.build_inputs(np.concatenate([a, b]), np.array([N_POINTS, N_POINTS], np.int32))
    anc = torch.as_tensor(np.random.default_rng(seed).choice(N_POINTS, cfg.keypts_num).astype(np.int32)).to(dev)
    params = T.trainable(enc.store)
    opt = T.MomentumClip(params, cfg.learning_rate, cfg.momentum, cfg.grad_clip_norm)
    return cfg, enc.store, inputs, anc, anc + N_POINTS, params, opt


def dp_step(rep, events=None):
    from d3feat_b200 import distributed as D, training as T
    from d3feat_b200.variables import use_params
    cfg, store, inputs, anc, pos, params, opt = rep
    ev = events or [None] * 3
    rec = lambda i: ev[i] is not None and ev[i].record()
    rec(0)
    opt.zero_grad()
    with use_params(store):
        desc, scores = T.forward(inputs, cfg)
        out = T.d3feat_loss(desc, scores, anc, pos, inputs["points"][0], cfg)
    out[0].backward()
    rec(1)
    D.reduce_gradients(params)
    opt.step()
    D.reduce_moving_statistics(store)
    D.gather_step_stats(out)
    rec(2)


def time_steps(rep, steps, warmup):
    import torch
    for _ in range(warmup):
        dp_step(rep)
    torch.cuda.synchronize()
    t = []
    for _ in range(steps):
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
        dp_step(rep, ev)
        torch.cuda.synchronize()
        t.append([ev[0].elapsed_time(ev[2]), ev[1].elapsed_time(ev[2])])
    med = np.median(np.array(t), axis=0)
    return dict(step_ms=float(med[0]), reduce_and_update_ms=float(med[1]))


def _rank_worker(rank, world, port, steps, warmup, out):
    import torch
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, timeout=datetime.timedelta(seconds=600))
    try:
        res = time_steps(replica(torch.device("cuda", rank), rank), steps, warmup)
        if rank == 0:
            with open(out, "w") as fh:
                json.dump(res, fh)
    finally:
        dist.destroy_process_group()


def time_world(world, steps, warmup, out_dir):
    import torch.multiprocessing as mp
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    out = os.path.join(out_dir, "dp_world%d.json" % world)
    mp.spawn(_rank_worker, args=(world, port, steps, warmup, out), nprocs=world, join=True)
    with open(out) as fh:
        return json.load(fh)


def kernel_times(dev, params):
    """Device ms per call of rank_mean at R = 1, 2, 8 and of the two update kernels, with their HBM bounds."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    from d3feat_b200 import distributed as D, training as T
    P = sum(p.numel() for p in params)
    nblk = sum(-(-p.numel() // 2048) for p in params)
    g = [torch.randn_like(p) * 0.1 for p in params]
    var = [p.detach().clone() for p in params]
    acc = [torch.zeros_like(p) for p in params]
    rows = []
    reps = 20
    cases = [("rank_mean R=%d" % R, "rank_mean_kernel", 4 * (R * P + P), torch.randn(R, P, device=dev))
             for R in (1, 2, 8)]
    for name, kern, nbytes, x in cases:
        out = torch.empty(P, device=dev)
        D.rank_mean(x, out=out)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(reps):
                D.rank_mean(x, out=out)
            torch.cuda.synchronize()
        rows.append((name, {kern: nbytes}, prof))
        del x
    T.momentum_clip_update(var, acc, g, 1e-3, 0.98, 100.0)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            T.momentum_clip_update(var, acc, g, 1e-3, 0.98, 100.0)
        torch.cuda.synchronize()
    rows.append(("momentum_clip_update", {"momentum_l2_partial_kernel": 4 * P + 8 * nblk,
                                          "momentum_update_kernel": 4 * 5 * P + 8 * nblk}, prof))
    res = []
    for name, need, prof in rows:
        kt = collections.defaultdict(float)
        for e in prof.events():
            if e.device_type == torch.autograd.DeviceType.CUDA:
                kt[e.name] += e.device_time / 1e3 / reps
        for k, b in need.items():
            t = sum(v for n, v in kt.items() if k in n)
            res.append(dict(call=name, kernel=k, ms=t, bytes=b, hbm_bound_ms=b / HBM * 1e3,
                            share_of_hbm_bound=(b / HBM * 1e3) / t if t > 0 else None))
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("dp_train_bench.py needs a GPU")
    os.makedirs(args.out, exist_ok=True)
    dev = torch.device("cuda", 0)
    rep = replica(dev, 0)
    params = rep[5]
    P = sum(p.numel() for p in params)
    res = dict(card=card(), workload="3DMatch config, 2 x %d-point room_fragment pair per rank, %d correspondences" % (
        N_POINTS, rep[0].keypts_num), trainable_tensors=len(params), P=P)
    res["world"] = {"1": time_steps(rep, args.steps, args.warmup)}
    n_gpu = torch.cuda.device_count()
    if n_gpu > 1:
        res["world"][str(n_gpu)] = time_world(n_gpu, args.steps, args.warmup, args.out)
    res["kernels"] = kernel_times(dev, params)
    with open(os.path.join(args.out, "dp_train_bench.json"), "w") as fh:
        json.dump(res, fh, indent=1)
    print(res["card"], "P = %d in %d tensors" % (P, len(params)))
    for w, r in res["world"].items():
        print("world %s: step %.3f ms, of which reduce + update %.3f ms" % (w, r["step_ms"], r["reduce_and_update_ms"]))
    for r in res["kernels"]:
        print("%-22s %-28s %8.4f ms  bound %8.4f ms  share %s" % (
            r["call"], r["kernel"], r["ms"], r["hbm_bound_ms"],
            "%.2f" % r["share_of_hbm_bound"] if r["share_of_hbm_bound"] else "-"))


if __name__ == "__main__":
    main()
