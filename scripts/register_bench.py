"""GPU: what RANSAC registration costs, as an op and inside a serving step. Writes OUT_DIR/register_bench.json and
prints it.

Op: d3f_register_pairs on P cloud pairs of k = 250 keypoints for P in {1, 28} and (ransac_n, max_iterations,
max_validation) in {(3, 50000, 1000), (4, 50000, 1000), (4, 4000000, 500)}: the 3DMatch evaluation's, the KITTI
tester's and the demo's settings. Every source slot has one correspondence, (i, nn(i)), of which 30 % are true
(a rigid copy of the source, 5 mm noise) and the rest random: registration stops once max_validation hypotheses are
validated. A CUDA graph of 10 back-to-back calls is replayed 10 times after a warm-up replay and timed with CUDA
events. The host numpy restatement (oracle/register_np.py, vectorised over hypotheses) is timed on the same input.

Pipeline: GraphPipeline(decoder=True, keypoints=250, match_pairs = every i < j of 8 x 30 000-point clouds) with and
without register={} (the 3DMatch defaults), in alternating runs, timed as scripts/keypoint_bench.py does. The
synthetic weights give uninformative descriptors, so the matches are mostly outliers. The card's name, power limit
and max SM clock are read in the same process.

    python scripts/register_bench.py --out DIR [--rounds 5] [--steps 24] [--warmup 6]
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

CASES = [(3, 50000, 1000), (4, 50000, 1000), (4, 4000000, 500)]


def make_input(k, P, rng):
    """points [8,k,3] (rigid copies of one cloud, 5 mm noise), count [8], pairs [P,2], corr [P,k,2], n_corr [P]"""
    B = 8
    base = rng.uniform(-1, 1, (k, 3))
    pts = []
    for _ in range(B):
        q = rng.normal(size=4)
        w, x, y, z = q / np.linalg.norm(q)
        R = np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                      [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                      [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])
        pts.append(base @ R.T + rng.uniform(-1, 1, 3) + rng.normal(scale=0.005, size=(k, 3)))
    pts = np.stack(pts).astype(np.float32)
    pairs = np.array([(i, j) for i in range(B) for j in range(i + 1, B)][:P], np.int32)
    nn = np.arange(k)[None].repeat(P, 0)
    out = rng.random((P, k)) >= 0.3
    nn[out] = rng.integers(0, k, int(out.sum()))
    corr = np.stack([np.arange(k)[None].repeat(P, 0), nn], 2).astype(np.int32)
    return pts, np.full(B, k, np.int32), pairs, corr, np.full(P, k, np.int32)


def time_op(inp, n, T, V, dev, reps, iters):
    """Device µs per d3f_register_pairs call (graph of `reps` calls, median over `iters` replays) and the outputs."""
    from d3feat_b200 import _lib
    lib = _lib.lib()
    pts, count, pairs, corr, n_corr = inp
    B, k, _ = pts.shape
    P, L, _ = corr.shape
    tp, tc, tq, tr, tn = (torch.from_numpy(a).to(dev) for a in (pts, count, pairs, corr, n_corr))
    pose = torch.empty((P, 4, 4), dtype=torch.float64, device=dev)
    ints = [torch.empty((P,), dtype=torch.int32, device=dev) for _ in range(3)]
    ws = _lib.workspace(lib.d3f_register_pairs_workspace_bytes(L, P, T, V), dev)

    def call():
        _lib.check(lib.d3f_register_pairs(_lib.ptr(tp), _lib.ptr(tc), B, k, _lib.ptr(tr), _lib.ptr(tn), L, _lib.ptr(tq),
                                          P, n, T, V, 0.05, 0.9, 0, _lib.ptr(pose), *[_lib.ptr(x) for x in ints],
                                          _lib.ptr(ws), ws.numel(), _lib.stream()),
                   "d3f_register_pairs")

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
    got = dict(pose=pose.cpu().numpy(), n_inliers=ints[0].cpu().numpy(), hypothesis=ints[1].cpu().numpy(),
               n_validated=ints[2].cpu().numpy())
    return float(np.median(per_call)), got


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="directory for register_bench.json")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=24)
    ap.add_argument("--warmup", type=int, default=6)
    ap.add_argument("--k", type=int, default=250, help="keypoints per cloud")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "register_bench.py needs a GPU"
    assert args.steps >= 20, "--steps: the median of at least 20 steps"

    from d3feat_b200 import synth, _lib
    from d3feat_b200.encoder import KPFCNN, GraphPipeline
    from oracle import register_np

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    _lib.lib()
    card = card_info()
    op = []
    for P in (1, 28):
        inp = make_input(args.k, P, np.random.default_rng(P))
        for n, T, V in CASES:
            us, got = time_op(inp, n, T, V, dev, reps=10, iters=10)
            t0 = time.perf_counter()
            want = register_np.register(*inp[:1], inp[1], inp[3], inp[4], inp[2], distance=0.05, ransac_n=n,
                                        edge_ratio=0.9, max_iterations=T, max_validation=V, seed=0)
            host_ms = (time.perf_counter() - t0) * 1e3
            same = all(np.array_equal(np.asarray(got[f]).view(np.int64) if f == "pose" else got[f],
                                      want[f].view(np.int64) if f == "pose" else want[f]) for f in got)
            op.append(dict(k=args.k, P=P, ransac_n=n, max_iterations=T, max_validation=V, device_us_per_call=us,
                           host_numpy_restatement_ms=host_ms, equal_to_restatement=bool(same),
                           n_validated=got["n_validated"].tolist()[:4], n_inliers=got["n_inliers"].tolist()[:4],
                           max_hypothesis=int(got["hypothesis"].max())))
            print(json.dumps(op[-1]), flush=True)

    cfg = synth.Config(architecture=synth.ARCH_3DMATCH)
    clouds = [synth.room_fragment(i, 30000) for i in range(8)]
    P0 = torch.from_numpy(np.concatenate(clouds, 0)).to(dev)
    L0 = torch.from_numpy(np.array([c.shape[0] for c in clouds], np.int32)).to(dev)
    enc = KPFCNN(cfg, synth.make_params(cfg, 0), [40, 40, 40, 40, 40], device=dev)
    pairs = [(i, j) for i in range(8) for j in range(i + 1, 8)]
    pipes = {"match": GraphPipeline.for_batch(enc, P0, L0, decoder=True, keypoints=args.k, match_pairs=pairs),
             "match+register": GraphPipeline.for_batch(enc, P0, L0, decoder=True, keypoints=args.k,
                                                       match_pairs=pairs, register={})}
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
                             added_ms_per_step=med["match+register"] - med["match"]))
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "register_bench.json"), "w") as fh:
        json.dump(res, fh, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
