"""GPU: what point-to-point ICP costs, as an op and inside a serving step. Writes OUT_DIR/icp_bench.json and prints it.

Op: d3f_icp_pairs on
  * room: 8 partial rigid copies (about 30 000 points each, 2 mm noise) of one synth.room_fragment scene, P = 1 and
    P = 28 (every i < j) pairs, distance 0.05, max_iterations 30;
  * lidar: a 120 000-point synth.lidar_scan (the kitti120k workload of bench.py) and a rigid copy of 90 % of it (1 cm noise) completed to 120 000 points by
    part of a second scan, distance 0.2, max_iterations 200 (the KITTI loader's refinement);
every pair starting from its true pose perturbed by 2 degrees and 3 cm, with Open3D's default relative thresholds
(1e-6). A CUDA graph of `reps` back-to-back calls is replayed after a warm-up replay and timed with CUDA events. The
host numpy restatement (oracle/icp_np.py) is timed on the same input where it is run (--oracle-all adds P = 28), and
the device result is compared with it bit for bit.

Pipeline: GraphPipeline(decoder=True, keypoints=250, match_pairs = every i < j of 8 x 30 000-point clouds,
register={}) with and without icp=dict(distance=0.05), in alternating runs, timed as scripts/keypoint_bench.py does. The
synthetic weights give uninformative descriptors, so the RANSAC poses ICP starts from are poor and most pairs stop
within a few iterations. The card's name, power limit and max SM clock are read in the same process.

    python scripts/icp_bench.py --out DIR [--rounds 5] [--steps 24] [--warmup 6] [--oracle-all]
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

FIELDS = ("pose", "fitness", "inlier_rmse", "n_correspondences", "iterations")


def rotation(rng, deg):
    axis = rng.normal(size=3)
    axis /= np.linalg.norm(axis)
    th = np.deg2rad(deg)
    K = np.array([[0, -axis[2], axis[1]], [axis[2], 0, -axis[0]], [-axis[1], axis[0], 0]])
    return np.eye(3) + np.sin(th) * K + (1 - np.cos(th)) * K @ K


def rigid(R, t):
    T = np.eye(4)
    T[:3, :3], T[:3, 3] = R, t
    return T


def copies(rng, base, n_copies, n, noise, deg, shift):
    """n_copies partial rigid copies of `base` (the rows below a random plane, cut to n) with noise: (clouds, poses)."""
    clouds, poses = [], []
    for _ in range(n_copies):
        d = rng.normal(size=3)
        proj = base @ d
        part = base[np.argsort(proj, kind="stable")[:n]]
        T = rigid(rotation(rng, deg), rng.uniform(-shift, shift, 3))
        clouds.append((part @ T[:3, :3].T + T[:3, 3] + rng.normal(scale=noise, size=part.shape)).astype(np.float32))
        poses.append(T)
    return clouds, poses


def perturbed(rng, T, deg=2.0, shift=0.03):
    d = rng.normal(size=3)
    return rigid(rotation(rng, deg), shift * d / np.linalg.norm(d)) @ T


def make_case(rng, kind, P):
    from d3feat_b200 import synth
    if kind == "room":
        clouds, poses = copies(rng, synth.room_fragment(0, 36000), 8, 30000, 0.002, 10.0, 0.2)
        pairs = [(i, j) for i in range(8) for j in range(i + 1, 8)][:P]
        tau, I = 0.05, 30
    else:
        # the scan, and a moved copy of 90 % of it with 12 000 rows of a second scan in place of the rest
        base = synth.lidar_scan(1, 120000, dl=0.04)
        (part,), (T,) = copies(rng, base, 1, 108000, 0.01, 3.0, 1.0)
        clouds, poses = [base, np.concatenate([part, synth.lidar_scan(2, 12000, dl=0.04)])], [np.eye(4), T]
        pairs = [(0, 1)]
        tau, I = 0.2, 200
    init = np.stack([perturbed(rng, poses[j] @ np.linalg.inv(poses[i])) for i, j in pairs])
    pts = np.concatenate(clouds)
    lo, hi = pts.min(0), pts.max(0)
    bbox = np.concatenate([lo - 0.05 * (hi - lo), hi + 0.05 * (hi - lo)]).astype(np.float32)
    return dict(points=pts, lengths=np.array([len(c) for c in clouds], np.int32), pairs=np.array(pairs, np.int32),
                init=init, bbox=bbox, distance=tau, max_iterations=I)


def time_op(case, dev, reps, iters):
    """Device µs per d3f_icp_pairs call (graph of `reps` calls, median over `iters` replays), the graph nodes of one
    call and the outputs."""
    from d3feat_b200 import _lib
    lib = _lib.lib()
    tp, tl, tq, ti = (torch.from_numpy(case[k]).to(dev) for k in ("points", "lengths", "pairs", "init"))
    N, B, P = tp.shape[0], tl.shape[0], tq.shape[0]
    bb = case["bbox"]
    bbp = bb.ctypes.data_as(_lib.C.c_void_p)
    pose = torch.empty((P, 4, 4), dtype=torch.float64, device=dev)
    fit, rmse = (torch.empty((P,), dtype=torch.float64, device=dev) for _ in range(2))
    nc, it = (torch.empty((P,), dtype=torch.int32, device=dev) for _ in range(2))
    ws = _lib.workspace(lib.d3f_icp_pairs_workspace_bytes(N, B, P, case["distance"], bbp), dev)

    def call():
        _lib.check(lib.d3f_icp_pairs(_lib.ptr(tp), _lib.ptr(tl), B, N, None, bbp, _lib.ptr(tq), P, _lib.ptr(ti),
                                     case["distance"], case["max_iterations"], 1e-6, 1e-6, _lib.ptr(pose),
                                     _lib.ptr(fit), _lib.ptr(rmse), _lib.ptr(nc), _lib.ptr(it), _lib.ptr(ws),
                                     ws.numel(), _lib.stream()),
                   "d3f_icp_pairs")

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        call()
    torch.cuda.current_stream().wait_stream(s)
    n0 = _lib.launch_count()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(reps):
            call()
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
    got = dict(pose=pose.cpu().numpy(), fitness=fit.cpu().numpy(), inlier_rmse=rmse.cpu().numpy(),
               n_correspondences=nc.cpu().numpy(), iterations=it.cpu().numpy())
    return float(np.median(per_call)), kernels, got


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="directory for icp_bench.json")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=24)
    ap.add_argument("--warmup", type=int, default=6)
    ap.add_argument("--oracle-all", action="store_true", help="also time the host restatement on P = 28")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "icp_bench.py needs a GPU"
    assert args.steps >= 20, "--steps: the median of at least 20 steps"

    from d3feat_b200 import synth, _lib
    from d3feat_b200.encoder import KPFCNN, GraphPipeline
    from oracle import icp_np

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    _lib.lib()
    card = card_info()
    print(json.dumps(card), flush=True)
    op = []
    for kind, P, reps in (("room", 1, 5), ("room", 28, 3), ("lidar", 1, 2)):
        case = make_case(np.random.default_rng(P + len(kind)), kind, P)
        us, kernels, got = time_op(case, dev, reps=reps, iters=5)
        row = dict(case=kind, P=P, points=int(case["points"].shape[0]), clouds=int(case["lengths"].shape[0]),
                   distance=case["distance"], max_iterations=case["max_iterations"], device_us_per_call=us,
                   kernels_per_call=kernels, iterations=got["iterations"].tolist(),
                   fitness=[round(float(x), 4) for x in got["fitness"]],
                   inlier_rmse=[float("%.4g" % x) for x in got["inlier_rmse"]])
        if P == 1 or args.oracle_all:
            t0 = time.perf_counter()
            want = icp_np.icp(case["points"], case["lengths"], case["pairs"], case["init"], distance=case["distance"],
                              max_iterations=case["max_iterations"])
            row["host_numpy_restatement_ms"] = (time.perf_counter() - t0) * 1e3
            row["equal_to_restatement"] = all(
                np.array_equal(np.asarray(got[f]).view(np.int64) if got[f].dtype == np.float64 else got[f],
                               want[f].view(np.int64) if want[f].dtype == np.float64 else want[f]) for f in FIELDS)
        op.append(row)
        print(json.dumps(row), flush=True)

    cfg = synth.Config(architecture=synth.ARCH_3DMATCH)
    clouds = [synth.room_fragment(i, 30000) for i in range(8)]
    P0 = torch.from_numpy(np.concatenate(clouds, 0)).to(dev)
    L0 = torch.from_numpy(np.array([c.shape[0] for c in clouds], np.int32)).to(dev)
    enc = KPFCNN(cfg, synth.make_params(cfg, 0), [40, 40, 40, 40, 40], device=dev)
    pairs = [(i, j) for i in range(8) for j in range(i + 1, 8)]
    kw = dict(decoder=True, keypoints=250, match_pairs=pairs, register={})
    pipes = {"register": GraphPipeline.for_batch(enc, P0, L0, **kw),
             "register+icp": GraphPipeline.for_batch(enc, P0, L0, icp=dict(distance=0.05), **kw)}
    runs = {name: [] for name in pipes}
    for r in range(args.rounds):
        names = list(pipes) if r % 2 == 0 else list(pipes)[::-1]       # alternate which variant goes first
        for name in names:
            runs[name].append(run(pipes[name], P0, L0, args.steps, args.warmup))
    med = {name: float(np.median(v)) for name, v in runs.items()}
    res = dict(card=card, op=op,
               pipeline=dict(workload="8 x 30000-point synthetic fragments, ARCH_3DMATCH (encoder + decoder), limits 40",
                             k=250, pairs=len(pairs), steps=args.steps, warmup=args.warmup, rounds=args.rounds,
                             kernels_per_step={name: int(p.kernels_per_step) for name, p in pipes.items()},
                             runs_ms=runs, median_ms=med,
                             added_ms_per_step=med["register+icp"] - med["register"]))
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "icp_bench.json"), "w") as fh:
        json.dump(res, fh, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
