"""Voxel down-sampling on the GPU: the op alone and inside the serving step.

    python scripts/voxel_bench.py --out DIR

1. The op alone (static form, d3f_voxel_down_sample): a CUDA graph of `--calls` back-to-back calls, timed with CUDA
   events, on 8 raw synthetic rooms at 0.03 m (about 300 000 raw points each, the size of a 3DMatch test fragment
   before voxel_down_sample) and 2 raw synthetic 64-beam scans at 0.3 m (2000 azimuth steps, about 120 000 returns
   each, a KITTI velodyne scan). Reported with the bytes the algorithm must move and the HBM bound at 3.35 TB/s, and
   the host time of the C restatement (oracle/voxel_oracle.c, one thread) on the same input.
2. The serving step: GraphPipeline(voxel_size=0.03) fed the raw rooms against the same pipeline fed the voxelised
   rooms, in alternating runs. How much of the voxel stage hides under the previous batch's encoder is not measured
   separately; the difference of the two step times is what the run shows.

Writes DIR/voxel_bench.json and prints it with the card's name and power limit."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

HBM = 3.35e12


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def algorithm_bytes(N, M, B, key_bits):
    """Bytes the sort-based algorithm moves at minimum: two reads of the raw rows (bounds, keys), the (key, row) pairs
    written once, read and written by every 8-bit radix pass (count reads keys, scatter reads and writes pairs), the
    head flags and their scan, the gather of every row by its voxel, the output."""
    passes = (key_bits + 7) // 8
    raw = 2 * 12 * N
    pairs = 12 * N
    sort = passes * (8 * N + 24 * N)
    heads_scan = 8 * N + 4 * N + 3 * 4 * N
    gather = 12 * N + 12 * N + 4 * N
    out = 12 * M + 4 * B
    return dict(raw=raw, pairs=pairs, sort=sort, heads_scan=heads_scan, gather=gather, output=out,
                total=raw + pairs + sort + heads_scan + gather + out, passes=passes)


def time_op(dev, pts, lens, v, calls):
    import torch
    from d3feat_b200 import voxel
    from oracle.voxel_native import port_voxel_down_sample
    p, l = torch.from_numpy(pts).to(dev), torch.from_numpy(lens).to(dev)
    want = port_voxel_down_sample(pts, lens, v)
    t0 = time.perf_counter()
    port_voxel_down_sample(pts, lens, v)
    host_ms = (time.perf_counter() - t0) * 1e3
    bbox = np.concatenate([pts.min(0), pts.max(0)])
    st = voxel.VoxelStage(len(pts), len(lens), v, bbox, dev)
    st.points.copy_(p)
    st.lengths.copy_(l)
    st.n.fill_(len(pts))
    out = torch.empty((len(pts), 3), dtype=torch.float32, device=dev)
    ol = torch.empty((len(lens),), dtype=torch.int32, device=dev)
    on = torch.empty((1,), dtype=torch.int32, device=dev)
    status = torch.zeros((1,), dtype=torch.int32, device=dev)
    s = torch.cuda.Stream(device=dev)
    s.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.stream(s):
        st.run(out, ol, on, status)
    torch.cuda.synchronize(dev)
    M = int(on.item())
    assert M == len(want[0]) and int(status.item()) == 0
    assert np.array_equal(out[:M].cpu().numpy().view(np.uint32), want[0].view(np.uint32)), "differs from the C port"
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        for _ in range(calls):
            st.run(out, ol, on, status)
    for _ in range(3):
        g.replay()
    torch.cuda.synchronize(dev)
    times = []
    for _ in range(5):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        g.replay()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b) * 1e3 / calls)
    ext = (bbox[3:] - bbox[:3]).astype(np.float64)
    bits = [max(1, int(np.ceil(np.log2(np.floor(e / v) + 3.0)))) for e in ext]
    key_bits = sum(bits) + int(np.ceil(np.log2(len(lens) + 1)))
    by = algorithm_bytes(len(pts), M, len(lens), key_bits)
    us = float(np.median(times))
    return dict(raw_points=int(len(pts)), clouds=int(len(lens)), voxel_size=v, voxels=M, key_bits=key_bits,
                us_per_call=us, us_spread=[float(min(times)), float(max(times))], bytes=by,
                hbm_bound_us=by["total"] / HBM * 1e6, share_of_hbm_bound=by["total"] / HBM * 1e6 / us,
                c_port_host_ms=host_ms)


def time_serving(dev, rooms, steps, rounds):
    import torch
    from d3feat_b200 import synth
    from d3feat_b200.encoder import GraphPipeline, KPFCNN
    from oracle.voxel_native import port_voxel_down_sample
    cfg = synth.Config(architecture=synth.ARCH_3DMATCH)
    enc = KPFCNN(cfg, synth.make_params(cfg, 0), [35, 33, 34, 36, 30], device=dev)
    raws = []
    for i in range(2):   # two batches of the same 8 rooms in different row orders, alternated
        rng = np.random.default_rng(i)
        clouds = [r[rng.permutation(len(r))] for r in rooms]
        raws.append((np.concatenate(clouds), np.array([len(c) for c in clouds], np.int32)))
    voxd = [port_voxel_down_sample(p, l, 0.03) for p, l in raws]
    dev_raw = [(torch.from_numpy(p).to(dev), torch.from_numpy(l).to(dev)) for p, l in raws]
    dev_vox = [(torch.from_numpy(p).to(dev), torch.from_numpy(l).to(dev)) for p, l in voxd]
    raw_pipe = GraphPipeline.for_batch(enc, *dev_raw[0], voxel_size=0.03, decoder=True, keypoints=250)
    vox_pipe = GraphPipeline(enc, raw_pipe.caps, len(rooms), raw_pipe.bbox, decoder=True, keypoints=250)

    def run(pipe, feed):
        pipe.prime(*feed[0])
        for i in range(steps):
            pipe.step(*feed[(i + 1) % 2])
        pipe.step()
        torch.cuda.synchronize(dev)

    for pipe, feed in ((raw_pipe, dev_raw), (vox_pipe, dev_vox)):
        run(pipe, feed)
    ms = {"raw scans (voxel_size=0.03)": [], "voxelised clouds": []}
    for _ in range(rounds):
        for name, pipe, feed in (("raw scans (voxel_size=0.03)", raw_pipe, dev_raw),
                                 ("voxelised clouds", vox_pipe, dev_vox)):
            t0 = time.perf_counter()
            run(pipe, feed)
            ms[name].append((time.perf_counter() - t0) * 1e3 / (steps + 1))
    raw_pipe.check()
    vox_pipe.check()
    return dict(steps_per_run=steps + 1, rounds=rounds, kernels_per_step={"raw": int(raw_pipe.kernels_per_step),
                                                                         "voxelised": int(vox_pipe.kernels_per_step)},
                level0_points=[int(x) for x in voxd[0][1]], ms_per_step={k: float(np.median(v)) for k, v in ms.items()},
                ms_per_step_runs=ms)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--steps", type=int, default=40)
    ap.add_argument("--rounds", type=int, default=4)
    a = ap.parse_args()
    import torch
    from d3feat_b200 import synth
    if not torch.cuda.is_available():
        sys.exit("voxel_bench: no CUDA device (nothing here is measured on the CPU)")
    dev = torch.device("cuda", 0)
    rooms = [synth.raw_room_scan(s, 300000) for s in range(8)]
    scans = [synth.raw_lidar_scan(s, 2000) for s in range(2)]
    res = dict(card=card())
    res["rooms_8x_0.03"] = time_op(dev, np.concatenate(rooms), np.array([len(r) for r in rooms], np.int32), 0.03,
                                   a.calls)
    res["scans_2x_0.3"] = time_op(dev, np.concatenate(scans), np.array([len(s) for s in scans], np.int32), 0.3,
                                  a.calls)
    res["serving_step_8_rooms"] = time_serving(dev, rooms, a.steps, a.rounds)
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, "voxel_bench.json"), "w") as fh:
        json.dump(res, fh, indent=1)
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
