"""GPU: per-kernel table of a bench step. Runs bench.py's default workload (8 x 30k points, GraphPipeline with two
encoder streams, the same seeds), times steps with CUDA events, then profiles replayed steps with torch.profiler
(CUDA activity) and prints one table: kernel, launches per step, total us per step, share of the serialised device
time, grouped into families. Writes the table as JSON to OUT_DIR/step_kernels.json.

    python scripts/step_kernels.py --out DIR [--steps 10]
"""
import argparse
import collections
import json
import os
import re
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np
import torch

FAMILIES = [
    ("tc_gemm", r"tc_gemm_kernel"),
    ("splitk_reduce", r"splitk_reduce_kernel"),
    ("stage 1", r"kpconv_stage1|prep_supports"),
    ("cin1", r"kpconv_cin1"),
    ("fused kpconv", r"kpconv_fused"),
    ("radius query", r"radius_query|cell_count|cell_scatter|cell_order"),
    ("grid/sort", r"radix_|scan_|batch_start|bbox_|cell_key|segment_head|cell_reduce|cell_feature|subsample_status|set_count"),
    ("pools", r"pool|colmin|l2_normalize|cloud_max|detection_score|affine_leaky"),
]


def family(name):
    for fam, pat in FAMILIES:
        if re.search(pat, name):
            return fam
    return "other"


def short(name):
    # "void d3f::tc_gemm_kernel<128>(float const*, ...)" -> "tc_gemm_kernel<128>"
    n = re.sub(r"^void\s+", "", name)
    n = re.sub(r"\(.*$", "", n)
    return n.replace("d3f::", "")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--out", required=True, help="directory for step_kernels.json")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "step_kernels.py needs a GPU"

    from d3feat_b200 import synth, _lib
    from d3feat_b200.encoder import KPFCNN, GraphPipeline

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    _lib.lib()
    cfg = synth.Config(architecture=synth.ARCH_ENCODER)
    params = synth.make_params(cfg, seed=0)
    limits = [40, 40, 40, 40, 40]
    clouds = [synth.room_fragment(i, 30000) for i in range(8)]
    P = np.concatenate(clouds, 0)
    L = np.array([c.shape[0] for c in clouds], np.int32)
    P_dev, L_dev = torch.from_numpy(P).to(dev), torch.from_numpy(L).to(dev)
    enc = KPFCNN(cfg, params, limits, device=dev)
    pipe = GraphPipeline.for_batch(enc, P_dev, L_dev, decoder=False, encoder_streams=2)
    pipe.prime(P_dev, L_dev)
    for _ in range(10):
        pipe.step(P_dev, L_dev)
    pipe.drain()

    # step time without the profiler: completion interval of consecutive steps, averaged over the encoder streams
    n = max(args.steps, 4)
    marks = [torch.cuda.Event(enable_timing=True) for _ in range(n + 1)]
    marks[0].record(pipe.s_enc)
    for i in range(n):
        pipe.step(P_dev, L_dev)
        marks[i + 1].record(pipe.s_enc)
    pipe.drain()
    torch.cuda.synchronize()
    w = len(pipe.s_encs)
    step_ms = float(np.median([marks[i].elapsed_time(marks[i + w]) / w for i in range(n - w + 1)]))

    from torch.profiler import profile, ProfilerActivity
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.steps):
            pipe.step(P_dev, L_dev)
        pipe.drain()
        torch.cuda.synchronize()
    pipe.check()

    per = collections.defaultdict(lambda: [0, 0.0])
    for ev in prof.events():
        if ev.device_type != torch.autograd.DeviceType.CUDA:
            continue
        nm = ev.name
        if nm.startswith(("Memcpy", "Memset", "cudaMemcpy", "cudaMemset")) or "fill" in nm.lower():
            key = "copies/fills"
        else:
            key = short(nm)
        per[key][0] += 1
        per[key][1] += ev.time_range.elapsed_us()
    rows = []
    total = sum(v[1] for v in per.values()) / args.steps
    for k, (cnt, us) in per.items():
        us /= args.steps
        rows.append(dict(kernel=k, family=family(k) if k != "copies/fills" else "copies/fills",
                         launches_per_step=cnt / args.steps, us_per_step=us, share=us / total if total else 0.0))
    rows.sort(key=lambda r: -r["us_per_step"])
    fams = collections.OrderedDict()
    for r in rows:
        f = fams.setdefault(r["family"], dict(family=r["family"], launches_per_step=0.0, us_per_step=0.0))
        f["launches_per_step"] += r["launches_per_step"]
        f["us_per_step"] += r["us_per_step"]
    for f in fams.values():
        f["share"] = f["us_per_step"] / total if total else 0.0
    fam_rows = sorted(fams.values(), key=lambda f: -f["us_per_step"])

    print("step time (events, no profiler): %.3f ms; serialised device time: %.3f ms (%.2fx the step)" % (
        step_ms, total / 1e3, total / 1e3 / step_ms))
    print("%-44s %9s %10s %7s" % ("family", "launches", "us/step", "share"))
    for f in fam_rows:
        print("%-44s %9.1f %10.1f %6.1f%%" % (f["family"], f["launches_per_step"], f["us_per_step"], 100 * f["share"]))
    print()
    print("%-44s %-14s %9s %10s %7s" % ("kernel", "family", "launches", "us/step", "share"))
    for r in rows:
        print("%-44s %-14s %9.1f %10.1f %6.1f%%" % (r["kernel"][:44], r["family"], r["launches_per_step"],
                                                    r["us_per_step"], 100 * r["share"]))
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "step_kernels.json"), "w") as fh:
        json.dump(dict(step_ms=step_ms, serialised_ms=total / 1e3, profiled_steps=args.steps,
                       gpu=torch.cuda.get_device_name(dev), families=fam_rows, kernels=rows), fh, indent=1)


if __name__ == "__main__":
    main()
