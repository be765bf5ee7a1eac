"""What the training loop (trainer.Trainer) costs on top of the bare step: one short epoch of Trainer.train() against a
plain loop of the same steps on the same pairs, with the train_step_bench.py setup (3DMatch architecture and training
configuration, 30 000-point synth.room_fragment scenes). Six rooms, each as two fragments (the second the same points
in another order with 1 mm of noise), give twelve anchors, so epoch_steps = 10 runs 11 steps; validation_size = 2,
snapshot_gap = 1.

    python scripts/trainer_bench.py --out DIR [--reps 2]

Each repetition runs the bare loop, then the trainer, each on a fresh store, timed by the host clock around work that
ends in a device synchronise. The trainer's epoch end is split into the snapshot (snap-1, its side file and the
kernel-point files), the validation, and the rest (the one read of the statistics, the means, training.txt and
parameters.txt). Writes DIR/trainer_bench.json with the card's name and power limit.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

N = 30000
ROOMS = 6
EPOCH_STEPS = 10


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def setup(dev):
    import torch
    from d3feat_b200 import pyramid, synth, trainer, training as T
    cfg = synth.Config(**dict(T.TRAINING_3DMATCH, epoch_steps=EPOCH_STEPS, max_epoch=1, validation_size=2,
                              snapshot_gap=1))
    rng = np.random.default_rng(0)
    parts = []
    for r in range(ROOMS):
        a = synth.room_fragment(r, N)
        b = (a[rng.permutation(N)] + rng.uniform(-1e-3, 1e-3, a.shape)).astype(np.float32)
        parts += [a, b]
    limits = pyramid.calibrate_neighbors(cfg, [parts[0]], device=dev)
    pts = torch.from_numpy(np.concatenate(parts)).to(dev)
    lens = np.full(2 * ROOMS, N, np.int32)
    anc_to_pos = {k: [k ^ 1] for k in range(2 * ROOMS)}
    train = trainer.ThreeDMatchSchedule(pts, lens, anc_to_pos, seed=1)
    val = trainer.ThreeDMatchSchedule(pts, lens, anc_to_pos, seed=2)
    return cfg, limits, train, val


def fresh(cfg, limits, train, val, dev, saving_path):
    from d3feat_b200 import synth, trainer
    from d3feat_b200.variables import ParamStore
    c = type(cfg)(**vars(cfg))
    store = ParamStore(synth.make_params(c, seed=0), dev)
    return trainer.Trainer(c, store, limits, train, lambda e, i: val(e, i), saving_path=saving_path)


def bare(tr, steps):
    """The same steps without the loop: source, seed and Trainer.train_step only."""
    import torch
    torch.cuda.synchronize()
    t = time.perf_counter()
    for i in range(steps):
        tr.train_step(tr.train_pairs(0, i, 0, 1), tr.step_seed(0, i))
    torch.cuda.synchronize()
    return time.perf_counter() - t


def timed(tr, name, parts):
    import torch
    fn = getattr(tr, name)

    def wrapped(*a, **k):
        torch.cuda.synchronize()
        t = time.perf_counter()
        out = fn(*a, **k)
        torch.cuda.synchronize()
        parts.setdefault(name, []).append(time.perf_counter() - t)
        return out
    setattr(tr, name, wrapped)


def run_trainer(tr):
    import torch
    parts = {}
    for name in ("_snapshot", "_side_file", "_kernel_points", "validation", "_epoch_end"):
        timed(tr, name, parts)
    torch.cuda.synchronize()
    t = time.perf_counter()
    tr.train()
    torch.cuda.synchronize()
    return time.perf_counter() - t, parts


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--reps", type=int, default=2)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("trainer_bench.py needs a GPU")
    dev = torch.device("cuda", 0)
    cfg, limits, train, val = setup(dev)
    steps = EPOCH_STEPS + 1
    warm = fresh(cfg, limits, train, val, dev, None)
    bare(warm, 3)
    warm.validation()
    reps = []
    with tempfile.TemporaryDirectory() as tmp:
        for r in range(args.reps):
            b = bare(fresh(cfg, limits, train, val, dev, None), steps)
            tr = fresh(cfg, limits, train, val, dev, os.path.join(tmp, "run%d" % r))
            total, parts = run_trainer(tr)
            assert tr.history[0]["epoch_n"] == steps
            first_kp, end_kp = parts["_kernel_points"]                  # kernel_points/epoch0 before the loop
            snapshot = parts["_snapshot"][0] + parts["_side_file"][0] + end_kp
            end = parts["_epoch_end"][0]
            rest = end - snapshot - parts["validation"][0]
            loop = total - end - first_kp
            reps.append(dict(bare_ms_per_step=1e3 * b / steps, trainer_ms_per_step=1e3 * loop / steps,
                             overhead_ms_per_step=1e3 * (loop - b) / steps, snapshot_s=snapshot,
                             validation_s=parts["validation"][0], means_and_logs_ms=1e3 * rest, train_s=total))
            print(json.dumps(reps[-1]))
    res = dict(card=card(), workload="3DMatch config, 2 x 30000-point room_fragment pairs, %d steps, validation_size 2"
               % steps, neighborhood_limits=limits, reps=reps)
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "trainer_bench.json"), "w") as fh:
        json.dump(res, fh, indent=1)
    print(res["card"])


if __name__ == "__main__":
    main()
