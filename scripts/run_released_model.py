"""Descriptors + detection scores of point-cloud fragments with a RELEASED reference snapshot, no TensorFlow:

    python scripts/run_released_model.py --log /path/to/results/Log_contraloss --out out_dir a.ply b.ply ...

(the demo_registration.py / tester.generate_descriptor flow: voxelise at first_subsampling_dl, features = ones,
model -> [N,32] descriptors and [N,1] scores, rows written in ascending score order). Needs an H100 (sm_90a).
"""
import argparse
import glob
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from d3feat_b200 import io_utils, pyramid, tf_checkpoint          # noqa: E402
from d3feat_b200 import tf_custom_ops as ops                        # noqa: E402
from d3feat_b200.encoder import KPFCNN                              # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log", required=True, help="results/Log_* directory (parameters.txt + snapshots/)")
    ap.add_argument("--snap", type=int, default=None, help="snapshot number (default: the latest)")
    ap.add_argument("--out", required=True)
    ap.add_argument("--scene", default="demo")
    ap.add_argument("clouds", nargs="+", help=".ply or .npy point clouds")
    args = ap.parse_args()

    cfg = io_utils.load_config(args.log)
    snaps = sorted(glob.glob(os.path.join(args.log, "snapshots", "snap-*.index")),
                   key=lambda p: int(os.path.basename(p)[5:-6]))
    if args.snap is not None:
        snaps = [p for p in snaps if os.path.basename(p) == "snap-%d.index" % args.snap]
    if not snaps:
        raise SystemExit("no snapshot under %s" % args.log)
    params = tf_checkpoint.load_params(snaps[-1][:-6])
    dev = torch.device("cuda", 0)

    clouds = []
    for path in args.clouds:
        raw = np.load(path).astype(np.float32) if path.endswith(".npy") else io_utils.read_ply_points(path)
        p = torch.from_numpy(raw).to(dev)
        sub, _ = ops.batch_grid_subsampling(p, torch.tensor([p.shape[0]], dtype=torch.int32, device=dev),
                                            cfg.first_subsampling_dl)
        clouds.append(sub.cpu().numpy())
        print("%s: %d raw points -> %d at dl=%.3f" % (path, raw.shape[0], sub.shape[0], cfg.first_subsampling_dl))
    limits = pyramid.calibrate_neighbors(cfg, clouds, device=dev)
    print("neighbourhood limits:", limits)
    enc = KPFCNN(cfg, params, limits, device=dev)
    for i, c in enumerate(clouds):
        out = enc(c, np.array([c.shape[0]], np.int32))
        paths = io_utils.write_fragment(args.out, args.scene, i, c, out["descriptors"].cpu().numpy(),
                                        out["scores"].cpu().numpy())
        print("fragment %d: %s" % (i, ", ".join(paths)))


if __name__ == "__main__":
    main()
