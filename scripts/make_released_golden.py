#!/usr/bin/env python
"""Write tests/golden/released_checkpoints.npz from the reference's released artefacts (argument: the reference
tree). What tests/test_checkpoint_io.py reads, as bytes, without the 56 MB tensor payloads:

  <tag>|index                the snapshot's .index file (names, dtypes, shapes, offsets, CRC32C of every tensor)
  <tag>|data_size            size of the snapshot's .data-00000-of-00001 file
  <tag>|parameters           the log's parameters.txt
  kitti61|data|<name>        the payload bytes of the 10 kernel-point tensors of snap-61
  kitti61|ply|<file>         kernel_points/epoch61/<file>.ply, written by the trainer from the same variables
  demo|cloud_bin_0_head      demo_data/cloud_bin_0.ply cut to its first 2000 vertices (vertex count edited)
  demo|cloud_bin_0_points    those 2000 vertices as read from the full file

    python scripts/make_released_golden.py <reference tree>
"""
import glob
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from d3feat_b200 import io_utils                 # noqa: E402
from d3feat_b200 import tf_checkpoint as ck      # noqa: E402

LOGS = (("kitti61", "results_kitti/Log_11011605", 61), ("contraloss54", "results/Log_contraloss", 54),
        ("circleloss48", "results/Log_circleloss", 48))
HEAD_VERTICES = 2000


def raw(path):
    with open(path, "rb") as fh:
        return np.frombuffer(fh.read(), np.uint8)


def main(ref):
    out = {}
    for tag, log, snap in LOGS:
        prefix = os.path.join(ref, log, "snapshots", "snap-%d" % snap)
        out[tag + "|index"] = raw(prefix + ".index")
        out[tag + "|data_size"] = np.array(os.path.getsize(prefix + ".data-00000-of-00001"), np.int64)
        out[tag + "|parameters"] = raw(os.path.join(ref, log, "parameters.txt"))
    prefix = os.path.join(ref, LOGS[0][1], "snapshots", "snap-61")
    _, entries = ck.read_index(prefix)
    data = raw(prefix + ".data-00000-of-00001")
    for name, e in entries.items():
        if name.endswith("kernel_points"):
            out["kitti61|data|" + name] = data[e["offset"]:e["offset"] + e["size"]].copy()
    for f in sorted(glob.glob(os.path.join(ref, LOGS[0][1], "kernel_points", "epoch61", "*.ply"))):
        out["kitti61|ply|" + os.path.basename(f)[:-4]] = raw(f)
    demo = os.path.join(ref, "demo_data", "cloud_bin_0.ply")
    full = raw(demo).tobytes()
    end = full.index(b"end_header\n") + len(b"end_header\n")
    header = full[:end].decode("ascii")
    n = int([ln for ln in header.splitlines() if ln.startswith("element vertex")][0].split()[-1])
    pts = io_utils.read_ply_points(demo)
    rec = (len(full) - end) // n
    head = header.replace("element vertex %d" % n, "element vertex %d" % HEAD_VERTICES).encode("ascii")
    out["demo|cloud_bin_0_head"] = np.frombuffer(head + full[end:end + HEAD_VERTICES * rec], np.uint8)
    out["demo|cloud_bin_0_points"] = pts[:HEAD_VERTICES]
    path = os.path.join(ROOT, "tests", "golden", "released_checkpoints.npz")
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path))


if __name__ == "__main__":
    main(sys.argv[1])
