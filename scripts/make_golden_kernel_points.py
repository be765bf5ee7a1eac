"""tests/golden/kernel_dispositions.npz: runs of the reference's own kernel-point optimiser
(kernels/kernel_points.py:41-181, kernel_point_optimization_debug, with load_kernels' 100 tries) for K in {7, 15, 32}
with 'center' and K = 15 with 'none' and 'verticals'. It imports the function from a D3Feat checkout and executes it;
nothing of it is copied. Development time only (needs the D3Feat sources):

    python scripts/make_golden_kernel_points.py /path/to/D3Feat

The function draws its initial points from numpy's global stream (seeded here, np.random.seed(1)); a trace of its
frame records them after the reshape of :83, and the loop index at the return. Per case "<fixed>_<K>|...":
  initial  [100, K, 3]   the points :76-83 drew, before the fixing of :85-91
  rows     [m]           rows 0-31, every 32nd row and the last 8 rows the loop wrote (the fixture stays small)
  saved    [m, 100]      saved_gradient_norms[rows] (rows from n on, up to 10000, are zero)
  iterations             n: the rows written (the `iter` at the break, plus one)
  points   [100, K, 3]   every try's returned points (radius 1, ratio 1)
  best_k                 np.argmin(saved_gradient_norms[-1]) (:214)
"""
import argparse
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CASES = (("center", 7), ("center", 15), ("center", 32), ("none", 15), ("verticals", 15))
TRIES = 100


def traced_run(fn, K, fixed):
    code = fn.__code__
    seen = {}

    def local(frame, event, arg):
        kp = frame.f_locals.get("kernel_points")
        if event == "line" and "initial" not in seen and kp is not None and kp.ndim == 3:
            seen["initial"] = np.array(kp, copy=True)       # after the reshape of :83, before the fixing
        if event == "return":
            seen["iter"] = frame.f_locals["iter"]
        return local

    def glob(frame, event, arg):
        return local if frame.f_code is code else None

    sys.settrace(glob)
    try:
        points, saved = fn(1.0, K, num_kernels=TRIES, dimension=3, fixed=fixed, verbose=0)
    finally:
        sys.settrace(None)
    return seen, points, saved


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("reference", help="root of a D3Feat checkout (holds kernels/kernel_points.py)")
    args = ap.parse_args()
    sys.path.insert(0, os.path.abspath(args.reference))
    from kernels.kernel_points import kernel_point_optimization_debug as fn
    out = {}
    for fixed, K in CASES:
        np.random.seed(1)
        t = time.time()
        seen, points, saved = traced_run(fn, K, fixed)
        n = int(seen["iter"]) + 1
        assert not saved[n:].any() and saved[n - 1].all()
        key = "%s_%d|" % (fixed, K)
        out[key + "initial"] = seen["initial"]
        rows = np.unique(np.concatenate([np.arange(min(n, 32)), np.arange(0, n, 32), np.arange(max(n - 8, 0), n)]))
        out[key + "rows"] = rows
        out[key + "saved"] = saved[rows]
        out[key + "iterations"] = np.int64(n)
        out[key + "points"] = points
        out[key + "best_k"] = np.int64(np.argmin(saved[-1, :]))
        print(fixed, K, "iterations", n, "best_k", int(out[key + "best_k"]), "%.1f s" % (time.time() - t))
    path = os.path.join(ROOT, "tests", "golden", "kernel_dispositions.npz")
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
