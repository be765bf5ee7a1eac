#!/usr/bin/env python
"""Write tests/golden/reference_digests.json: SHA-256 digests of what the reference's own compiled C++ cores
(oracle/_ref, built by `make -C oracle ref`) return on the inputs of the tests that compare against them, in the
canonical forms those tests use (point sets row-sorted by bits, neighbour rows ordered by (d2, index)). A digest pins
a result of any size bit for bit in 64 characters, so the comparisons run where the reference cores cannot be built.

    python scripts/make_golden_ref_digests.py
"""
import hashlib
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import native as on          # noqa: E402
from d3feat_b200 import synth            # noqa: E402


def digest(a):
    a = np.ascontiguousarray(a)
    return dict(shape=list(a.shape), dtype=str(a.dtype), sha256=hashlib.sha256(a.tobytes()).hexdigest())


def point_set(points):
    """Row-sorted uint32 bit patterns: the canonical form of an unordered point set."""
    return on.sort_rows(np.ascontiguousarray(points, np.float32).view(np.uint32))[0]


def subsampling(points, lengths, dl):
    rp, rb = on.ref_batch_subsampling(points, lengths, dl)
    o, clouds = 0, []
    for n in rb:
        clouds.append(digest(point_set(rp[o:o + n])))
        o += n
    return dict(lengths=[int(n) for n in rb], clouds=clouds)


def neighbors(q, s, qb, sb, r):
    ref = on.ref_batch_neighbors(q, s, qb, sb, r)
    return digest(on.canonicalize_neighbors(ref, q, s, s.shape[0])[0].astype(np.int32))


def main():
    assert on.have_ref(), "oracle/_ref is not built"
    out = {}
    # tests/test_oracle_golden.py::test_port_vs_compiled_reference_random
    rng = np.random.default_rng(0)
    trials = []
    for _ in range(3):
        n1, n2 = rng.integers(200, 1500, 2)
        P = rng.uniform(-1, 1, (n1 + n2, 3)).astype(np.float32)
        L = np.array([n1, n2], np.int32)
        r = float(rng.uniform(0.1, 0.3))
        trials.append(dict(neighbors=neighbors(P, P, L, L, r), subsampling=subsampling(P, L, r)))
    out["random_trials"] = trials
    # tests/test_gpu_real_configs.py::test_micro_1m_bit_exact_vs_reference_cores
    P = synth.surface_cloud(0, 1000000)
    n = np.array([P.shape[0]], np.int32)
    sub = subsampling(P, n, 0.03)
    rp, _ = on.port_batch_subsampling(P, n, 0.03)           # same point set as the reference (checked by the digest)
    assert digest(point_set(rp)) == sub["clouds"][0]
    m = np.array([rp.shape[0]], np.int32)
    out["micro_1m"] = dict(subsampling=sub, neighbors=neighbors(rp, rp, m, m, 0.075))
    path = os.path.join(ROOT, "tests", "golden", "reference_digests.json")
    with open(path, "w") as fh:
        json.dump(out, fh, indent=1)
    print(path)


if __name__ == "__main__":
    main()
