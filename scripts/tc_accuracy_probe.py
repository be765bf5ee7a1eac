"""GPU probe: max-norm relative error of the wgmma 3xTF32 GEMM vs float64 as a function of K."""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from d3feat_b200 import convolution_ops as co
dev = torch.device("cuda", 0)
for (M, K, N) in [(512, 32, 128), (512, 256, 128), (512, 1024, 128), (512, 4096, 128), (512, 7680, 512), (2048, 7680, 512)]:
    for dist in ("normal", "positive"):
        rng = np.random.default_rng(K)
        x = rng.normal(size=(M, K)).astype(np.float32)
        w = (rng.normal(size=(K, N)) / np.sqrt(K)).astype(np.float32)
        if dist == "positive":
            x, w = np.abs(x), np.abs(w)
        ref = x.astype(np.float64) @ w.astype(np.float64)
        tx, tw = torch.from_numpy(x).to(dev), torch.from_numpy(w).to(dev)
        res = {}
        for tc in (True, False):
            co.USE_TENSOR_CORES = tc
            o = co.unary_convolution(tx, tw).cpu().numpy().astype(np.float64)
            res[tc] = (np.abs(o - ref).max() / np.abs(ref).max(), np.mean(o - ref) / np.abs(ref).mean())
        print(f"M={M} K={K} N={N} {dist:8s} tc: max={res[True][0]:.2e} bias={res[True][1]:+.2e} | ffma: max={res[False][0]:.2e} bias={res[False][1]:+.2e}")
