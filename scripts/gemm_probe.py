"""GPU: time the wgmma GEMM at the encoder's characteristic shapes (CUDA events, warm)."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from d3feat_b200 import convolution_ops as co
dev = torch.device("cuda", 0)
shapes = [(4177, 3840, 256), (1204, 7680, 512), (26112, 480, 32), (240000, 32, 128), (240000, 64, 128), (60336, 64, 256), (1204, 1024, 2048),
          (240000, 480, 32), (240000, 64, 32), (240000, 128, 32), (60336, 960, 64), (60336, 128, 64), (60336, 480, 32)]
only = os.environ.get("ONLY_SHAPE")
for i, (M, K, N) in enumerate(shapes):
    if only is not None and int(only) != i:
        continue
    x = torch.randn(M, K, device=dev); w = torch.randn(K, N, device=dev) / K ** 0.5
    for _ in range(3): co.unary_convolution(x, w)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    n = 20
    e0.record()
    for _ in range(n): co.unary_convolution(x, w)
    e1.record(); torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / n
    fl = 2.0 * M * K * N
    by = 4.0 * (M * K + 2 * K * N + M * N)
    print("M=%6d K=%5d N=%5d  %.3f ms  %.1f TFLOP/s(fp32-equiv)  %.2f TB/s(min bytes)  nk=%d ctas=%d" % (M, K, N, ms, fl / ms / 1e9, by / ms / 1e9, (K + 31) // 32, ((M + 127) // 128) * ((N + 127) // 128)))
