"""GPU: the wgmma (3xTF32, register accumulator) GEMM path vs float64, and vs the CUDA-core fp32 path."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def t(a, dev):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def rel_err(a, b):
    a = np.asarray(a, np.float64)
    b = np.asarray(b, np.float64)
    return np.abs(a - b).max() / max(np.abs(b).max(), 1e-30)


@pytest.mark.parametrize("M,K,N", [(128, 32, 32), (128, 64, 128), (1000, 480, 32), (300, 96, 45), (645, 1024, 256),
                                   (195, 512, 2048), (5000, 128, 64), (77, 36, 200), (4096, 7680, 512)])
def test_tc_gemm_matches_float64(cuda, monkeypatch, M, K, N):
    from d3feat_b200 import convolution_ops as co
    rng = np.random.default_rng(M + K + N)
    x = rng.normal(size=(M, K)).astype(np.float32)
    w = (rng.normal(size=(K, N)) / np.sqrt(K)).astype(np.float32)
    ref = x.astype(np.float64) @ w.astype(np.float64)
    tx, tw = t(x, cuda), t(w, cuda)
    monkeypatch.setattr(co, "USE_TENSOR_CORES", True)
    out_tc = co.unary_convolution(tx, tw).cpu().numpy()
    monkeypatch.setattr(co, "USE_TENSOR_CORES", False)
    out_cc = co.unary_convolution(tx, tw).cpu().numpy()
    e_tc, e_cc = rel_err(out_tc, ref), rel_err(out_cc, ref)
    # 3xTF32 keeps ~21 mantissa bits per product; the tensor pipe's own accumulate is restarted every 32-wide k-chunk
    # and the chunks are summed with round-to-nearest (tc_gemm.cu)
    assert e_tc < 3e-5, (e_tc, e_cc)
    assert e_cc < 1e-5, (e_tc, e_cc)


def test_tc_gemm_epilogue_and_row_tail(cuda, monkeypatch):
    from d3feat_b200 import convolution_ops as co
    monkeypatch.setattr(co, "USE_TENSOR_CORES", True)
    rng = np.random.default_rng(0)
    M, K, N = 333, 64, 96
    x = rng.normal(size=(M, K)).astype(np.float32)
    w = (rng.normal(size=(K, N)) / 8).astype(np.float32)
    scale = rng.uniform(0.5, 1.5, N).astype(np.float32)
    shift = rng.normal(size=N).astype(np.float32)
    res = rng.normal(size=(M, N)).astype(np.float32)
    out = co.unary_convolution(t(x, cuda), t(w, cuda), epilogue=(t(scale, cuda), t(shift, cuda), 0.2),
                               residual=t(res, cuda)).cpu().numpy()
    y = (x.astype(np.float64) @ w.astype(np.float64)) * scale + shift + res
    y = np.where(y > 0, y, 0.2 * y)
    assert rel_err(out, y) < 1e-5


def test_packed_weight_cache_tracks_tensor_identity(cuda, monkeypatch):
    from d3feat_b200 import convolution_ops as co
    monkeypatch.setattr(co, "USE_TENSOR_CORES", True)
    x = torch.randn(256, 64, device=cuda)
    outs = []
    for i in range(4):                       # fresh weight tensors of the same shape (addresses get recycled)
        w = torch.randn(64, 64, device=cuda)
        out = co.unary_convolution(x, w)
        ref = (x.double() @ w.double())
        assert (out.double() - ref).abs().max() / ref.abs().max() < 1e-5
        del w
    w = torch.randn(64, 64, device=cuda)
    a = co.unary_convolution(x, w)
    w.mul_(2.0)                              # in-place update bumps _version -> re-pack
    b = co.unary_convolution(x, w)
    assert torch.allclose(b, 2 * a, rtol=1e-5, atol=1e-5)


@pytest.mark.parametrize("N,C1,C2,Cout", [(5000, 32, 64, 128), (3001, 64, 128, 256), (700, 512, 1024, 2048),
                                          (900, 48, 64, 96), (1, 32, 32, 32)])
def test_unary_pair_convolution(cuda, N, C1, C2, Cout):
    """conv3 + shortcut + add + LeakyReLU as one GEMM over the concatenated K (BN scales folded into the weights)
    vs the float64 evaluation of the two separate unaries; (48, 64) does not tile and takes the two-call path."""
    from d3feat_b200 import convolution_ops as co
    rng = np.random.default_rng(N + C1)
    x1 = rng.normal(size=(N, C1)).astype(np.float32)
    x2 = rng.normal(size=(N, C2)).astype(np.float32)
    w1 = (rng.normal(size=(C1, Cout)) / np.sqrt(C1)).astype(np.float32)
    w2 = (rng.normal(size=(C2, Cout)) / np.sqrt(C2)).astype(np.float32)
    s1, s2 = (rng.uniform(0.5, 1.5, Cout).astype(np.float32) for _ in range(2))
    t1, t2 = (rng.normal(size=Cout).astype(np.float32) for _ in range(2))
    tt = lambda a: torch.from_numpy(a).to(cuda)
    W1, W2 = tt(w1), tt(w2)
    args = (tt(x1), W1, (tt(s1), tt(t1)), tt(x2), W2, (tt(s2), tt(t2)), 0.2)
    y = co.unary_pair_convolution(*args).cpu().numpy()
    y_again = co.unary_pair_convolution(*args).cpu().numpy()          # second call: cached folded weights
    ref = (x1.astype(np.float64) @ w1) * s1 + t1 + (x2.astype(np.float64) @ w2) * s2 + t2
    ref = np.where(ref > 0, ref, 0.2 * ref)
    assert np.abs(y - ref).max() <= 3e-5 * np.abs(ref).max()
    assert np.array_equal(y, y_again)
    with pytest.raises(ValueError):
        co.unary_pair_convolution(tt(x1), W1, (tt(s1), tt(t1)), tt(x2[:, :-4]), W2, (tt(s2), tt(t2)), 0.2)


@pytest.mark.parametrize("M,K,N", [(40000, 64, 32), (38001, 480, 32), (45003, 128, 64), (39000, 960, 64),
                                   (20011, 96, 128), (19000, 192, 256), (38000, 256, 64), (40000, 512, 48),
                                   (19001, 320, 128), (240000, 480, 32)])
@pytest.mark.parametrize("stream", [0, 1])
def test_streaming_gemm_large_m(cuda, monkeypatch, M, K, N, stream):
    """Huge-M GEMMs vs float64, through the default one-tile-per-CTA kernels (stream = 0) and through the opt-in
    persistent launch (D3F_TC_STREAM=1: one CTA per SM walks several tiles, the operand ring running across
    tiles). Ragged last tile, partial column tile (N = 48), BN + LeakyReLU + residual epilogue,
    several n-tiles per row block, and a device-side row count below the launch capacity."""
    from d3feat_b200 import convolution_ops as co
    monkeypatch.setattr(co, "USE_TENSOR_CORES", True)
    monkeypatch.setenv("D3F_TC_STREAM", str(stream))
    rng = np.random.default_rng(M + K + N)
    x = rng.normal(size=(M, K)).astype(np.float32)
    w = (rng.normal(size=(K, N)) / np.sqrt(K)).astype(np.float32)
    scale = rng.uniform(0.5, 1.5, N).astype(np.float32)
    shift = rng.normal(size=N).astype(np.float32)
    res = rng.normal(size=(M, N)).astype(np.float32)
    tx, tw = t(x, cuda), t(w, cuda)
    out = co.unary_convolution(tx, tw).cpu().numpy()
    ref = x.astype(np.float64) @ w.astype(np.float64)
    assert rel_err(out, ref) < 3e-5
    out = co.unary_convolution(tx, tw, epilogue=(t(scale, cuda), t(shift, cuda), 0.2), residual=t(res, cuda)).cpu().numpy()
    y = ref * scale + shift + res
    y = np.where(y > 0, y, 0.2 * y)
    assert rel_err(out, y) < 3e-5
    # device-side row count
    m_true = M - 777
    rows = torch.tensor([m_true], dtype=torch.int32, device=cuda)
    part = co.unary_convolution(tx, tw, rows=rows)
    torch.cuda.synchronize()
    assert rel_err(part[:m_true].cpu().numpy(), ref[:m_true]) < 3e-5


def test_streaming_pair_convolution_large_m(cuda):
    """conv3 + shortcut as one GEMM over the concatenated K through the streaming variant (level-0 shape)."""
    from d3feat_b200 import convolution_ops as co
    rng = np.random.default_rng(5)
    N, C1, C2, Cout = 30011, 32, 64, 128
    x1 = rng.normal(size=(N, C1)).astype(np.float32)
    x2 = rng.normal(size=(N, C2)).astype(np.float32)
    w1 = (rng.normal(size=(C1, Cout)) / np.sqrt(C1)).astype(np.float32)
    w2 = (rng.normal(size=(C2, Cout)) / np.sqrt(C2)).astype(np.float32)
    s1, s2 = (rng.uniform(0.5, 1.5, Cout).astype(np.float32) for _ in range(2))
    t1, t2 = (rng.normal(size=Cout).astype(np.float32) for _ in range(2))
    y = co.unary_pair_convolution(t(x1, cuda), t(w1, cuda), (t(s1, cuda), t(t1, cuda)), t(x2, cuda), t(w2, cuda),
                                  (t(s2, cuda), t(t2, cuda)), 0.2).cpu().numpy()
    ref = (x1.astype(np.float64) @ w1) * s1 + t1 + (x2.astype(np.float64) @ w2) * s2 + t2
    ref = np.where(ref > 0, ref, 0.2 * ref)
    assert np.abs(y - ref).max() <= 3e-5 * np.abs(ref).max()
