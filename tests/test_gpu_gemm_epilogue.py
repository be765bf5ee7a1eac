"""GPU: the shared-memory epilogue of the wgmma GEMM (tc_gemm.cu). Every store path -- 16-byte row pieces when N is a
multiple of 4, single floats otherwise, ragged row and column tiles, a device row count below the capacity, the row
map of a cell-ordered KPConv -- against float64, bit for bit against the same product through the other store path, and
against a sentinel-filled output for writes out of bounds."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

TOL = 3e-5          # 3xTF32 with chunked accumulation, as in test_gpu_tensor_core.py
SENTINEL = -12345.0


def rel_err(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return np.abs(a - b).max() / max(np.abs(b).max(), 1e-30)


def unary_into(out, x, w, M, *, scale=None, shift=None, bias=None, residual=None, alpha=-1.0, rows=None):
    """d3f_unary_forward writing into a caller-owned (sentinel-filled) buffer."""
    from d3feat_b200 import _lib
    from d3feat_b200 import convolution_ops as co
    K, N = w.shape
    _lib.check(_lib.lib().d3f_unary_forward(_lib.ptr(x), _lib.ptr(w), _lib.ptr(co.packed_weight(w)), M, K, N,
                                            _lib.ptr(scale), _lib.ptr(shift), _lib.ptr(bias), _lib.ptr(residual),
                                            alpha, _lib.ptr(out), _lib.stream(), _lib.ptr(rows)), "d3f_unary_forward")


def reference(x, w, scale, shift, bias, res, alpha):
    y = x.astype(np.float64) @ w.astype(np.float64)
    if scale is not None:
        y = y * scale + shift
    if bias is not None:
        y = y + bias
    if res is not None:
        y = y + res
    if alpha is not None:
        y = np.where(y > 0, y, alpha * y)
    return y


SHAPES = [(1, 32, 1), (127, 64, 31), (128, 32, 32), (129, 128, 33), (128, 64, 64), (8191, 480, 100), (8191, 128, 256),
          (129, 480, 128), (127, 32, 256), (240000, 64, 128), (240000, 32, 32)]


@pytest.mark.parametrize("M,K,N", SHAPES)
@pytest.mark.parametrize("variant", ["plain", "bn_leaky_res", "bias_rows"])
def test_epilogue_variants_and_bounds(cuda, monkeypatch, M, K, N, variant):
    from d3feat_b200 import convolution_ops as co
    monkeypatch.setattr(co, "USE_TENSOR_CORES", True)
    rng = np.random.default_rng(7 * M + 3 * K + N)
    x = rng.normal(size=(M, K)).astype(np.float32)
    w = (rng.normal(size=(K, N)) / np.sqrt(K)).astype(np.float32)
    scale = shift = bias = res = alpha = None
    m_true = M
    if variant == "bn_leaky_res":
        scale, shift = rng.uniform(0.5, 1.5, N).astype(np.float32), rng.normal(size=N).astype(np.float32)
        res, alpha = rng.normal(size=(M, N)).astype(np.float32), 0.2
    elif variant == "bias_rows":                 # no BN, no LeakyReLU, a device row count below the capacity
        bias = rng.normal(size=N).astype(np.float32)
        m_true = M - min(M - 1, 77) if M > 1 else 1
    dv = lambda a: None if a is None else torch.from_numpy(np.ascontiguousarray(a)).to(cuda)
    tx, tw = dv(x), dv(w)
    guard = 64
    out = torch.full((M * N + guard,), SENTINEL, dtype=torch.float32, device=cuda)
    rows = torch.tensor([m_true], dtype=torch.int32, device=cuda) if m_true != M else None
    unary_into(out, tx, tw, M, scale=dv(scale), shift=dv(shift), bias=dv(bias), residual=dv(res),
               alpha=-1.0 if alpha is None else alpha, rows=rows)
    got = out.cpu().numpy()
    ref = reference(x, w, scale, shift, bias, res, alpha)
    assert rel_err(got[:m_true * N].reshape(m_true, N), ref[:m_true]) < TOL
    # nothing past row *m_dev, nothing past the matrix
    assert np.all(got[m_true * N:] == SENTINEL)

    # The same product as columns [0, N) of a GEMM one column wider: N and N + 1 cannot both be multiples of 4, so one
    # of the two goes out as 16-byte pieces and the other float by float (often through another column tile width).
    # Each output element sees the same operations in the same order, hence the same bits.
    w1 = np.concatenate([w, rng.normal(size=(K, 1)).astype(np.float32)], 1)
    ext = lambda v: None if v is None else np.concatenate([v, np.ones(1, np.float32)])
    res1 = None if res is None else np.concatenate([res, np.zeros((M, 1), np.float32)], 1)
    out1 = torch.full((M * (N + 1) + guard,), SENTINEL, dtype=torch.float32, device=cuda)
    unary_into(out1, tx, dv(w1), M, scale=dv(ext(scale)), shift=dv(ext(shift)), bias=dv(ext(bias)),
               residual=dv(res1), alpha=-1.0 if alpha is None else alpha, rows=rows)
    got1 = out1.cpu().numpy()
    assert np.array_equal(got1[:m_true * (N + 1)].reshape(m_true, N + 1)[:, :N], got[:m_true * N].reshape(m_true, N))
    assert np.all(got1[m_true * (N + 1):] == SENTINEL)


@pytest.mark.parametrize("M,C1,C2,N", [(129, 32, 64, 128), (8191, 32, 64, 100), (240000, 32, 64, 128)])
def test_pair_gemm_epilogue(cuda, M, C1, C2, N):
    """K = 96 as [32 | 64]: the two-matrix A operand with the bias + LeakyReLU epilogue."""
    from d3feat_b200 import convolution_ops as co
    rng = np.random.default_rng(M + N)
    x1, x2 = rng.normal(size=(M, C1)).astype(np.float32), rng.normal(size=(M, C2)).astype(np.float32)
    w1 = (rng.normal(size=(C1, N)) / np.sqrt(C1)).astype(np.float32)
    w2 = (rng.normal(size=(C2, N)) / np.sqrt(C2)).astype(np.float32)
    s1, s2 = (rng.uniform(0.5, 1.5, N).astype(np.float32) for _ in range(2))
    t1, t2 = (rng.normal(size=N).astype(np.float32) for _ in range(2))
    dv = lambda a: torch.from_numpy(a).to(cuda)
    W1, W2 = dv(w1), dv(w2)
    y = co.unary_pair_convolution(dv(x1), W1, (dv(s1), dv(t1)), dv(x2), W2, (dv(s2), dv(t2)), 0.2).cpu().numpy()
    ref = (x1.astype(np.float64) @ w1) * s1 + t1 + (x2.astype(np.float64) @ w2) * s2 + t2
    ref = np.where(ref > 0, ref, 0.2 * ref)
    assert rel_err(y, ref) < TOL


@pytest.mark.parametrize("Cin,Cout", [(32, 32), (64, 100)])
def test_row_map_scatter_matches_identity(cuda, Cin, Cout):
    """KPConv's contraction (rowscale, K = 15 Cin) scatters its rows through the query order. A permuted order, the
    identity order and no order at all give every query the same output row, bit for bit."""
    from d3feat_b200 import convolution_ops as co
    rng = np.random.default_rng(Cin + Cout)
    n, H, K = 3001, 24, 15
    pts = rng.uniform(0, 1, size=(n, 3)).astype(np.float32)
    idx = rng.integers(0, n + 1, size=(n, H)).astype(np.int32)        # n = the shadow index
    f = rng.normal(size=(n, Cin)).astype(np.float32)
    W = (rng.normal(size=(K, Cin, Cout)) / np.sqrt(K * Cin)).astype(np.float32)
    Kp = rng.uniform(-0.1, 0.1, size=(K, 3)).astype(np.float32)
    dv = lambda a: torch.from_numpy(a).to(cuda)
    P, I, F, Wd, Kd = dv(pts), dv(idx), dv(f), dv(W), dv(Kp)
    outs = []
    for order in (None, np.arange(n, dtype=np.int32), rng.permutation(n).astype(np.int32)):
        o = None if order is None else dv(order)
        outs.append(co.KPConv_ops(P, P, I, F, Kd, Wd, 0.12, "linear", "sum", query_order=o).cpu().numpy())
    assert np.isfinite(outs[0]).all() and np.abs(outs[0]).max() > 0
    assert np.array_equal(outs[0], outs[1])
    assert np.array_equal(outs[0], outs[2])
