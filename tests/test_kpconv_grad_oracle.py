"""The float64 restatement of the KPConv and unary gradients, and the argument checks of the autograd wrappers.

The restatement (tests/_kpconv_grad_oracle.py: kpconv_features_grad, kpconv_weights_grad, unary_*_grad) is checked
against the existing forward restatement kpconv_ops (oracle/kpconv_np.py), which no gradient code touches:
  * the adjoint identity <dL/df, df'> = <dout, F(df')> and <dL/dW, dW'> = <dout, F_W(dW')>, with F the forward with
    the neighbour count nn held at its value from f, to float64 rounding;
  * central differences of <dout, kpconv_ops(...)> on small cases.
Every influence and mode, K in {1, 15, 64}, Cin = 1, shadow padding (and -1 padding), duplicate supports in a row and
supports that no query reaches.

With the library replaced by a stub whose every symbol raises, the gradient entry points refuse wrong gradient dtypes,
devices and shapes, and the autograd wrappers refuse what has no gradient here, before anything reaches the library.
"""
import numpy as np
import pytest
import torch

from oracle import kpconv_np as ok
import _kpconv_grad_oracle as og

INFLUENCES = ["constant", "linear", "gaussian"]
MODES = ["sum", "closest"]


def make_case(rng, Nq=14, Ns=18, H=9, Cin=5, Cout=4, K=15, extent=0.5, unreached=3):
    """A small cloud with radius neighbours, shadow and -1 padding, a duplicated support in some rows and `unreached`
    supports (the last ones) that no query names."""
    s = rng.uniform(0, 1, (Ns, 3)).astype(np.float32)
    q = rng.uniform(0, 1, (Nq, 3)).astype(np.float32)
    reach = Ns - unreached
    idx = np.full((Nq, H), Ns, np.int64)
    for i in range(Nq):
        d = np.linalg.norm(s[:reach] - q[i], axis=1)
        near = np.argsort(d, kind="stable")[:H - 2]
        near = near[d[near] < 2.5 * extent]
        idx[i, :len(near)] = near
        if len(near) and i % 3 == 0:
            idx[i, len(near)] = near[0]                   # duplicate support in the row
        if i % 4 == 1:
            idx[i, -1] = -1                               # -1 padding of the non-batch op
    f = rng.normal(size=(Ns, Cin))
    f += np.sign(f.sum(1, keepdims=True)) * 0.3           # row sums away from 0: the nn vote is stable under +-eps
    f[::5] = -np.abs(f[::5])                              # some rows vote 0
    Kp = rng.normal(size=(K, 3)) * 0.6 * extent
    if K > 1:
        Kp[0] = 0
    W = rng.normal(size=(K, Cin, Cout))
    dout = rng.normal(size=(Nq, Cout))
    return q, s, idx.astype(np.int32), f.astype(np.float32), Kp.astype(np.float32), W.astype(np.float32), dout, extent


def nn_count(x, idx):
    xs = np.concatenate([x, np.zeros((1, x.shape[1]))], 0)
    Ns = x.shape[0]
    ii = np.where((idx < 0) | (idx > Ns), Ns, idx)
    return np.maximum((xs[ii].sum(-1) > 0).sum(-1), 1).astype(np.float64)


def forward(q, s, idx, f, Kp, W, extent, influence, mode, nn_from=None):
    """kpconv_ops in float64, with nn held at its value from `nn_from` when given."""
    out = ok.kpconv_ops(q, s, idx, f, Kp, W, extent, influence, mode, dtype=np.float64)
    if nn_from is not None:
        out = out * (nn_count(np.asarray(f, np.float64), idx) / nn_count(np.asarray(nn_from, np.float64), idx))[:, None]
    return out


CASES = [(inf, mode, K, Cin) for inf in INFLUENCES for mode in MODES for K, Cin in ((1, 5), (15, 5), (64, 3))]
CASES += [(inf, mode, 15, 1) for inf in INFLUENCES for mode in MODES]


@pytest.mark.parametrize("influence,mode,K,Cin", CASES)
def test_adjoint_identity(influence, mode, K, Cin):
    rng = np.random.default_rng(K * 10 + Cin + 100 * INFLUENCES.index(influence) + 1000 * MODES.index(mode))
    q, s, idx, f, Kp, W, dout, ext = make_case(rng, K=K, Cin=Cin)
    df, df_mag, _ = og.kpconv_features_grad(q, s, idx, f, Kp, W, ext, influence, mode, dout)
    dW, dW_mag, _ = og.kpconv_weights_grad(q, s, idx, f, Kp, W, ext, influence, mode, dout)
    assert df.shape == f.shape and dW.shape == W.shape
    reached = np.zeros(s.shape[0], bool)
    reached[idx[(idx >= 0) & (idx < s.shape[0])]] = True
    assert not reached[-3:].any() and np.all(df[~reached] == 0)
    for trial in range(3):
        pf = rng.normal(size=f.shape)
        pW = rng.normal(size=W.shape)
        lhs = np.sum(df * pf)
        rhs = np.sum(dout * forward(q, s, idx, pf, Kp, W, ext, influence, mode, nn_from=f))
        assert abs(lhs - rhs) <= 1e-12 * np.sum(df_mag * np.abs(pf)) + 1e-300, (lhs, rhs)
        lhs = np.sum(dW * pW)
        rhs = np.sum(dout * forward(q, s, idx, f, Kp, pW, ext, influence, mode))
        assert abs(lhs - rhs) <= 1e-12 * np.sum(dW_mag * np.abs(pW)) + 1e-300, (lhs, rhs)


@pytest.mark.parametrize("influence", INFLUENCES)
@pytest.mark.parametrize("mode", MODES)
def test_central_differences(influence, mode):
    rng = np.random.default_rng(7 + INFLUENCES.index(influence) + 10 * MODES.index(mode))
    q, s, idx, f, Kp, W, dout, ext = make_case(rng, Nq=10, Ns=12, H=7, Cin=3, Cout=2, K=15, unreached=2)
    f64, W64 = f.astype(np.float64), W.astype(np.float64)
    df, _, _ = og.kpconv_features_grad(q, s, idx, f, Kp, W, ext, influence, mode, dout)
    dW, _, _ = og.kpconv_weights_grad(q, s, idx, f, Kp, W, ext, influence, mode, dout)
    loss = lambda ff, ww: np.sum(dout * ok.kpconv_ops(q, s, idx, ff, Kp, ww, ext, influence, mode, dtype=np.float64))
    eps = 1e-6
    for _ in range(6):
        i, c = rng.integers(f.shape[0]), rng.integers(f.shape[1])
        e = np.zeros_like(f64)
        e[i, c] = eps
        num = (loss(f64 + e, W64) - loss(f64 - e, W64)) / (2 * eps)
        assert abs(num - df[i, c]) <= 1e-6 * (1 + abs(df[i, c])), (i, c, num, df[i, c])
        k, c, o = rng.integers(W.shape[0]), rng.integers(W.shape[1]), rng.integers(W.shape[2])
        e = np.zeros_like(W64)
        e[k, c, o] = eps
        num = (loss(f64, W64 + e) - loss(f64, W64 - e)) / (2 * eps)
        assert abs(num - dW[k, c, o]) <= 1e-6 * (1 + abs(dW[k, c, o])), (k, c, o, num, dW[k, c, o])


def test_unary_restatement():
    rng = np.random.default_rng(3)
    x, w, g = rng.normal(size=(9, 5)), rng.normal(size=(5, 4)), rng.normal(size=(9, 4))
    dx, dx_mag, _ = og.unary_features_grad(x, w, g)
    dw, dw_mag, _ = og.unary_weights_grad(x, w, g)
    px, pw = rng.normal(size=x.shape), rng.normal(size=w.shape)
    assert abs(np.sum(dx * px) - np.sum(g * ok.unary_convolution(px, w))) <= 1e-12 * np.sum(dx_mag * np.abs(px))
    assert abs(np.sum(dw * pw) - np.sum(g * ok.unary_convolution(x, pw))) <= 1e-12 * np.sum(dw_mag * np.abs(pw))


# ---- the wrappers refuse before the library ----------------------------------------------------------------------

class Stub:
    def __getattr__(self, symbol):
        raise AssertionError("reached the library: %s" % symbol)


@pytest.fixture
def host(monkeypatch):
    from d3feat_b200 import _lib
    monkeypatch.setattr(_lib, "DEVICE_TYPE", "cpu")
    monkeypatch.setattr(_lib, "lib", lambda: Stub())


def kp_args(req_f=False, req_w=False):
    Nq, Ns, H, K, Cin, Cout = 5, 7, 4, 15, 8, 6
    z = lambda *sh, dt=torch.float32: torch.zeros(sh, dtype=dt)
    f, W = z(Ns, Cin).requires_grad_(req_f), z(K, Cin, Cout).requires_grad_(req_w)
    return [z(Nq, 3), z(Ns, 3), z(Nq, H, dt=torch.int32), f, z(K, 3), W, 0.3, "linear", "sum"], (Nq, Cout)


WRONG_GRAD = [("float64", lambda sh: torch.zeros(sh, dtype=torch.float64)),
              ("float16", lambda sh: torch.zeros(sh, dtype=torch.float16)),
              ("int32", lambda sh: torch.zeros(sh, dtype=torch.int32)),
              ("device", lambda sh: torch.zeros(sh, device="meta")),
              ("rows+1", lambda sh: torch.zeros((sh[0] + 1, sh[1]))),
              ("cols+1", lambda sh: torch.zeros((sh[0], sh[1] + 1))),
              ("rank+1", lambda sh: torch.zeros((1,) + sh)),
              ("list", lambda sh: np.zeros(sh, np.float32).tolist())]


@pytest.mark.parametrize("case", [c for c, _ in WRONG_GRAD])
def test_kpconv_backward_refuses_bad_grad(host, case):
    from d3feat_b200 import convolution_ops as co
    args, shape = kp_args()
    g = dict(WRONG_GRAD)[case](shape)
    with pytest.raises(ValueError, match="kpconv_backward: grad_out"):
        co.kpconv_backward(*args, g)


@pytest.mark.parametrize("case", [c for c, _ in WRONG_GRAD])
def test_unary_backward_refuses_bad_grad(host, case):
    from d3feat_b200 import convolution_ops as co
    x, w = torch.zeros(6, 8), torch.zeros(8, 5)
    g = dict(WRONG_GRAD)[case]((6, 5))
    with pytest.raises(ValueError, match="unary_backward: grad_out"):
        co.unary_backward(x, w, g)


def test_backward_checks_the_forward_arguments_too(host):
    from d3feat_b200 import convolution_ops as co
    args, shape = kp_args()
    args[2] = args[2].long()
    with pytest.raises(ValueError, match="kpconv_backward: neighbors_indices"):
        co.kpconv_backward(*args, torch.zeros(shape))
    with pytest.raises(ValueError, match="unary_backward: K_values"):
        co.unary_backward(torch.zeros(6, 8), torch.zeros(9, 5), torch.zeros(6, 5))
    with pytest.raises(ValueError, match="unary_backward: rows"):
        co.unary_backward(torch.zeros(6, 8), torch.zeros(8, 5), torch.zeros(6, 5),
                          rows=torch.zeros(2, dtype=torch.int32))


def test_legal_backward_reaches_the_library(host):
    from d3feat_b200 import convolution_ops as co
    args, shape = kp_args()
    with pytest.raises(AssertionError, match="reached the library"):
        co.kpconv_backward(*args, torch.zeros(shape))
    with pytest.raises(AssertionError, match="reached the library"):
        co.unary_backward(torch.zeros(6, 8), torch.zeros(8, 5), torch.zeros(6, 5))
    assert co.kpconv_backward(*args, torch.zeros(shape), features_grad=False, weights_grad=False) == (None, None)


def _unsupported():
    from d3feat_b200 import convolution_ops as co, network_blocks as nb
    z = torch.zeros
    c = lambda: z(6)
    args, _ = kp_args(req_f=True)
    argsw, _ = kp_args(req_w=True)
    x = lambda: z(6, 8).requires_grad_(True)
    return {
        "KPConv_ops epilogue": lambda: co.KPConv_ops(*args, epilogue=(c(), c(), 0.2)),
        "KPConv_ops bias": lambda: co.KPConv_ops(*argsw, bias=c()),
        "KPConv_ops bias requires grad": lambda: co.KPConv_ops(*kp_args()[0], bias=c().requires_grad_(True)),
        "unary epilogue": lambda: co.unary_convolution(x(), z(8, 6), epilogue=(c(), c(), None)),
        "unary residual": lambda: co.unary_convolution(z(6, 8), z(8, 6).requires_grad_(True), residual=z(6, 6)),
        "KPConv_deform_ops": lambda: co.KPConv_deform_ops(*args[:5], z(5, 15, 3), None, *args[5:]),
        "KPConv_deformable": lambda: co.KPConv_deformable(args[0], args[1], args[2], args[3], argsw[5]),
        "unary_pair_convolution": lambda: co.unary_pair_convolution(x(), z(8, 6), (c(), c()), z(6, 4), z(4, 6),
                                                                    (c(), c()), 0.2),
        "ind_max_pool": lambda: nb.ind_max_pool(x(), z(3, 2, dtype=torch.int32)),
        "closest_pool": lambda: nb.closest_pool(x(), z(3, 2, dtype=torch.int32)),
    }


@pytest.mark.parametrize("name", sorted(_unsupported()))
def test_unsupported_gradient_is_refused(host, name):
    op = name.split()[0]
    with pytest.raises(NotImplementedError, match=op):
        _unsupported()[name]()
    with torch.no_grad():                 # the same call without a gradient is the plain forward
        with pytest.raises((AssertionError, ValueError)):
            _unsupported()[name]()


def test_plain_path_without_grad(host, monkeypatch):
    """No input requiring grad, or grad mode off: the autograd Functions are not entered."""
    from d3feat_b200 import convolution_ops as co
    entered = []
    monkeypatch.setattr(co._KPConvFn, "apply", lambda *a: entered.append("kpconv"))
    monkeypatch.setattr(co._UnaryFn, "apply", lambda *a: entered.append("unary"))
    for args in (kp_args()[0],):
        with pytest.raises(AssertionError, match="reached the library"):
            co.KPConv_ops(*args)
    with torch.no_grad():
        with pytest.raises(AssertionError, match="reached the library"):
            co.KPConv_ops(*kp_args(req_f=True, req_w=True)[0])
        with pytest.raises(AssertionError, match="reached the library"):
            co.unary_convolution(torch.zeros(4, 3, requires_grad=True), torch.zeros(3, 2, requires_grad=True))
    assert entered == []
    co.KPConv_ops(*kp_args(req_w=True)[0])
    co.unary_convolution(torch.zeros(4, 3), torch.zeros(3, 2, requires_grad=True))
    assert entered == ["kpconv", "unary"]
