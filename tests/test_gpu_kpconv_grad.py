"""GPU: the feature and weight gradients of rigid KPConv and of the unary convolution, element by element against the
float64 restatement (tests/_kpconv_grad_oracle.py: kpconv_features_grad / kpconv_weights_grad / unary_*_grad):

    |gpu - ref| <= 1e-5 * mag          (tests/_oracle.py TOL; `alt` for closest-mode ties and nn votes)

over the channel pairs of the forward tests, every influence x mode, K in {1, 7, 15, 64}, a query order, capacity-sized
buffers with device row counts, Nq = 0, and the level-0 and level-1 layers of the bench workload's pyramid. Also:
loss.backward() through KPConv / unary_convolution fills .grad with the direct entry points' values, the gradients are
bitwise identical run to run and across streams, and without a gradient the forward launches the same kernels and
gives the same bits as before.
"""
import numpy as np
import pytest
import torch

from oracle import kpconv_np as ok
import _kpconv_grad_oracle as og
from _oracle import assert_close

pytestmark = pytest.mark.gpu


def t(a, dev):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def make_case(rng, Nq, Ns, H, Cin, Cout, K=15, extent=0.06, unreached=0):
    """Radius neighbours (brute force) of Nq queries among Ns supports, shadow padding, duplicates in some rows; the
    last `unreached` supports are named by no query."""
    s = rng.uniform(0, 1, (Ns, 3)).astype(np.float32)
    q = s[:Nq].copy() if Nq <= Ns else rng.uniform(0, 1, (Nq, 3)).astype(np.float32)
    reach = Ns - unreached
    idx = np.full((Nq, H), Ns, np.int32)
    r = 2.5 * extent
    for a in range(0, Nq, 512):
        d2 = ((q[a:a + 512, None, :] - s[None, :reach, :]) ** 2).sum(-1)
        order = np.argsort(d2, axis=1, kind="stable")[:, :H]
        ok_ = np.take_along_axis(d2, order, 1) < r * r
        idx[a:a + 512] = np.where(ok_, order, Ns)
    idx[::7, -1] = idx[::7, 0]                                   # a duplicated support in some rows
    f = rng.normal(size=(Ns, Cin)).astype(np.float32)
    Kp = rng.normal(size=(K, 3))
    if K > 1:
        Kp[0] = 0
        Kp[1:] *= 1.5 * extent / np.linalg.norm(Kp[1:], axis=1, keepdims=True)
    else:
        Kp[:] = 0
    W = (rng.normal(size=(K, Cin, Cout)) * np.sqrt(2.0 / Cout)).astype(np.float32)
    dout = rng.normal(size=(Nq, Cout)).astype(np.float32)
    return q, s, idx, f, Kp.astype(np.float32), W, dout


def gpu_grads(dev, q, s, idx, f, Kp, W, dout, extent, influence="linear", mode="sum", **kw):
    from d3feat_b200 import convolution_ops as co
    df, dW = co.kpconv_backward(t(q, dev), t(s, dev), t(idx, dev), t(f, dev), t(Kp, dev), t(W, dev), extent, influence,
                                mode, t(dout, dev), **kw)
    return df.cpu().numpy(), dW.cpu().numpy()


def check(what, q, s, idx, f, Kp, W, dout, extent, influence, mode, df, dW):
    ref, mag, alt = og.kpconv_features_grad(q, s, idx, f, Kp, W, extent, influence, mode, dout)
    assert_close(df, ref, mag, what=what + " df", alt=alt)
    ref, mag, alt = og.kpconv_weights_grad(q, s, idx, f, Kp, W, extent, influence, mode, dout)
    assert_close(dW, ref, mag, what=what + " dW", alt=alt)


@pytest.mark.parametrize("Cin,Cout,Nq,Ns", [(1, 64, 3000, 3000), (32, 32, 3000, 3000), (64, 64, 900, 3000),
                                            (128, 128, 700, 700), (256, 256, 300, 300), (48, 40, 500, 500)])
def test_kpconv_grad_matches_restatement(cuda, Cin, Cout, Nq, Ns):
    rng = np.random.default_rng(Cin * 1000 + Cout)
    extent = 0.06 if Ns >= 2000 else 0.12
    q, s, idx, f, Kp, W, dout = make_case(rng, Nq, Ns, 40, Cin, Cout, extent=extent, unreached=5)
    if Cin == 1:
        f = np.ones_like(f)
    df, dW = gpu_grads(cuda, q, s, idx, f, Kp, W, dout, extent)
    assert np.all(df[-5:] == 0), "supports no query reaches must get a zero gradient"
    check("grad %dx%d" % (Cin, Cout), q, s, idx, f, Kp, W, dout, extent, "linear", "sum", df, dW)


@pytest.mark.parametrize("influence", ["constant", "linear", "gaussian"])
@pytest.mark.parametrize("mode", ["sum", "closest"])
@pytest.mark.parametrize("Cin", [1, 32])
def test_kpconv_grad_influence_and_mode(cuda, influence, mode, Cin):
    rng = np.random.default_rng(5 + Cin)
    q, s, idx, f, Kp, W, dout = make_case(rng, 800, 800, 32, Cin, 48, extent=0.1)
    f[::3] = -np.abs(f[::3])
    df, dW = gpu_grads(cuda, q, s, idx, f, Kp, W, dout, 0.1, influence, mode)
    check("grad %s/%s Cin=%d" % (influence, mode, Cin), q, s, idx, f, Kp, W, dout, 0.1, influence, mode, df, dW)


@pytest.mark.parametrize("K", [1, 7, 15, 64])
@pytest.mark.parametrize("mode", ["sum", "closest"])
def test_kpconv_grad_any_K(cuda, K, mode):
    rng = np.random.default_rng(40 + K)
    q, s, idx, f, Kp, W, dout = make_case(rng, 500, 600, 24, 12, 20, K=K, extent=0.12, unreached=3)
    df, dW = gpu_grads(cuda, q, s, idx, f, Kp, W, dout, 0.12, "linear", mode)
    check("grad K=%d %s" % (K, mode), q, s, idx, f, Kp, W, dout, 0.12, "linear", mode, df, dW)


@pytest.mark.parametrize("Cin,Cout", [(1, 64), (32, 32), (64, 64)])
def test_kpconv_grad_through_query_order(cuda, Cin, Cout):
    """Autograd through KPConv_ops(query_order=...) gives the gradients of the plain call, bit for bit."""
    from d3feat_b200 import convolution_ops as co
    rng = np.random.default_rng(11 + Cin)
    q, s, idx, f, Kp, W, dout = make_case(rng, 2500, 2500, 40, Cin, Cout, extent=0.08)
    perm = t(rng.permutation(2500).astype(np.int32), cuda)
    grads = []
    for order in (None, perm):
        ft, Wt = t(f, cuda).requires_grad_(True), t(W, cuda).requires_grad_(True)
        out = co.KPConv_ops(t(q, cuda), t(s, cuda), t(idx, cuda), ft, t(Kp, cuda), Wt, 0.08, "linear", "sum",
                            query_order=order)
        out.backward(t(dout, cuda))
        grads.append((ft.grad, Wt.grad))
    assert torch.equal(grads[0][0], grads[1][0]) and torch.equal(grads[0][1], grads[1][1])
    check("grad order %dx%d" % (Cin, Cout), q, s, idx, f, Kp, W, dout, 0.08, "linear", "sum",
          grads[1][0].cpu().numpy(), grads[1][1].cpu().numpy())


@pytest.mark.parametrize("Cin,Cout", [(1, 64), (32, 32), (48, 40)])
def test_kpconv_grad_capacity_buffers(cuda, Cin, Cout):
    """Capacity-sized buffers with device row counts: rows past the counts hold NaN (points, features, grad_out) and
    out-of-range indices; dL/df rows past rows_s are zero, nothing past the counts is read."""
    rng = np.random.default_rng(77 + Cin)
    nq, ns, Nq, Ns = 700, 900, 1000, 1300
    q, s, idx, f, Kp, W, dout = make_case(rng, nq, ns, 32, Cin, Cout, extent=0.1, unreached=4)
    if Cin == 1:
        f = np.abs(f)
    qc = np.full((Nq, 3), np.nan, np.float32); qc[:nq] = q
    sc = np.full((Ns, 3), np.nan, np.float32); sc[:ns] = s
    fc = np.full((Ns, Cin), np.nan, np.float32); fc[:ns] = f
    gc = np.full((Nq, Cout), np.nan, np.float32); gc[:nq] = dout
    ic = rng.integers(0, Ns + 1, (Nq, 32)).astype(np.int32); ic[:nq] = idx   # shadow = ns; > ns inside: shadow too
    ic[:nq:5, 3] = ns + 7
    rq, rs = (torch.tensor([v], dtype=torch.int32, device=cuda) for v in (nq, ns))
    df, dW = gpu_grads(cuda, qc, sc, ic, fc, Kp, W, gc, 0.1, rows_q=rq, rows_s=rs)
    assert np.all(df[ns:] == 0) and np.isfinite(df).all() and np.isfinite(dW).all()
    ref_idx = np.where(ic[:nq] > ns, ns, ic[:nq])
    check("grad capacity %dx%d" % (Cin, Cout), q, s, ref_idx, f, Kp, W, dout, 0.1, "linear", "sum", df[:ns], dW)


def test_kpconv_grad_empty(cuda):
    from d3feat_b200 import convolution_ops as co
    z = lambda *sh, dt=torch.float32: torch.zeros(sh, dtype=dt, device=cuda)
    df, dW = co.kpconv_backward(z(0, 3), z(7, 3), z(0, 4, dt=torch.int32), torch.ones(7, 32, device=cuda), z(15, 3),
                                torch.ones(15, 32, 16, device=cuda), 0.3, "linear", "sum", z(0, 16))
    assert df.shape == (7, 32) and dW.shape == (15, 32, 16)
    assert bool((df == 0).all()) and bool((dW == 0).all())
    df, dW = co.kpconv_backward(z(5, 3), z(0, 3), z(5, 4, dt=torch.int32), z(0, 32), z(15, 3), z(15, 32, 16), 0.3,
                                "linear", "sum", torch.ones(5, 16, device=cuda))
    assert df.shape == (0, 32) and bool((dW == 0).all())


@pytest.mark.parametrize("N,Cin,Cout", [(5000, 32, 64), (3000, 64, 32), (1000, 37, 19), (300000, 32, 32)])
@pytest.mark.parametrize("with_rows", [False, True])
def test_unary_grad_matches_restatement(cuda, N, Cin, Cout, with_rows):
    from d3feat_b200 import convolution_ops as co
    rng = np.random.default_rng(N + Cin)
    x = rng.normal(size=(N, Cin)).astype(np.float32)
    w = rng.normal(size=(Cin, Cout)).astype(np.float32)
    g = rng.normal(size=(N, Cout)).astype(np.float32)
    n = N - N // 3 if with_rows else N
    if with_rows:
        x[n:] = np.nan
        g[n:] = np.nan
    rows = torch.tensor([n], dtype=torch.int32, device=cuda) if with_rows else None
    dx, dw = co.unary_backward(t(x, cuda), t(w, cuda), t(g, cuda), rows=rows)
    dx, dw = dx.cpu().numpy(), dw.cpu().numpy()
    assert np.all(dx[n:] == 0)
    ref, mag, alt = og.unary_features_grad(x[:n], w, g[:n])
    assert_close(dx[:n], ref, mag, what="unary dx %d %dx%d" % (N, Cin, Cout), alt=alt)
    ref, mag, alt = og.unary_weights_grad(x[:n], w, g[:n])
    assert_close(dw, ref, mag, what="unary dW %d %dx%d" % (N, Cin, Cout), alt=alt)


def test_backward_through_autograd_equals_direct(cuda):
    from d3feat_b200 import convolution_ops as co
    rng = np.random.default_rng(3)
    q, s, idx, f, Kp, W, dout = make_case(rng, 1500, 1500, 32, 32, 64, extent=0.1)
    qt, st, it = t(q, cuda), t(s, cuda), t(idx, cuda)
    ft, Wt = t(f, cuda).requires_grad_(True), t(W, cuda).requires_grad_(True)
    W2 = t(rng.normal(size=(64, 16)).astype(np.float32), cuda).requires_grad_(True)
    feats = co.KPConv(qt, st, it, ft, Wt, KP_extent=0.1)
    y = co.unary_convolution(feats, W2)
    g = t(rng.normal(size=(1500, 16)).astype(np.float32), cuda)
    (y * g).sum().backward()
    # the direct entry points, chained by hand
    dfeats, dW2 = co.unary_backward(feats.detach(), W2.detach(), g)
    Kp_used = co._kernel_points(0.15, 15, cuda, "center")
    df, dW = co.kpconv_backward(qt, st, it, ft.detach(), Kp_used, Wt.detach(), 0.1, "linear", "sum", dfeats)
    assert torch.equal(W2.grad, dW2) and torch.equal(Wt.grad, dW) and torch.equal(ft.grad, df)
    # only what requires grad is computed
    ft2 = t(f, cuda).requires_grad_(True)
    co.KPConv_ops(qt, st, it, ft2, Kp_used, t(W, cuda), 0.1, "linear", "sum").backward(t(dout, cuda)[:, :64])
    assert torch.equal(ft2.grad, co.kpconv_backward(qt, st, it, ft2.detach(), Kp_used, t(W, cuda), 0.1, "linear",
                                                    "sum", t(dout, cuda)[:, :64], weights_grad=False)[0])


def test_gradients_are_deterministic_across_calls_and_streams(cuda):
    from d3feat_b200 import convolution_ops as co
    rng = np.random.default_rng(9)
    q, s, idx, f, Kp, W, dout = make_case(rng, 6000, 6000, 40, 32, 32, extent=0.05)
    args = [t(a, cuda) for a in (q, s, idx, f, Kp, W)] + [0.05, "linear", "sum", t(dout, cuda)]
    x, w, g = (t(rng.normal(size=sh).astype(np.float32), cuda) for sh in ((9000, 64), (64, 32), (9000, 32)))
    first = co.kpconv_backward(*args) + co.unary_backward(x, w, g)
    again = co.kpconv_backward(*args) + co.unary_backward(x, w, g)
    streams = [torch.cuda.Stream() for _ in range(2)]
    res = []
    for st in streams:
        st.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(st):
            res.append(co.kpconv_backward(*args) + co.unary_backward(x, w, g))
    torch.cuda.synchronize()
    for other in [again] + res:
        for a, b in zip(first, other):
            assert torch.equal(a, b)


def test_no_grad_path_is_the_forward(cuda):
    """Without a gradient (no input requires grad, or torch.no_grad()) the ops launch the kernels of the plain forward
    and give its bits; with one, the forward inside the autograd Function is the same launch sequence too. Kernel
    names come from torch.profiler in a fresh process (a long pytest process can leave CUPTI recording nothing);
    the library's own launch counter is compared here as well."""
    import os
    import subprocess
    import sys
    _no_grad_check(lambda fn: (fn(), None))
    tests = os.path.dirname(os.path.abspath(__file__))
    code = ("import sys; sys.path[:0] = [%r, %r]; import test_gpu_kpconv_grad as m; "
            "from test_gpu_kernel_variants import launched; m._no_grad_check(launched); print('ok')"
            % (tests, os.path.dirname(tests)))
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "ok" in r.stdout, r.stdout[-2000:] + r.stderr[-4000:]


def _no_grad_check(launched):
    """launched(fn) -> (fn(), set of kernel names or None)."""
    from d3feat_b200 import _lib, convolution_ops as co
    cuda = torch.device("cuda", 0)
    counted = launched

    def launched(fn):
        c0 = _lib.launch_count()
        out, names = counted(fn)
        return out, (names, _lib.launch_count() - c0)
    rng = np.random.default_rng(12)
    for Cin, Cout in ((1, 64), (32, 32), (64, 64), (48, 40)):
        q, s, idx, f, Kp, W, _ = make_case(rng, 2000, 2000, 40, Cin, Cout, extent=0.08)
        base = [t(a, cuda) for a in (q, s, idx, f, Kp, W)]
        fr, Wr = base[3].clone().requires_grad_(True), base[5].clone().requires_grad_(True)
        grad_args = base[:3] + [fr, base[4], Wr]

        def plain():
            return co.KPConv_ops(*base, 0.08, "linear", "sum")

        def no_grad():
            with torch.no_grad():
                return co.KPConv_ops(*grad_args, 0.08, "linear", "sum")

        def with_grad():
            return co.KPConv_ops(*grad_args, 0.08, "linear", "sum")
        plain(), no_grad(), with_grad()             # pack the weight images outside the profiled calls
        out0, n0 = launched(plain)
        out1, n1 = launched(no_grad)
        out2, n2 = launched(with_grad)
        assert n0 == n1 == n2, (n0, n1, n2)
        assert torch.equal(out0, out1) and torch.equal(out0, out2.detach()) and out2.grad_fn is not None
        assert out1.grad_fn is None
    x, w = (t(rng.normal(size=sh).astype(np.float32), cuda) for sh in ((5000, 32), (32, 64)))
    wr = w.clone().requires_grad_(True)
    co.unary_convolution(x, w), co.unary_convolution(x, wr)
    u0, m0 = launched(lambda: co.unary_convolution(x, w))
    with torch.no_grad():
        u1, m1 = launched(lambda: co.unary_convolution(x, wr))
    u2, m2 = launched(lambda: co.unary_convolution(x, wr))
    assert m0 == m1 == m2 and torch.equal(u0, u1) and torch.equal(u0, u2.detach())


def _bench_pyramid(dev):
    from d3feat_b200 import synth
    from d3feat_b200.encoder import KPFCNN
    cfg = synth.Config(architecture=synth.ARCH_ENCODER)
    clouds = [synth.room_fragment(i, 30000) for i in range(8)]
    pts = np.concatenate(clouds, 0).astype(np.float32)
    lens = np.array([len(c) for c in clouds], np.int32)
    enc = KPFCNN(cfg, synth.make_params(cfg, seed=0), [40] * 5, device=dev)
    return cfg, enc.build_inputs(pts, lens)


@pytest.mark.parametrize("level,C", [(0, 32), (1, 64)])
def test_kpconv_grad_bench_pyramid(cuda, level, C):
    """The level-0 (32 -> 32) and level-1 (64 -> 64) layer shapes of the 8 x 30 000 bench workload, on the pyramid the
    library builds (calibrated neighbour columns): dL/dW everywhere, dL/df on sampled support rows."""
    cfg, inputs = _bench_pyramid(cuda)
    pts = inputs["points"][level].cpu().numpy()
    idx = inputs["neighbors"][level].cpu().numpy()
    N = pts.shape[0]
    extent = cfg.KP_extent * cfg.first_subsampling_dl * 2 ** level
    rng = np.random.default_rng(level)
    f = rng.normal(size=(N, C)).astype(np.float32)
    Kp = rng.normal(size=(15, 3))
    Kp[0] = 0
    Kp[1:] *= 1.5 * extent / np.linalg.norm(Kp[1:], axis=1, keepdims=True)
    Kp = Kp.astype(np.float32)
    W = (rng.normal(size=(15, C, C)) * np.sqrt(2.0 / C)).astype(np.float32)
    dout = rng.normal(size=(N, C)).astype(np.float32)
    df, dW = gpu_grads(cuda, pts, pts, idx, f, Kp, W, dout, extent)
    ref, mag, alt = og.kpconv_weights_grad(pts, pts, idx, f, Kp, W, extent, "linear", "sum", dout)
    assert_close(dW, ref, mag, what="grad bench level %d dW" % level, alt=alt)
    sample = np.sort(rng.choice(N, 300, replace=False))
    users = np.nonzero(np.isin(idx, sample).any(1))[0]           # every query that reaches a sampled support
    ref, mag, alt = og.kpconv_features_grad(pts[users], pts, idx[users], f, Kp, W, extent, "linear", "sum",
                                            dout[users])
    assert_close(df[sample], ref[sample], mag[sample], what="grad bench level %d df" % level, alt=alt[sample])
