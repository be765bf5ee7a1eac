"""CPU: the float64 check of the training replay (tests/test_gpu_training_replay.py) is tight enough to matter.

  * the explicit adjoints with magnitudes (tests/_training_oracle.py) equal the autograd restatement to ~1e-12
    (detection scores, batch norm, the max pool, the gather, l2_normalize), and every magnitude bounds its |ref|;
  * at the replay's op shapes, _oracle.assert_close at TOL accepts a float32 evaluation of each op that follows the
    kernel's arithmetic, and rejects numpy emulations of plausible kernel bugs: batch norm's dx without the
    xhat * dgamma / N term, the first, a middle or the short last 2048-row block partial dropped from dgamma / dbeta,
    and, at x = 1e3 + N(0, 1), the missing xhat term, a zero or doubled dx and a halved dgamma; max-pool ties routed
    all to the first entry, the max-pool shadow share dropped, a repeated gather index counted once, the l2 eps branch
    inverted, the detection cloud-max share dropped, the detection neighbour-mean term added to the query row instead
    of the neighbour. For each, whether the old max-norm check (max |err| / max |ref| at 1e-5 and at TOL_NET = 3e-3)
    would have accepted it is asserted as well: the inverted l2 eps branch passes TOL_NET;
  * with the ops replaced by shape-only fakes, training.forward + d3feat_loss records the per-kind call counts that
    _training_replay.expected_calls derives from ARCH_3DMATCH, skips the no-grad forward inside the convolutions'
    Functions, and gives every record its upstream gradient.
"""
import numpy as np
import pytest
import torch

import _training_oracle as ot
import _training_replay as rp
from _oracle import TOL, ratio

F32, F64 = np.float32, np.float64
TOL_NET = 3e-3
ROW_BLOCK = 2048


def worst(out, ref, mag, alt=None):
    return float(ratio(out, ref, mag, alt).max())


def maxnorm(out, ref):
    return float(np.abs(np.asarray(out, F64) - ref).max() / np.abs(ref).max())


def rejects(name, bug, ref, mag, alt=None, *, old):
    """The element-wise check rejects `bug`. old = (accepted by max-norm at 1e-5, accepted by max-norm at TOL_NET):
    what the old check would have said, asserted both ways."""
    r = worst(bug, ref, mag, alt)
    m = maxnorm(bug, ref)
    print("%-36s element-wise %.3g x TOL, max-norm %.3g" % (name, r / TOL, m))
    assert r > TOL, name
    assert (m <= TOL, m <= TOL_NET) == tuple(old), (name, m)


# ---------------------------------------------------------------------------------------------------- adjoints

def test_detection_adjoint_equals_autograd():
    rng = np.random.default_rng(0)
    for lengths, N, H in [([300], 300, 12), ([120, 90, 0, 70], 300, 9), ([200], 240, 0), ([2100, 500], 2600, 6)]:
        x = rng.normal(size=(N, 8)) + 0.2
        x[::13] = 0.0
        x[5, 3] = x[:lengths[0]].max()                            # the cloud maximum tied across two rows
        nb = rng.integers(0, N, size=(N, H))
        if H:
            nb[:, -1] = N
            nb[::7, 0] = -1
        g = rng.normal(size=(N, 1))
        xt = ot.t64(x).requires_grad_(True)
        ot.detection_scores(xt, nb, lengths).backward(ot.t64(g))
        ref, mag, alt, amb = ot.detection_scores_grad(x, nb, lengths, g)
        want = xt.grad.numpy()
        assert np.abs(ref - want).max() <= 1e-12 * np.abs(want).max()
        assert np.all(mag >= np.abs(ref) * (1 - 1e-12)) and not amb.any()


def test_op_adjoints_equal_autograd():
    rng = np.random.default_rng(1)
    x = rng.normal(size=(50, 6)) * 2 + 0.5
    gm, bt, r, go = rng.uniform(0.5, 1.5, 6), rng.normal(size=6), rng.normal(size=(50, 6)), rng.normal(size=(50, 6))
    xt, gt, bt_, rt = (ot.t64(a).requires_grad_(True) for a in (x, gm, bt, r))
    out, mean, var = ot.batch_norm_train(xt, gt, bt_, rt, 0.2)
    out.backward(ot.t64(go))
    bw = ot.batch_norm_train_grads(x, out.detach().numpy(), go, gm, 0.2)
    fw = ot.batch_norm_train_forward_ref(x, gm, bt, r, 0.2)
    for got, want in ((bw["dx"][0], xt.grad), (bw["dgamma"][0], gt.grad), (bw["dbeta"][0], bt_.grad),
                      (bw["dres"][0], rt.grad), (fw["out"][0], out), (fw["mean"][0], mean),
                      (fw["invstd"][0], 1 / torch.sqrt(var + 1e-6))):
        want = want.detach().numpy()
        assert np.abs(got - want).max() <= 1e-12 * np.abs(want).max()
    for v, m in list(bw.values()) + list(fw.values()):
        assert np.all(m >= np.abs(v) * (1 - 1e-12))
    inds = rng.integers(0, 50, size=(20, 5))
    inds[:, -1] = 50
    x[:, 2] = 0.75
    g = rng.normal(size=(20, 6))
    xt = ot.t64(x).requires_grad_(True)
    ot.ind_max_pool(xt, inds).backward(ot.t64(g))
    dx, mag = ot.ind_max_pool_grad(x, inds, g)
    assert np.abs(dx - xt.grad.numpy()).max() <= 1e-12 and np.all(mag >= np.abs(dx) - 1e-12)
    gi = np.array([3, 3, 0, 50, 8, 3, -1])
    g = rng.normal(size=(7, 6))
    xt = ot.t64(x).requires_grad_(True)
    ot.gather_rows(xt, gi).backward(ot.t64(g))
    assert np.abs(ot.gather_rows_grad(gi, g, 50)[0] - xt.grad.numpy()).max() <= 1e-12
    y = rng.normal(size=(9, 6))
    y[2] *= 1e-7
    g = rng.normal(size=(9, 6))
    yt = ot.t64(y).requires_grad_(True)
    ot.l2_normalize(yt).backward(ot.t64(g))
    assert np.abs(ot.l2_normalize_grad(y, g)[0] - yt.grad.numpy()).max() <= 1e-12 * np.abs(yt.grad.numpy()).max()


# ---------------------------------------------------------------------------------------------------- sensitivity

def bn_kernel(x, out, dout, gamma, alpha, bug=None):
    """train_ops.cu's batch norm in numpy: the statistics and the backward's sums as float64 partials over 2048-row
    blocks added in block order, float32 everywhere else. Returns the gradients and the float32 mean / invstd."""
    N = x.shape[0]
    xd = x.astype(F64)
    mean = xd.mean(0).astype(F32)
    invstd = (1 / np.sqrt(np.square(xd - mean).mean(0).astype(F32).astype(F64) + 1e-6)).astype(F32)
    dz = np.where(out > 0, dout, F32(alpha) * dout).astype(F32)
    xh64 = (xd - mean) * invstd.astype(F64)
    blocks = list(range(0, N, ROW_BLOCK))
    if bug is not None and bug.startswith("dropped block"):
        del blocks[int(bug.split()[-1])]
    sb = sum(dz[a:a + ROW_BLOCK].astype(F64).sum(0) for a in blocks)
    sg = sum((dz[a:a + ROW_BLOCK] * xh64[a:a + ROW_BLOCK]).sum(0) for a in blocks)
    a_, b_ = (sb / N).astype(F32), (sg / N).astype(F32)
    if bug == "dgamma halved":
        sg = sg / 2
    xh = ((x - mean) * invstd).astype(F32)
    term = 0 if bug == "no xhat term" else xh * b_
    dx = (gamma.astype(F32) * invstd * (dz - a_ - term)).astype(F32)
    if bug == "dx zero":
        dx = np.zeros_like(dx)
    if bug == "dx doubled":
        dx = 2 * dx
    return dict(dx=dx, dgamma=sg.astype(F32), dbeta=sb.astype(F32), mean=mean, invstd=invstd)


def bn_case(rng, N, C, shift, correlated):
    x = (shift + rng.normal(size=(N, C)) * rng.uniform(0.5, 3, C) + rng.normal(size=C)).astype(F32)
    gamma = rng.uniform(0.5, 1.5, C).astype(F32)
    xd = x.astype(F64)
    out = (xd - xd.mean(0)).astype(F32)
    # correlated: the output gradient follows the centred input, so dgamma / N is of order one
    dout = (out if correlated else rng.normal(size=(N, C))).astype(F32)
    return x, out, dout, gamma


def bn_check(x, out, dout, gamma):
    """The float64 reference and magnitudes on the kernel's own batch statistics (batch_norm_backward's inputs), after
    the float32 evaluation and the kernel emulation pass."""
    k = bn_kernel(x, out, dout, gamma, 0.2)
    ref = ot.batch_norm_train_grads(x, out, dout, gamma, 0.2, mean=k["mean"], invstd=k["invstd"])
    f32 = ot.batch_norm_train_grads(x, out, dout, gamma, 0.2, dtype=F32, mean=k["mean"], invstd=k["invstd"])
    for n in ("dx", "dgamma", "dbeta"):
        assert worst(f32[n][0], *ref[n]) <= TOL and worst(k[n], *ref[n]) <= TOL, n
    return ref


def test_batch_norm_check_accepts_fp32_and_rejects_bugs():
    rng = np.random.default_rng(2)
    x, out, dout, gamma = bn_case(rng, 3 * ROW_BLOCK + 5, 64, 0.0, False)   # level-0 shape, short last block
    ref = bn_check(x, out, dout, gamma)
    rejects("bn dx without xhat*dgamma/N", bn_kernel(x, out, dout, gamma, 0.2, "no xhat term")["dx"], *ref["dx"],
            old=(False, False))
    for blk in (0, 1, 3):                                        # the first, a middle full and the short last block
        bug = bn_kernel(x, out, dout, gamma, 0.2, "dropped block %d" % blk)
        rejects("bn dgamma, block %d dropped" % blk, bug["dgamma"], *ref["dgamma"], old=(False, False))
        rejects("bn dbeta, block %d dropped" % blk, bug["dbeta"], *ref["dbeta"], old=(False, False))


@pytest.mark.parametrize("N,C", [(6145, 64), (2049, 33)])
@pytest.mark.parametrize("correlated", [False, True])
def test_batch_norm_check_mean_far_above_std(N, C, correlated):
    """x = 1e3 + N(0, 1), the GPU test's case: the check stays tight there."""
    x, out, dout, gamma = bn_case(np.random.default_rng(N + C), N, C, 1e3, correlated)
    ref = bn_check(x, out, dout, gamma)
    tag = "bn 1e3+N(0,1) %dx%d%s" % (N, C, " corr" if correlated else "")
    bug = lambda b: bn_kernel(x, out, dout, gamma, 0.2, b)
    rejects(tag + " no xhat", bug("no xhat term")["dx"], *ref["dx"], old=(False, False))
    rejects(tag + " dx zero", bug("dx zero")["dx"], *ref["dx"], old=(False, False))
    rejects(tag + " dx x2", bug("dx doubled")["dx"], *ref["dx"], old=(False, False))
    rejects(tag + " dgamma/2", bug("dgamma halved")["dgamma"], *ref["dgamma"], old=(False, False))


def pool_kernel(x, inds, dout, bug=None):
    """ind_max_pool_backward in numpy float32: the tie split, the shadow share through the column minimum."""
    N1, C = x.shape
    cmin = x.min(0)
    xs = np.concatenate([x, cmin[None]], 0)
    ii = np.where((inds < 0) | (inds >= N1), N1, inds)
    v = xs[ii]
    tie = v == v.max(1, keepdims=True)
    if bug == "ties to first":
        tie = tie & (np.cumsum(tie, 1) == 1)
    sh = np.where(tie, (dout / tie.sum(1))[:, None, :], F32(0)).astype(F32)
    acc = np.zeros((N1 + 1, C), F64)
    np.add.at(acc, ii.reshape(-1), sh.reshape(-1, C).astype(F64))
    at_min = x == cmin[None]
    share = (acc[N1].astype(F32) / at_min.sum(0)).astype(F32)
    dx = acc[:N1].astype(F32)
    if bug != "no shadow share":
        dx = dx + at_min * share
    return dx


def test_max_pool_check_accepts_fp32_and_rejects_bugs():
    rng = np.random.default_rng(3)
    N1, N2, H, C = 6000, 1700, 30, 64                              # level 0 -> 1 of the replay's 3DMatch pair
    x = np.where(rng.random((N1, C)) < 0.3, 0, rng.normal(size=(N1, C))).astype(F32)   # LeakyReLU-like zeros: ties
    x[:, 7] = 0.5                                                  # an all-equal column
    inds = rng.integers(0, N1, size=(N2, H)).astype(np.int32)
    inds[:, -8:] = N1                                              # shadow padding
    inds[-40:] = N1                                                # pooled rows with no real neighbour
    dout = rng.normal(size=(N2, C)).astype(F32)
    ref, mag = ot.ind_max_pool_grad(x, inds, dout)
    assert worst(ot.ind_max_pool_grad(x, inds, dout, dtype=F32)[0], ref, mag) <= TOL
    assert worst(pool_kernel(x, inds, dout), ref, mag) <= TOL
    rejects("pool ties to the first entry", pool_kernel(x, inds, dout, "ties to first"), ref, mag, old=(False, False))
    rejects("pool shadow share dropped", pool_kernel(x, inds, dout, "no shadow share"), ref, mag, old=(False, False))


def test_gather_check_accepts_fp32_and_rejects_bugs():
    rng = np.random.default_rng(4)
    n_rows, k, C = 30000, 256, 32                                  # the loss's keypoint gathers of descriptors
    inds = rng.choice(15000, k, replace=True).astype(np.int32)     # drawn with replacement: repeats
    inds[:3] = inds[3]
    dout = (rng.normal(size=(k, C)) * 1e-2).astype(F32)
    ref, mag = ot.gather_rows_grad(inds, dout, n_rows)
    assert worst(ot.gather_rows_grad(inds, dout, n_rows, dtype=F32)[0], ref, mag) <= TOL
    _, first = np.unique(inds, return_index=True)
    bug = ot.gather_rows_grad(inds[first], dout[first], n_rows, dtype=F32)[0]
    rejects("gather repeat counted once", bug, ref, mag, old=(False, False))


def test_l2_check_accepts_fp32_and_rejects_bugs():
    rng = np.random.default_rng(5)
    x = rng.normal(size=(30000, 32)).astype(F32)
    x[::997] *= F32(1e-7)                                          # a few rows below eps
    g = rng.normal(size=x.shape).astype(F32)
    ref, mag = ot.l2_normalize_grad(x, g)
    assert worst(ot.l2_normalize_grad(x, g, dtype=F32)[0], ref, mag) <= TOL
    s = np.square(x.astype(F64)).sum(1, keepdims=True)
    inv = (1 / np.sqrt(np.maximum(s, 1e-10))).astype(F32)
    y = x * inv
    bug = np.where(s < 1e-10, (g - y * (y * g).sum(1, keepdims=True)) * inv, g * inv)
    rejects("l2 eps branch inverted", bug, ref, mag, old=(False, True))


def det_case(rng, lengths, H=30, D=32):
    N = sum(lengths)
    x = (rng.normal(size=(N, D)) + 0.3).astype(F32)
    nb = np.full((N, H), N, np.int32)
    a = 0
    for n in lengths:
        nb[a:a + n, :H - 4] = rng.integers(a, a + n, size=(n, H - 4))
        a += n
    g = np.zeros((N, 1), F32)
    rows = rng.choice(N, 512, replace=False)                       # the anchors' and positives' scores
    g[rows, 0] = rng.normal(size=512) * 1e-2
    return x, nb, g


def test_detection_check_accepts_fp32_and_rejects_bugs():
    rng = np.random.default_rng(6)
    lengths = [3100, 2900]
    x, nb, g = det_case(rng, lengths)
    ref, mag, alt, amb = ot.detection_scores_grad(x, nb, lengths, g)
    f32, _, _, _, t = ot.detection_scores_grad(x, nb, lengths, g, dtype=F32, parts=True)
    assert amb.mean() < 1e-3
    assert worst(f32, ref, mag, alt) <= TOL
    rejects("det cloud-max share dropped", t["gx"] + t["scatter"], ref, mag, alt, old=(False, False))
    nvalid = ((nb >= 0) & (nb < x.shape[0])).sum(1, keepdims=True)
    rejects("det A on the query row", t["gx"] + t["A"] * nvalid + t["share"], ref, mag, alt, old=(False, False))


# ---------------------------------------------------------------------------------------------------- recorder

class Stub:
    def __getattr__(self, symbol):
        raise AssertionError("reached the library: %s" % symbol)


def test_recorder_counts_calls_on_shape_only_fakes(monkeypatch):
    from d3feat_b200 import _lib, synth, training as T, convolution_ops as co, variables as V
    monkeypatch.setattr(_lib, "DEVICE_TYPE", "cpu")
    monkeypatch.setattr(_lib, "lib", lambda: Stub())

    def bn(x, scope, config, residual=None, alpha=None):
        pre = scope + "/batch_normalization/"
        y = x * V.current_store().get(pre + "gamma") + V.current_store().get(pre + "beta")
        y = y if residual is None else y + residual
        return y if alpha is None else torch.where(y > 0, y, alpha * y)

    def unary(features, K_values, **kw):
        if torch.is_grad_enabled() and (features.requires_grad or K_values.requires_grad):
            with torch.no_grad():                                  # the forward _UnaryFn runs inside its own
                co.unary_convolution(features, K_values)
        return features @ K_values

    def kpconv(q, s, idx, f, Kp, W, extent, influence, mode, **kw):
        if torch.is_grad_enabled() and (f.requires_grad or W.requires_grad):
            with torch.no_grad():
                co.KPConv_ops(q, s, idx, f, Kp, W, extent, influence, mode, **kw)
        return (f[idx[:, 0].long()] @ W.sum(0)) / (1 + extent)

    monkeypatch.setattr(T, "batch_norm", bn)
    monkeypatch.setattr(co, "unary_convolution", unary)
    monkeypatch.setattr(co, "KPConv_ops", kpconv)
    monkeypatch.setattr(T, "ind_max_pool", lambda x, inds: x[inds.long()].amax(1))
    monkeypatch.setattr(T, "closest_pool", lambda x, inds: x[inds[:, 0].long()])
    monkeypatch.setattr(T, "gather_rows", lambda x, inds: x[inds.long()])
    monkeypatch.setattr(T, "l2_normalize", lambda x: x / x.norm(dim=1, keepdim=True).clamp_min(1e-6))
    monkeypatch.setattr(T, "detection_scores", lambda x, nb, lens: x.sigmoid().amax(1, keepdim=True))

    cfg = synth.Config(**dict(T.TRAINING_3DMATCH, weights_decay=0.0, first_features_dim=8))
    n = [40, 20, 10, 6, 4]
    z = lambda *sh: torch.zeros(sh, dtype=torch.int32)
    inputs = dict(points=[torch.zeros(m, 3) for m in n], neighbors=[z(m, 4) for m in n],
                  pools=[z(n[i + 1], 4) for i in range(4)], upsamples=[z(n[i], 4) for i in range(4)],
                  lengths=[torch.tensor([m // 2, m - m // 2], dtype=torch.int32) for m in n],
                  features=torch.ones(n[0], 1))
    store = V.ParamStore(synth.make_params(cfg, seed=0), "cpu")
    params = T.trainable(store)
    anc = torch.arange(256, dtype=torch.int32) % 20
    rec = rp.Recorder()
    with rec.patched(), V.use_params(store):
        desc, scores = T.forward(inputs, cfg)
        loss = T.d3feat_loss(desc, scores, anc, anc + 20, torch.rand(n[0], 3), cfg)[0]
    assert T.batch_norm is bn and co.KPConv_ops is kpconv          # restored
    loss.backward()
    want = rp.expected_calls(cfg)
    assert want == dict(kpconv=10, kpconv_strided=4, unary=28, bn=37, pool=4, gather=8, l2=1, det=1)
    assert rp.counts(rec.calls) == want
    for r in rec.calls:
        assert r["grad_out"] is not None and r["grad_out"].shape == r["out"].shape, (r["kind"], r["index"])
    used = [id(p) for r in rec.calls for p, _ in rp.param_grads(r, dict(dW=0, dgamma=0, dbeta=0))]
    assert sorted(used) == sorted(set(used)) and set(used) == {id(p) for p in params}
