"""GPU: the training graph (d3feat_b200/training.py) against its float64 restatement (tests/_training_oracle.py).

  * every new op's output and gradient element by element within TOL = 1e-5 x that element's magnitude of the
    explicit float64 adjoints (_training_oracle: batch_norm_train_grads, ind_max_pool_grad, ...; _oracle.assert_close),
    batch norm's batch statistics and moving statistics too: batch norm with and without residual / LeakyReLU, the
    offset form, N = 1 and N = 0, N at the 2048-row partial blocks x C around the 32-column tiles, columns with
    |mean| >> std; the max pool with ties, duplicate indices, shadow and -1 entries, an all-equal column, and shadow
    entry counts at the 2048-entry partials; the row gather with repeats and one row gathered 1e5 times;
    l2_normalize with rows below eps; detection scores with B = 1, 2, 5, rows of no cloud, a cloud of 7000 rows, a
    cloud maximum tied across rows, and no neighbour columns;
  * the whole rigid network plus the loss on a seeded two-fragment batch: every parameter gradient within 3e-3 x its
    magnitude (TOL_NET says why not 1e-4), after checking that the seed's global decisions (cloud maxima, keypoint
    channel maxima, closest negatives) are far wider than the fp32 forward error;
  * gradients bitwise identical over two calls and two streams; loss.backward() equal bit for bit to the direct
    entry points; twenty SGD steps lower the loss; the trained store round-trips through a checkpoint and the
    inference KPFCNN then equals EncoderOracle with the trained moving statistics.
"""
import numpy as np
import pytest
import torch

import _training_oracle as ot
from _oracle import TOL, assert_close
from oracle import kpconv_np as ok

pytestmark = pytest.mark.gpu

TOL_OP = 1e-5
# The network's fp32 forward is within ~3e-6 x mag of float64, but the seed (like any real batch) has LeakyReLU inputs
# and max-pool gaps closer to their switch than that (some within 1e-7): fp32 and float64 take the other branch there,
# which moves those elements' gradients by O(1). Observed on an H100: at most 1.3e-3 x mag (layer_0/resnetb_1, whose
# output feeds the first max pool, the one with the narrowest gaps); 1e-4 was the proposal.
TOL_NET = 3e-3
LIMITS = [34, 34, 34, 34, 34]
WORST = {}


def g(a, dev, dt=torch.float32):
    return torch.as_tensor(np.ascontiguousarray(a)).to(device=dev, dtype=dt)


def close(what, got, ref, tol, m=None):
    """max |got - ref| <= tol * m, m = the largest |ref| unless given (the rounding scale of the computation)."""
    got = np.asarray(got.detach().cpu().numpy() if torch.is_tensor(got) else got, np.float64)
    ref = ref.detach().numpy() if torch.is_tensor(ref) else np.asarray(ref, np.float64)
    assert got.shape == ref.shape, (what, got.shape, ref.shape)
    if m is None:
        m = max(np.abs(ref).max(), 1e-30) if ref.size else 1.0
    err = float(np.abs(got - ref).max() / m) if ref.size else 0.0
    WORST[what] = max(WORST.get(what, 0.0), err)
    assert err <= tol, "%s: error %.3g x mag > %g" % (what, err, tol)


def grads_of(fn_gpu, xs, dev, gout_seed=0):
    """fn's output and input gradients on the GPU (float32 inputs, as numpy) for one seeded output gradient, which is
    returned too: (out, [dx...], gout)."""
    xg = [g(np.asarray(x, np.float32), dev).requires_grad_(True) for x in xs]
    y = fn_gpu(*xg)
    go = np.random.default_rng(gout_seed).normal(size=tuple(y.shape)).astype(np.float32)
    y.backward(g(go, dev))
    return y.detach().cpu().numpy(), [a.grad.cpu().numpy() for a in xg], go


# ---------------------------------------------------------------------------------------------------- ops
# Every op's output and gradients element by element against the explicit float64 adjoints of _training_oracle
# (ref, mag): |gpu - ref| <= TOL * mag (tests/_oracle.py).

def check_batch_norm(dev, x, res, alpha, seed=0, what="bn"):
    from d3feat_b200 import training as T
    N, C = x.shape
    rng = np.random.default_rng(seed)
    x = np.float32(x)
    gm, bt = np.float32(rng.uniform(0.5, 1.5, C)), np.float32(rng.normal(size=C) * 0.1)
    r = np.float32(rng.normal(size=(N, C))) if res else None
    mm, mv = np.float32(rng.normal(size=C) * 0.1), np.float32(rng.uniform(0.5, 1.5, C))
    mmg, mvg = g(mm, dev), g(mv, dev)

    def gpu(x, gm, bt, *r):
        return T._BatchNormFn.apply(x, gm, bt, r[0] if r else None, mmg, mvg, 0.98, alpha)

    out, grads, go = grads_of(gpu, [x, gm, bt] + ([r] if res else []), dev, seed)
    fw = ot.batch_norm_train_forward_ref(x, gm, bt, r, alpha, mm, mv, float(np.float32(1 - 0.98)))
    assert_close(out, *fw["out"], what=what + " out")
    assert_close(mmg.cpu(), *fw["moving_mean"], what=what + " moving_mean")
    assert_close(mvg.cpu(), *fw["moving_var"], what=what + " moving_var")
    # the batch statistics the backward reads (the forward is deterministic: the same bits as the step's)
    _, mean, invstd = T.batch_norm_forward(g(x, dev), g(gm, dev), g(bt, dev), g(mm, dev), g(mv, dev), 0.98)
    mean, invstd = mean.cpu().numpy(), invstd.cpu().numpy()
    assert_close(mean, *fw["mean"], what=what + " mean")
    assert_close(invstd, *fw["invstd"], what=what + " invstd")
    bw = ot.batch_norm_train_grads(x, out, go, gm, alpha, mean=mean, invstd=invstd)
    for n, got in zip(["dx", "dgamma", "dbeta", "dres"], grads):
        assert_close(got, *bw[n], what=what + " " + n)


@pytest.mark.parametrize("N,C,res,alpha", [(5000, 64, False, 0.2), (3000, 128, True, 0.2), (2100, 32, True, None),
                                           (1, 16, False, 0.2), (4097, 3, False, None)])
def test_batch_norm(cuda, N, C, res, alpha):
    rng = np.random.default_rng(N + C)
    x = rng.normal(size=(N, C)) * rng.uniform(0.5, 3, C) + rng.normal(size=C)
    check_batch_norm(cuda, x, res, alpha, N + C)


@pytest.mark.parametrize("N", [2047, 2048, 2049, 3 * 2048 + 1])
@pytest.mark.parametrize("C", [1, 31, 33, 256])
def test_batch_norm_block_boundaries(cuda, N, C):
    """N at the 2048-row blocks of colsum_partial_kernel's partials, C around its 32-column tiles."""
    rng = np.random.default_rng(N * 7 + C)
    x = rng.normal(size=(N, C)) * rng.uniform(0.5, 3, C) + rng.normal(size=C)
    check_batch_norm(cuda, x, (N + C) % 2 == 1, 0.2 if C != 33 else None, N + C, "bn %dx%d" % (N, C))


@pytest.mark.parametrize("N,C", [(6145, 64), (2049, 33)])
def test_batch_norm_mean_far_above_std(cuda, N, C):
    """x = 1e3 + N(0, 1): x - mean cancels 10 bits; the variance, xhat and dx must not lose them. The output gradient
    is the centred x itself (the same draws), so dgamma / N is of order one and xhat's error reaches dx."""
    rng = np.random.default_rng(N)
    check_batch_norm(cuda, 1e3 + rng.normal(size=(N, C)), True, 0.2, N, "bn mean>>std %dx%d" % (N, C))


def test_batch_norm_offset_and_empty(cuda):
    from d3feat_b200 import training as T
    rng = np.random.default_rng(3)
    x, off, r = (np.float32(a) for a in (rng.normal(size=(700, 24)), rng.normal(size=24), rng.normal(size=(700, 24))))
    out, grads, go = grads_of(lambda x, o, r: T._BatchNormFn.apply(x, None, o, r, None, None, 0.98, 0.2), [x, off, r],
                              cuda)
    assert_close(out, *ot.batch_norm_train_forward_ref(x, None, off, r, 0.2)["out"], what="offset out")
    bw = ot.batch_norm_train_grads(x, out, go, None, 0.2)
    for n, got in zip(["dx", "dbeta", "dres"], grads):
        assert_close(got, *bw[n], what="offset " + n)
    # N = 0: empty output, moving statistics untouched, zero dgamma / dbeta
    mm, mv = torch.full((8,), 0.5, device=cuda), torch.full((8,), 2.0, device=cuda)
    gm = torch.ones(8, device=cuda, requires_grad=True)
    bt = torch.zeros(8, device=cuda, requires_grad=True)
    x0 = torch.zeros((0, 8), device=cuda, requires_grad=True)
    y = T._BatchNormFn.apply(x0, gm, bt, None, mm, mv, 0.98, 0.2)
    assert y.shape == (0, 8)
    y.sum().backward()
    assert torch.equal(mm, torch.full_like(mm, 0.5)) and torch.equal(mv, torch.full_like(mv, 2.0))
    assert torch.equal(gm.grad, torch.zeros_like(gm)) and torch.equal(bt.grad, torch.zeros_like(bt))


def pool_case(rng, N1=900, N2=400, H=12, C=40):
    x = rng.normal(size=(N1, C)).astype(np.float32)
    x[:, 3] = 1.25                                             # an all-equal column: every pooled entry ties
    x[::7, 5] = x[:, 5].min()                                  # several rows at the column minimum
    inds = rng.integers(0, N1, size=(N2, H)).astype(np.int32)
    inds[:, -2:] = N1                                          # shadow entries in every row
    inds[::5, -3] = -1
    inds[::3, 1] = inds[::3, 0]                                # a duplicated index in a row
    inds[::11, :] = N1                                         # rows with no real neighbour: the column minimum
    return x, inds


def check_pool(dev, x, inds, what):
    from d3feat_b200 import training as T
    ig = g(inds, dev, torch.int32)
    out, (dx,), go = grads_of(lambda x: T._MaxPoolFn.apply(x, ig), [x], dev)
    assert np.array_equal(out, ot.ind_max_pool(ot.t64(x), inds).numpy())      # a selection: exact
    assert_close(dx, *ot.ind_max_pool_grad(x, inds, go), what=what)


@pytest.mark.parametrize("seed", [0, 1])
def test_ind_max_pool(cuda, seed):
    x, inds = pool_case(np.random.default_rng(seed))
    check_pool(cuda, x, inds, "pool dx seed %d" % seed)


@pytest.mark.parametrize("N2,H,n_shadow", [(91, 45, 2047), (91, 45, 2049), (128, 16, 2048), (241, 17, 4097),
                                           (683, 3, 2049)])
def test_ind_max_pool_shadow_blocks(cuda, N2, H, n_shadow):
    """N2*H (4095, 4097, 2048, 2049) and the number of shadow entries just below, at and above multiples of 2048:
    shadow_partial_kernel sums the shadow's gradient in 2048-entry partials. The all-shadow rows come last, so the
    last partial holds gradient the column minimum must receive."""
    rng = np.random.default_rng(N2 + H + n_shadow)
    N1, C = 700, 36
    x = rng.normal(size=(N1, C)).astype(np.float32)
    x[::9, 2] = x[:, 2].min()
    inds = rng.integers(0, N1, size=(N2, H)).astype(np.int32)
    full, extra = divmod(min(n_shadow, N2 * H), H)
    flat = inds.reshape(-1)
    flat[N2 * H - full * H:] = N1                              # the last `full` rows: shadow only
    head = N2 * H - full * H
    if extra:
        pick = rng.choice(head, extra, replace=False)
        flat[pick] = np.where(pick % 2 == 0, N1, -1)           # the rest of the shadow entries, some of them -1
    assert int(((inds < 0) | (inds >= N1)).sum()) == min(n_shadow, N2 * H)
    check_pool(cuda, x, inds, "pool shadow %dx%d/%d" % (N2, H, n_shadow))


def test_gather_rows(cuda):
    from d3feat_b200 import training as T
    rng = np.random.default_rng(5)
    x = rng.normal(size=(3000, 33))
    inds = rng.integers(0, 3000, size=5000).astype(np.int32)
    inds[::9] = 3000                                           # shadow: zero row, gradient dropped
    inds[:300] = 17                                            # one row gathered 300 times
    ig = g(inds, cuda, torch.int32)
    out, (dx,), go = grads_of(lambda x: T._GatherFn.apply(x, ig), [x], cuda)
    assert np.array_equal(out, ot.gather_rows(ot.t64(np.float32(x)), inds).numpy())
    assert_close(dx, *ot.gather_rows_grad(inds, go, 3000), what="gather dx")


def test_gather_one_row_1e5_times(cuda):
    from d3feat_b200 import training as T
    rng = np.random.default_rng(15)
    x = rng.normal(size=(500, 32))
    inds = rng.integers(0, 500, size=120000).astype(np.int32)
    inds[rng.choice(120000, 100000, replace=False)] = 42       # row 42 gathered 1e5 times, interleaved
    ig = g(inds, cuda, torch.int32)
    _, (dx,), go = grads_of(lambda x: T.gather_rows(x, ig), [x], cuda)
    assert_close(dx, *ot.gather_rows_grad(inds, go, 500), what="gather 1e5 repeats dx")


def test_l2_normalize(cuda):
    from d3feat_b200 import training as T
    rng = np.random.default_rng(6)
    x = rng.normal(size=(4000, 32))
    x[::13] *= 1e-7                                            # sum x^2 below eps = 1e-10
    out, (dx,), go = grads_of(T.l2_normalize, [x], cuda)
    xf = np.float32(x)
    assert_close(out, ot.l2_normalize(ot.t64(xf)).numpy(), np.abs(ot.l2_normalize(ot.t64(np.abs(xf))).numpy()),
                 what="l2 out")
    assert_close(dx, *ot.l2_normalize_grad(xf, go), what="l2 dx")


def det_case(rng, lengths, N, H=20, D=32):
    x = rng.normal(size=(N, D)) + 0.3
    x[::17, :] = 0.0                                           # zero rows: no count_nonzero vote
    nb = rng.integers(0, N, size=(N, H)).astype(np.int32)
    start = np.concatenate([[0], np.cumsum(lengths)])
    for b in range(len(lengths)):                              # neighbours within the row's own cloud
        a, e = start[b], min(start[b + 1], N)
        if e > a:
            nb[a:e] = rng.integers(a, e, size=(e - a, H))
    nb[:, -3:] = N                                             # shadow
    return x, nb


def check_det(dev, x, nb, lengths, what):
    from d3feat_b200 import training as T
    N = x.shape[0]
    nbg, lg = g(nb, dev, torch.int32), g(np.asarray(lengths, np.int32), dev, torch.int32)
    out, (dx,), go = grads_of(lambda x: T.detection_scores(x, nbg, lg), [x], dev)
    xf = np.float32(x)
    rows = min(N, sum(lengths))                                # rows past the last cloud: unspecified score
    ref = ot.detection_scores(ot.t64(xf), nb, lengths).numpy()
    assert np.all(np.abs(out[:rows] - ref[:rows]) <= TOL * np.abs(ref[:rows]).max())
    ref, mag, alt, amb = ot.detection_scores_grad(xf, nb, lengths, go)
    print("%s: %d of %d rows checked against both channels" % (what, int(amb.sum()), N))
    assert amb.sum() <= max(1, 1e-3 * N)
    assert_close(dx, ref, mag, what=what, alt=alt)


@pytest.mark.parametrize("lengths,N", [([2500], 2500), ([1200, 1300], 2500), ([500, 700, 0, 900, 300], 2600)])
def test_detection_scores(cuda, lengths, N):
    x, nb = det_case(np.random.default_rng(len(lengths)), lengths, N)
    check_det(cuda, x, nb, lengths, "det dx B=%d" % len(lengths))


def test_detection_scores_large_cloud_and_tied_maximum(cuda):
    """A 7000-row cloud (det_cloud_grad_kernel sums its dL/dinv in 2048-row chunks) next to a 2100-row one, each
    with its maximum tied across several rows."""
    lengths = [7000, 2100]
    rng = np.random.default_rng(21)
    x, nb = det_case(rng, lengths, sum(lengths))
    for a, e, rows in ((0, 7000, [5, 2048, 4097, 6999]), (7000, 9100, [7001, 9099])):
        m = x[a:e].max() + 0.5
        for i, r in enumerate(rows):
            x[r, i % 32] = m
    check_det(cuda, x, nb, lengths, "det dx large cloud, tied max")


def test_detection_scores_no_neighbours(cuda):
    """H = 0: every mean is zero (count clamped to 1), nothing is scattered."""
    lengths = [1500, 1100]
    x, _ = det_case(np.random.default_rng(22), lengths, 2600)
    check_det(cuda, x, np.zeros((2600, 0), np.int32), lengths, "det dx H=0")


# ---------------------------------------------------------------------------------------------------- network

def pair(seed=0, n=1500, k=256):
    from d3feat_b200 import synth
    a = synth.room_fragment(seed, n)
    th = 0.3
    R = np.array([[np.cos(th), -np.sin(th), 0], [np.sin(th), np.cos(th), 0], [0, 0, 1]])
    b = (a @ R.T + np.array([0.5, -0.2, 0.1])).astype(np.float32)
    rng = np.random.default_rng(seed)
    anc = rng.choice(n, k, replace=True).astype(np.int32)
    return np.concatenate([a, b]), np.array([n, n], np.int32), anc, (anc + n).astype(np.int32)


def config():
    from d3feat_b200 import synth, training as T
    return synth.Config(**T.TRAINING_3DMATCH)


def gpu_step(dev, cfg, params, pts, lens, anc, pos, stream=None):
    """One forward + loss + backward on a fresh store: (store, outputs, {name: grad})."""
    from d3feat_b200 import training as T
    from d3feat_b200.encoder import KPFCNN
    from d3feat_b200.variables import ParamStore, use_params
    store = ParamStore(params, dev)
    enc = KPFCNN(cfg, store, LIMITS, device=dev)
    with torch.cuda.stream(stream or torch.cuda.current_stream()):
        inputs = enc.build_inputs(pts, lens)
        T.trainable(store)
        with use_params(store):
            desc, scores = T.forward(inputs, cfg)
            out = T.d3feat_loss(desc, scores, g(anc, dev, torch.int32), g(pos, dev, torch.int32), inputs["points"][0],
                                cfg)
        out[0].backward()
    torch.cuda.synchronize()
    grads = {n: t.grad.clone() for n, t in store.t.items() if t.grad is not None}
    return store, inputs, (desc, scores) + tuple(out), grads


def host_inputs(inputs):
    return {k: [t.cpu().numpy() for t in v] if isinstance(v, list) else v.cpu().numpy()
            for k, v in inputs.items() if k in ("points", "neighbors", "pools", "upsamples", "lengths", "features")}


@pytest.fixture(scope="module")
def net_run(cuda):
    from d3feat_b200 import synth
    cfg = config()
    params = synth.make_params(cfg, seed=0)
    pts, lens, anc, pos = pair()
    store, inputs, outs, grads = gpu_step(cuda, cfg, params, pts, lens, anc, pos)
    hi = host_inputs(inputs)
    p64 = {k: ot.t64(v).requires_grad_(k.rsplit("/", 1)[-1] in ("weights", "gamma", "beta", "offset"))
           for k, v in params.items()}
    net = ot.Network(cfg, p64)
    d, s = net.forward(hi)
    ref = ot.d3feat_loss(d, s, anc, pos, hi["points"][0], cfg, [p64[n] for n in sorted(p64) if "weights" in n],
                         net.decisions)
    ref[0].backward()
    return dict(cfg=cfg, params=params, pair=(pts, lens, anc, pos), store=store, outs=outs, grads=grads, net=net,
                p64=p64, ref=(d, s) + tuple(ref))


def test_network_decisions_are_wider_than_fp32_error(net_run):
    outs, ref, dec = net_run["outs"], net_run["ref"], net_run["net"].decisions
    fwd_err = max(float(np.abs(outs[i].detach().cpu().numpy() - ref[i].detach().numpy()).max() / ot.mag(ref[i]))
                  for i in (0, 1))
    print("forward error %.3g; margins: cloud max %s, keypoint score %.3g, closest negative %.3g, min sum x^2 %.3g" % (
        fwd_err, ["%.3g" % v for v in dec["cloud_max_gap"]], dec["keypoint_score_gap"], dec["closest_negative_gap"],
        dec["l2_sum_vs_eps"]))
    assert fwd_err < 1e-4
    for m in dec["cloud_max_gap"] + [dec["keypoint_score_gap"], dec["closest_negative_gap"]]:
        assert m > 100 * fwd_err
    assert dec["l2_sum_vs_eps"] > 1e-6


def test_network_gradients(net_run):
    outs, ref = net_run["outs"], net_run["ref"]
    for i, n in enumerate(["descriptors", "scores", "loss", "desc_loss", "det_loss", "accuracy", "d_pos", "d_neg"]):
        close("net " + n, outs[i], ref[i], TOL_NET)
    grads, p64 = net_run["grads"], net_run["p64"]
    assert set(grads) == {n for n, t in p64.items() if t.requires_grad}
    errs = {}
    for n, gr in sorted(grads.items()):
        ref = p64[n].grad.numpy()
        errs[n] = float(np.abs(gr.cpu().numpy() - ref).max() / max(np.abs(ref).max(), 1e-30))
    for n in sorted(errs, key=errs.get)[-8:]:
        print("gradient error %.3g x mag: %s" % (errs[n], n))
    for n, gr in sorted(grads.items()):
        close("net grad", gr, p64[n].grad, TOL_NET)
    store = net_run["store"]
    for n, t in p64.items():
        if "moving" in n:
            close("net moving statistics", store.get(n), t, TOL_OP * 10)


def test_gradients_are_deterministic_across_calls_and_streams(cuda, net_run):
    cfg, params = net_run["cfg"], net_run["params"]
    _, _, _, g1 = gpu_step(cuda, cfg, params, *net_run["pair"])
    _, _, _, g2 = gpu_step(cuda, cfg, params, *net_run["pair"], stream=torch.cuda.Stream(cuda))
    for n, gr in net_run["grads"].items():
        assert torch.equal(gr, g1[n]) and torch.equal(gr, g2[n]), n


def test_autograd_equals_direct_entry_points(cuda):
    from d3feat_b200 import training as T
    rng = np.random.default_rng(9)
    x, inds = pool_case(rng)
    xg, ig = g(x, cuda).requires_grad_(True), g(inds, cuda, torch.int32)
    out = T.ind_max_pool(xg, ig)
    go = g(rng.normal(size=out.shape), cuda)
    out.backward(go)
    assert torch.equal(xg.grad, T.ind_max_pool_backward(xg.detach(), ig, out.detach(), go))
    y = g(rng.normal(size=(500, 32)), cuda).requires_grad_(True)
    o = T.l2_normalize(y)
    go = g(rng.normal(size=o.shape), cuda)
    o.backward(go)
    assert torch.equal(y.grad, T.l2_normalize_backward(y.detach(), go))
    y.grad = None
    gi = g(rng.integers(0, 500, 700), cuda, torch.int32)
    o = T.gather_rows(y, gi)
    go = g(rng.normal(size=o.shape), cuda)
    o.backward(go)
    assert torch.equal(y.grad, T.gather_rows_backward(gi, go, 500))


def test_sgd_lowers_the_loss_and_the_trained_store_round_trips(cuda, net_run, tmp_path):
    from d3feat_b200 import synth, training as T, tf_checkpoint as ck
    from d3feat_b200.encoder import KPFCNN
    from d3feat_b200.variables import ParamStore, use_params
    cfg, (pts, lens, anc, pos) = net_run["cfg"], net_run["pair"]
    cfg.learning_rate = 1e-2
    store = ParamStore(net_run["params"], cuda)
    enc = KPFCNN(cfg, store, LIMITS, device=cuda)
    inputs = enc.build_inputs(pts, lens)
    params = T.trainable(store)
    opt = torch.optim.SGD(params, lr=cfg.learning_rate, momentum=cfg.momentum)
    ag, pg = g(anc, cuda, torch.int32), g(pos, cuda, torch.int32)
    losses = []
    for _ in range(20):
        with use_params(store):
            desc, scores = T.forward(inputs, cfg)
            loss = T.d3feat_loss(desc, scores, ag, pg, inputs["points"][0], cfg)[0]
        opt.zero_grad()
        loss.backward()
        for p in params:
            torch.nn.utils.clip_grad_norm_([p], cfg.grad_clip_norm)
        opt.step()
        losses.append(float(loss.detach()))
    print("loss over 20 SGD steps:", ["%.4f" % v for v in losses])
    assert losses[-1] < losses[0]
    # checkpoint round trip, then the inference network with the trained moving statistics
    prefix = str(tmp_path / "trained")
    ck.write_checkpoint(prefix, {ck.MODEL_SCOPE + n: t.detach().cpu().numpy() for n, t in store.t.items()})
    loaded = ck.load_params(prefix)
    assert set(loaded) == set(store.t)
    for n, t in store.t.items():
        assert np.array_equal(loaded[n], t.detach().cpu().numpy()), n
    cfg_enc = synth.Config(**T.TRAINING_3DMATCH)
    inf = KPFCNN(cfg_enc, loaded, LIMITS, device=cuda)
    with torch.no_grad():
        out = inf(pts, lens, decoder=False)
    hi = host_inputs(out["inputs"])
    F_ref = ok.EncoderOracle(cfg_enc, loaded, np.float64).encoder(hi)
    for a, b in zip(out["F"], F_ref):
        close("trained encoder", a, b, 1e-4)


def teardown_module():
    print("\nlargest error per check (x mag):", ", ".join("%s %.3g" % kv for kv in sorted(WORST.items())))
