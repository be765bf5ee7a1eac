"""CPU: the float64 restatement of the training graph (tests/_training_oracle.py) and the argument checks of
d3feat_b200/training.py.

  * each restated op's autograd gradient against central differences (torch.autograd.gradcheck) on inputs without
    ties: batch norm with N = 1 and 5, with residual and LeakyReLU, the offset form; the max pool with shadow and -1
    entries; the row gather with repeats; l2_normalize with a row below eps; detection scores with B = 1, 2 and 5 and
    rows of no cloud;
  * at ties, the max pool's gradient against a hand-written adjoint of TF's rule (reduce_max splits evenly over the
    tied entries, the shadow's shares go through reduce_min to the rows at the column minimum), with duplicate indices,
    all-shadow rows and an all-equal column, and against central differences along tie-preserving directions;
  * the restated network with inference batch norm equals oracle/kpconv_np's EncoderOracle, decoder and detection
    scores;
  * with the library replaced by a stub, the direct entry points refuse wrong dtypes, devices and shapes, and
    training.forward refuses static inputs and deformable blocks, before anything reaches the library.
"""
import numpy as np
import pytest
import torch

import _training_oracle as ot
from oracle import kpconv_np as ok

D = torch.float64


def gradcheck(fn, *xs):
    xs = [ot.t64(x).requires_grad_(True) for x in xs]
    assert torch.autograd.gradcheck(fn, xs, eps=1e-6, atol=1e-6, rtol=1e-5)


@pytest.mark.parametrize("N,res,alpha", [(5, False, 0.2), (5, True, 0.2), (7, True, None), (1, False, 0.2)])
def test_batch_norm_central_differences(N, res, alpha):
    rng = np.random.default_rng(N)
    x = rng.normal(size=(N, 4)) * 2 + 0.5
    args = [x, rng.uniform(0.5, 1.5, 4), rng.normal(size=4)] + ([rng.normal(size=(N, 4))] if res else [])
    gradcheck(lambda x, g, b, *r: ot.batch_norm_train(x, g, b, r[0] if r else None, alpha)[0], *args)
    gradcheck(lambda x, b, *r: ot.batch_norm_train(x, None, b, r[0] if r else None, alpha)[0], *(args[:1] + args[2:]))


def test_batch_norm_one_and_no_rows():
    x = ot.t64(np.array([[1.5, -2.0, 0.25]])).requires_grad_(True)
    g, b = ot.t64([1.2, 0.7, 1.0]).requires_grad_(True), ot.t64([0.1, -0.3, 0.0]).requires_grad_(True)
    y, mean, var = ot.batch_norm_train(x, g, b)
    assert torch.allclose(y.detach(), b.detach()[None], atol=1e-12) and torch.equal(var, torch.zeros(3, dtype=D))
    y.sum().backward()
    assert torch.allclose(x.grad, torch.zeros_like(x), atol=1e-9) and torch.equal(g.grad, torch.zeros(3, dtype=D))
    assert torch.equal(b.grad, torch.ones(3, dtype=D))
    y0, m0, v0 = ot.batch_norm_train(torch.zeros((0, 3), dtype=D), g, b)
    assert y0.shape == (0, 3) and m0 is None and v0 is None


def test_pool_gather_l2_central_differences():
    rng = np.random.default_rng(1)
    x = rng.normal(size=(9, 3))
    inds = rng.integers(0, 9, size=(6, 4))
    inds[:, -1] = 9
    inds[2, 0] = -1
    gradcheck(lambda x: ot.ind_max_pool(x, inds), x)
    gi = np.array([3, 3, 0, 9, 8, 3, -1])
    gradcheck(lambda x: ot.gather_rows(x, gi), x)
    y = rng.normal(size=(5, 6))
    y[2] *= 1e-7                                   # sum x^2 < 1e-10
    gradcheck(ot.l2_normalize, y)


@pytest.mark.parametrize("lengths,N", [([12], 12), ([5, 7], 12), ([3, 2, 0, 4, 2], 14)])
def test_detection_central_differences(lengths, N):
    rng = np.random.default_rng(N + len(lengths))
    x = rng.normal(size=(N, 5)) + 0.2
    nb = rng.integers(0, N, size=(N, 4))
    nb[:, -1] = N
    gradcheck(lambda x: ot.detection_scores(x, nb, lengths), x)


def pool_adjoint(x, inds, g):
    """Hand-written adjoint of reduce_max(gather(x || reduce_min(x), inds)) with TF's even tie splits."""
    N1, C = x.shape
    cmin = x.min(0)
    xs = np.concatenate([x, cmin[None]], 0)
    ii = np.where((inds < 0) | (inds >= N1), N1, inds)
    v = xs[ii]                                     # [N2, H, C]
    out = v.max(1)
    tie = v == out[:, None, :]
    share = g / tie.sum(1)
    dxs = np.zeros_like(xs)
    for q in range(inds.shape[0]):
        for h in range(inds.shape[1]):
            dxs[ii[q, h]] += np.where(tie[q, h], share[q], 0.0)
    at_min = x == cmin[None]
    return dxs[:N1] + at_min * (dxs[N1] / at_min.sum(0))[None]


def test_pool_ties_split_evenly():
    rng = np.random.default_rng(2)
    x = rng.normal(size=(10, 4))
    x[:, 1] = 0.75                                 # all-equal column
    x[[2, 6], 2] = x[:, 2].min() - 1               # two rows at the column minimum
    inds = rng.integers(0, 10, size=(7, 5))
    inds[:, 1] = inds[:, 0]                        # duplicate index
    inds[:, -1] = 10
    inds[3] = 10                                   # a row of shadows only
    inds[4, 2] = -1
    g = rng.normal(size=(7, 4))
    xt = ot.t64(x).requires_grad_(True)
    ot.ind_max_pool(xt, inds).backward(ot.t64(g))
    want = pool_adjoint(x, inds, g)
    assert np.allclose(xt.grad.numpy(), want, rtol=1e-13, atol=1e-13)
    # central differences along directions that keep every tie (shift whole columns): the sum of the shares
    for c in range(4):
        d = np.zeros_like(x)
        d[:, c] = 1.0
        f = lambda t: float((ot.ind_max_pool(ot.t64(x + t * d), inds) * ot.t64(g)).sum())
        fd = (f(1e-6) - f(-1e-6)) / 2e-6
        assert abs(fd - float((want * d).sum())) < 1e-6 * max(1.0, abs(fd))


def small_pyramid(cfg, n=(1200, 1000)):
    from d3feat_b200 import synth
    from oracle import native as on
    pts = np.concatenate([synth.room_fragment(i, m) for i, m in enumerate(n)], 0)
    lens = np.array(n, np.int32)
    inputs = ok.descriptor_input_pyramid(cfg, pts, lens, [30] * cfg.num_layers, on.port_batch_neighbors,
                                         on.port_batch_subsampling)
    inputs["features"] = np.ones((pts.shape[0], 1), np.float32)
    return inputs


def test_inference_graph_equals_the_encoder_oracle():
    from d3feat_b200 import synth
    cfg = synth.Config(first_features_dim=16)
    params = synth.make_params(cfg, seed=3)
    inputs = small_pyramid(cfg)
    net = ot.Network(cfg, {k: ot.t64(v) for k, v in params.items()}, inference=True)
    with torch.no_grad():
        desc, scores = net.forward(inputs)
    ref = ok.EncoderOracle(cfg, params, np.float64)
    F = ref.encoder(inputs)
    want_desc, want_scores = ref.decoder(inputs, F, return_scores=True)
    assert np.allclose(desc.numpy(), want_desc, rtol=1e-10, atol=1e-12)
    assert np.allclose(scores.numpy(), want_scores, rtol=1e-10, atol=1e-12)


class Stub:
    def __getattr__(self, symbol):
        raise AssertionError("reached the library: %s" % symbol)


@pytest.fixture
def host(monkeypatch):
    from d3feat_b200 import _lib
    monkeypatch.setattr(_lib, "DEVICE_TYPE", "cpu")
    monkeypatch.setattr(_lib, "lib", lambda: Stub())


z = torch.zeros
WRONG = [
    ("dtype", lambda sh: z(sh, dtype=torch.float64)),
    ("shape", lambda sh: z((sh[0] + 1,) + tuple(sh[1:]))),
    ("device", lambda sh: z(sh, device="meta")),
]


@pytest.mark.parametrize("case", [c for c, _ in WRONG])
def test_entry_points_refuse_bad_arguments(host, case):
    from d3feat_b200 import training as T
    bad = dict(WRONG)[case]
    i32 = lambda *sh: z(sh, dtype=torch.int32)
    calls = [
        ("batch_norm_backward: grad_out", lambda: T.batch_norm_backward(z(6, 4), z(6, 4), bad((6, 4)), z(4), z(4), z(4))),
        ("batch_norm_forward: residual", lambda: T.batch_norm_forward(z(6, 4), z(4), z(4), z(4), z(4), 0.98, bad((6, 4)))),
        ("ind_max_pool_backward: grad_out", lambda: T.ind_max_pool_backward(z(6, 4), i32(3, 2), z(3, 4), bad((3, 4)))),
        ("gather_rows_backward: grad_out", lambda: T.gather_rows_backward(i32(3), bad((3, 4)), 6)),
        ("l2_normalize_backward: grad_out", lambda: T.l2_normalize_backward(z(6, 4), bad((6, 4)))),
        ("detection_scores_backward: grad_scores",
         lambda: T.detection_scores_backward(z(6, 4), i32(6, 3), i32(2), bad((6, 1)))),
    ]
    for what, call in calls:
        with pytest.raises(ValueError, match=what):
            call()


def test_legal_calls_reach_the_library(host):
    from d3feat_b200 import training as T
    i32 = lambda *sh: z(sh, dtype=torch.int32)
    for call in (lambda: T.batch_norm_backward(z(6, 4), z(6, 4), z(6, 4), z(4), z(4), z(4)),
                 lambda: T.ind_max_pool_backward(z(6, 4), i32(3, 2), z(3, 4), z(3, 4)),
                 lambda: T.gather_rows_backward(i32(3), z(3, 4), 6),
                 lambda: T.l2_normalize_backward(z(6, 4), z(6, 4)),
                 lambda: T.detection_scores_backward(z(6, 4), i32(6, 3), i32(2), z(6, 1))):
        with pytest.raises(AssertionError, match="reached the library"):
            call()


def test_forward_refuses_static_inputs_and_deformable_blocks(host):
    from d3feat_b200 import synth, training as T
    cfg = synth.Config()
    with pytest.raises(ValueError, match="static"):
        T.forward({"rows": [z(1, dtype=torch.int32)], "features": z(3, 1)}, cfg)
    cfg = synth.Config(architecture=synth.ARCH_KITTI_DEFORM)
    with pytest.raises(NotImplementedError, match="deformable"):
        T.forward({"features": z(3, 1)}, cfg)


def test_trainable_marks_weights_and_affines_only():
    from d3feat_b200 import synth, training as T
    from d3feat_b200.variables import ParamStore
    cfg = synth.Config(architecture=synth.ARCH_ENCODER[:4], first_features_dim=8)
    store = ParamStore(synth.make_params(cfg, seed=0), "cpu")
    params = T.trainable(store)
    names = {n for n, t in store.t.items() if t.requires_grad}
    assert len(params) == len(names) > 0
    assert all(n.rsplit("/", 1)[-1] in ("weights", "gamma", "beta", "offset") for n in names)
    assert not any(t.requires_grad for n, t in store.t.items() if "moving" in n or "kernel_points" in n)
