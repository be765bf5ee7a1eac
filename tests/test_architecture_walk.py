"""The architecture walk (network_blocks.architecture) on the CPU: the inference blocks, the training blocks and the
seeded parameters (synth.make_params) name and size every variable alike.

The library is stubbed (any launch fails the test) and the convolutions, pools, normalisations and detection scores are
replaced by shape-only fakes that check their operands agree. The parameter store records every name looked up, and
weight_variable every shape a block asks for. Run through assemble_FCNN_blocks / assemble_CNN_blocks and
training.forward, the names looked up must be exactly those make_params creates (which test_checkpoint_io.py compares
with the released checkpoints) and the shapes asked for must be theirs."""
import pytest
import torch


class Stub:
    def __getattr__(self, symbol):
        raise AssertionError("reached the library: %s" % symbol)


class Recorder(dict):
    """The store's tensors; every name read is recorded in order."""

    def __init__(self, t):
        super().__init__(t)
        self.read = []

    def __getitem__(self, name):
        self.read.append(name)
        return super().__getitem__(name)


def _rows(n, c, *like):
    return torch.zeros((int(n), int(c)), requires_grad=any(t is not None and t.requires_grad for t in like))


def _check_affine(affine, c):
    if affine is not None:
        assert tuple(affine[0].shape) == tuple(affine[1].shape) == (c,)


@pytest.fixture
def fakes(monkeypatch):
    """Stub the library and replace every op the blocks reach with a shape-only fake; yields the {weights name: shape}
    the blocks asked weight_variable for."""
    from d3feat_b200 import _lib, convolution_ops as co, network_blocks as nb, training as T, variables as V
    monkeypatch.setattr(_lib, "DEVICE_TYPE", "cpu")
    monkeypatch.setattr(_lib, "lib", lambda: Stub())
    asked = {}
    weight_variable = nb.weight_variable

    def weights(shape):
        asked[V.scoped("weights")] = tuple(int(s) for s in shape)
        return weight_variable(shape)

    def kpconv(q, s, idx, f, Kp, W, extent, influence, mode, *, epilogue=None, bias=None, **kw):
        K, cin, cout = W.shape
        assert f.shape[1] == cin and s.shape[0] == f.shape[0] and idx.shape[0] == q.shape[0]
        assert tuple(Kp.shape) == (K, 3)
        _check_affine(epilogue, cout)
        assert bias is None or tuple(bias.shape) == (cout,)
        return _rows(q.shape[0], cout, f, W)

    def kpconv_deform(q, s, idx, f, Kp, off, mod, W, extent, influence, mode, *, epilogue=None, **kw):
        K, cin, cout = W.shape
        assert f.shape[1] == cin and tuple(off.shape) == (q.shape[0], K, 3)
        _check_affine(epilogue, cout)
        return _rows(q.shape[0], cout)

    def unary(x, w, *, epilogue=None, residual=None, rows=None):
        assert x.shape[1] == w.shape[0]
        _check_affine(epilogue, w.shape[1])
        assert residual is None or tuple(residual.shape) == (x.shape[0], w.shape[1])
        return _rows(x.shape[0], w.shape[1], x, w)

    def unary_pair(x1, w1, a1, x2, w2, a2, alpha, *, rows=None):
        assert x1.shape[1] == w1.shape[0] and x2.shape[1] == w2.shape[0] and w1.shape[1] == w2.shape[1]
        assert x1.shape[0] == x2.shape[0]
        _check_affine(a1, w1.shape[1])
        _check_affine(a2, w2.shape[1])
        return _rows(x1.shape[0], w1.shape[1])

    def pool(x, inds, **kw):
        return _rows(inds.shape[0], x.shape[1], x)

    def per_row(x, *args, **kw):
        return _rows(x.shape[0], 1, x)

    def same(x, *args, **kw):
        return _rows(x.shape[0], x.shape[1], x)

    def batch_norm_forward(x, gamma, beta, moving_mean, moving_var, momentum, residual=None, alpha=None):
        c = x.shape[1]
        assert all(t is None or tuple(t.shape) == (c,) for t in (gamma, beta, moving_mean, moving_var))
        assert residual is None or residual.shape == x.shape
        return torch.zeros_like(x), torch.zeros(c), torch.zeros(c)

    for m, name, fn in ((nb, "weight_variable", weights), (co, "KPConv_ops", kpconv),
                        (co, "KPConv_deform_ops", kpconv_deform), (co, "unary_convolution", unary),
                        (co, "unary_pair_convolution", unary_pair), (nb, "ind_max_pool", pool),
                        (nb, "closest_pool", pool), (nb, "detection_scores", per_row), (nb, "l2_normalize", same),
                        (nb, "_affine_leaky", same), (T, "batch_norm_forward", batch_norm_forward)):
        monkeypatch.setattr(m, name, fn)
    yield asked


def pyramid(cfg, n0=64):
    """Exact-shape inputs with the level sizes and index widths of a real pyramid (all indices 0)."""
    L = cfg.num_layers
    n = [n0 >> l for l in range(L)]
    i32 = lambda *sh: torch.zeros(sh, dtype=torch.int32)
    return dict(points=[torch.zeros(n[l], 3) for l in range(L)], neighbors=[i32(n[l], 7) for l in range(L)],
                pools=[i32(n[l + 1], 6) for l in range(L - 1)], upsamples=[i32(n[l], 4) for l in range(L - 1)],
                lengths=[i32(2) for _ in range(L)], features=torch.ones(n[0], cfg.in_features_dim))


def store_of(params):
    from d3feat_b200.variables import ParamStore
    store = ParamStore(params, "cpu")
    store.t = Recorder(store.t)
    return store


def config(arch, **kw):
    from d3feat_b200 import synth
    return synth.Config(architecture=list(arch), first_features_dim=8, **kw)


def archs():
    from d3feat_b200 import synth
    return dict(d3feat_3dmatch=synth.ARCH_3DMATCH, kitti_deformable=synth.ARCH_KITTI_DEFORM,
                kitti_deformable_decoder=synth.ARCH_KITTI_DEFORM + synth.ARCH_3DMATCH[10:],
                encoder=synth.ARCH_ENCODER)


def without_batch_norm(params):
    """The parameters of use_batch_norm = False: every batch norm replaced by its '<scope>/offset' bias."""
    out = {}
    for k, v in params.items():
        scope, sep, var = k.partition("/batch_normalization/")
        if not sep:
            out[k] = v
        elif var == "beta":
            out[scope + "/offset"] = v
    return out


def weight_shapes(params):
    return {k: tuple(v.shape) for k, v in params.items() if k.endswith("/weights")}


@pytest.mark.parametrize("batch_norm", [True, False], ids=["batch_norm", "offset"])
@pytest.mark.parametrize("name", ["d3feat_3dmatch", "kitti_deformable", "kitti_deformable_decoder", "encoder"])
def test_inference_looks_up_exactly_the_seeded_names(fakes, name, batch_norm):
    from d3feat_b200 import network_blocks as nb, synth
    from d3feat_b200.variables import use_params
    cfg = config(archs()[name], use_batch_norm=batch_norm)
    params = synth.make_params(cfg, seed=1)
    if not batch_norm:
        params = without_batch_norm(params)
    store, inputs = store_of(params), pyramid(cfg)
    has_decoder = any("upsample" in b for b in cfg.architecture)
    with use_params(store):
        if has_decoder:
            desc, scores = nb.assemble_FCNN_blocks(inputs, cfg)
            assert tuple(desc.shape) == (64, 32) and tuple(scores.shape) == (64, 1)
        else:
            F = nb.assemble_CNN_blocks(inputs, cfg, 1.0)
            assert [f.shape[0] for f in F] == [64 >> l for l in range(cfg.num_layers)]
            assert F[-1].shape[1] == 32 * cfg.first_features_dim      # 2 * fdim of layer 4
    assert set(store.t.read) == set(params)
    assert fakes == weight_shapes(params)


@pytest.mark.parametrize("batch_norm", [True, False], ids=["batch_norm", "offset"])
def test_training_looks_up_exactly_the_seeded_names(fakes, batch_norm):
    from d3feat_b200 import synth, training as T
    from d3feat_b200.variables import use_params
    cfg = config(synth.ARCH_3DMATCH, use_batch_norm=batch_norm)
    params = synth.make_params(cfg, seed=2)
    if not batch_norm:
        params = without_batch_norm(params)
    store = store_of(params)
    with use_params(store):
        desc, scores = T.forward(pyramid(cfg), cfg)
    assert tuple(desc.shape) == (64, 32) and tuple(scores.shape) == (64, 1)
    assert set(store.t.read) == set(params)
    assert fakes == weight_shapes(params)


def test_schedule_of_the_3dmatch_architecture():
    from d3feat_b200 import network_blocks as nb, synth
    cfg = synth.Config()
    encoder, decoder = nb.architecture(cfg)
    r0 = cfg.first_subsampling_dl * cfg.density_parameter
    assert [s.scope for s in encoder] == [
        "layer_0/simple_0", "layer_0/resnetb_1", "layer_0/resnetb_strided_2", "layer_1/resnetb_0",
        "layer_1/resnetb_strided_1", "layer_2/resnetb_0", "layer_2/resnetb_strided_1", "layer_3/resnetb_0",
        "layer_3/resnetb_strided_1", "layer_4/resnetb_0"]
    assert [(s.layer, s.fdim, s.skip) for s in encoder] == [
        (0, 64, False), (0, 64, False), (0, 64, True), (1, 128, False), (1, 128, True), (2, 256, False),
        (2, 256, True), (3, 512, False), (3, 512, True), (4, 1024, False)]
    assert [s.radius for s in encoder] == [r0 * 2 ** s.layer for s in encoder]
    assert [s.scope for s in decoder] == [
        "uplayer_4/nearest_upsample_0", "uplayer_3/unary_0", "uplayer_3/nearest_upsample_1", "uplayer_2/unary_0",
        "uplayer_2/nearest_upsample_1", "uplayer_1/unary_0", "uplayer_1/nearest_upsample_1", "uplayer_0/unary_0",
        "uplayer_0/last_unary_1"]
    assert [(s.fdim, s.concat) for s in decoder] == [
        (1024, True), (512, False), (512, True), (256, False), (256, True), (128, False), (128, True), (64, False),
        (64, False)]
    assert not any(s.skip for s in decoder) and not any(s.concat for s in encoder)
    assert [s.radius for s in decoder] == [r0 * 2 ** s.layer for s in decoder]
    kitti = nb.architecture(synth.Config(architecture=synth.ARCH_KITTI_DEFORM))
    assert [(s.block, s.scope) for s in kitti[0]][-3:] == [
        ("resnetb_deformable", "layer_3/resnetb_0"), ("resnetb_deformable_strided", "layer_3/resnetb_strided_1"),
        ("resnetb_deformable", "layer_4/resnetb_0")]
    assert kitti[1] == []


def test_an_architecture_without_decoder_is_refused_before_any_launch(fakes):
    from d3feat_b200 import network_blocks as nb, synth, training as T
    from d3feat_b200.variables import use_params
    cfg = config(synth.ARCH_ENCODER)
    with use_params(store_of(synth.make_params(cfg, seed=0))):
        with pytest.raises(ValueError, match="no upsample block"):
            nb.assemble_FCNN_decoder(pyramid(cfg), cfg, [torch.zeros(4, 128)])
        with pytest.raises(ValueError, match="no upsample block"):
            T.forward(pyramid(cfg), cfg)
    assert fakes == {}
