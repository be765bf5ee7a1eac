"""GPU parity: fused KPConv, unary GEMM + epilogues, pools and the whole encoder vs the numpy restatement.

Tolerance (north_star): 1e-4 relative on fp32 features. It is applied as
    max |gpu - ref64| <= 1e-4 * max |ref64|      (per tensor; max-norm relative error)
against the float64 evaluation of the restatement, so that the reference's own fp32 summation-order noise
(measured ~1e-6..1e-5, tests/test_oracle_golden.py) is not mistaken for our error.
"""
import numpy as np
import pytest
import torch

from oracle import native as on
from oracle import kpconv_np as ok

pytestmark = pytest.mark.gpu

RTOL = 1e-4


def t(a, dev):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def rel_err(a, b):
    a = np.asarray(a, np.float64)
    b = np.asarray(b, np.float64)
    return np.abs(a - b).max() / max(np.abs(b).max(), 1e-30)


def make_case(rng, Nq, Ns, H, Cin, Cout, K=15, extent=0.06, shadow_frac=0.25):
    s = rng.uniform(0, 1, (Ns, 3)).astype(np.float32)
    q = s[:Nq].copy() if Nq <= Ns else rng.uniform(0, 1, (Nq, 3)).astype(np.float32)
    # neighbours: real radius search so that geometry is meaningful, plus shadow padding
    idx = on.port_batch_neighbors(q, s, [Nq], [Ns], 2.5 * extent, max_cols=H)
    if idx.shape[1] < H:
        idx = np.concatenate([idx, np.full((Nq, H - idx.shape[1]), Ns, np.int32)], 1)
    f = rng.normal(size=(Ns, Cin)).astype(np.float32)
    Kp = np.concatenate([np.zeros((1, 3)), rng.normal(size=(K - 1, 3))], 0)
    Kp[1:] *= 1.5 * extent / np.linalg.norm(Kp[1:], axis=1, keepdims=True)
    W = (rng.normal(size=(K, Cin, Cout)) * np.sqrt(2.0 / Cout)).astype(np.float32)
    return q, s, idx.astype(np.int32), f, Kp.astype(np.float32), W


@pytest.mark.parametrize("Cin,Cout,Nq,Ns", [(1, 64, 3000, 3000), (32, 32, 3000, 3000), (64, 64, 900, 3000),
                                            (128, 128, 700, 700), (256, 256, 300, 300), (48, 40, 500, 500)])
def test_kpconv_ops_matches_restatement(cuda, Cin, Cout, Nq, Ns):
    from d3feat_b200 import convolution_ops as co
    rng = np.random.default_rng(Cin * 1000 + Cout)
    extent = 0.06 if Ns >= 2000 else 0.12
    q, s, idx, f, Kp, W = make_case(rng, Nq, Ns, 40, Cin, Cout, extent=extent)
    if Cin == 1:
        f = np.ones_like(f)            # first layer of the network (datasets/ThreeDMatch.py:316)
    out = co.KPConv_ops(t(q, cuda), t(s, cuda), t(idx, cuda), t(f, cuda), t(Kp, cuda), t(W, cuda), extent, "linear",
                        "sum").cpu().numpy()
    ref = ok.kpconv_ops(q, s, idx, f, Kp, W, extent, "linear", "sum", dtype=np.float64)
    assert out.shape == ref.shape
    assert rel_err(out, ref) < RTOL


@pytest.mark.parametrize("influence", ["constant", "linear", "gaussian"])
@pytest.mark.parametrize("mode", ["sum", "closest"])
def test_kpconv_influence_and_mode(cuda, influence, mode):
    from d3feat_b200 import convolution_ops as co
    rng = np.random.default_rng(5)
    q, s, idx, f, Kp, W = make_case(rng, 800, 800, 32, 32, 48, extent=0.1)
    out = co.KPConv_ops(t(q, cuda), t(s, cuda), t(idx, cuda), t(f, cuda), t(Kp, cuda), t(W, cuda), 0.1, influence,
                        mode).cpu().numpy()
    ref = ok.kpconv_ops(q, s, idx, f, Kp, W, 0.1, influence, mode, dtype=np.float64)
    assert rel_err(out, ref) < RTOL


def test_kpconv_enum_errors_and_fused_epilogue(cuda):
    from d3feat_b200 import convolution_ops as co
    rng = np.random.default_rng(6)
    q, s, idx, f, Kp, W = make_case(rng, 400, 400, 24, 32, 32, extent=0.12)
    args = [t(x, cuda) for x in (q, s, idx, f, Kp, W)]
    with pytest.raises(ValueError):
        co.KPConv_ops(*args, 0.12, "cubic", "sum")
    with pytest.raises(ValueError):
        co.KPConv_ops(*args, 0.12, "linear", "mean")
    scale = rng.uniform(0.5, 1.5, 32).astype(np.float32)
    shift = rng.normal(size=32).astype(np.float32)
    out = co.KPConv_ops(*args, 0.12, "linear", "sum", epilogue=(t(scale, cuda), t(shift, cuda), 0.2)).cpu().numpy()
    ref = ok.kpconv_ops(q, s, idx, f, Kp, W, 0.12, "linear", "sum", dtype=np.float64) * scale + shift
    ref = np.where(ref > 0, ref, 0.2 * ref)
    assert rel_err(out, ref) < RTOL


def test_normalisation_counts_positive_feature_rows(cuda):
    """nn counts neighbours whose feature-row SUM is > 0 (convolution_ops.py:249-253), not real neighbours."""
    from d3feat_b200 import convolution_ops as co
    rng = np.random.default_rng(7)
    q, s, idx, f, Kp, W = make_case(rng, 500, 500, 20, 32, 32, extent=0.12)
    f[::3] = -np.abs(f[::3])            # a third of the supports have a negative row sum
    out = co.KPConv_ops(t(q, cuda), t(s, cuda), t(idx, cuda), t(f, cuda), t(Kp, cuda), t(W, cuda), 0.12, "linear",
                        "sum").cpu().numpy()
    ref = ok.kpconv_ops(q, s, idx, f, Kp, W, 0.12, "linear", "sum", dtype=np.float64)
    assert rel_err(out, ref) < RTOL


@pytest.mark.parametrize("Cin,Cout", [(1, 64), (32, 32), (64, 64), (128, 128), (48, 40)])
def test_query_order_is_only_a_scheduling_hint(cuda, Cin, Cout):
    """Walking the queries in a permuted (hash-grid cell) order must not change any output row."""
    from d3feat_b200 import convolution_ops as co, tf_custom_ops as ops
    rng = np.random.default_rng(11 + Cin)
    q, s, idx, f, Kp, W = make_case(rng, 2500, 2500, 40, Cin, Cout, extent=0.08)
    args = [t(x, cuda) for x in (q, s, idx, f, Kp, W)]
    base = co.KPConv_ops(*args, 0.08, "linear", "sum")
    perm = t(rng.permutation(2500).astype(np.int32), cuda)
    assert torch.equal(co.KPConv_ops(*args, 0.08, "linear", "sum", query_order=perm), base)
    one = torch.tensor([2500], dtype=torch.int32, device=cuda)
    grid = ops.NeighborGrid(args[1], one, 0.2)
    order = grid.order()
    assert sorted(order.cpu().tolist()) == list(range(2500))
    assert torch.equal(co.KPConv_ops(*args, 0.08, "linear", "sum", query_order=order), base)


@pytest.mark.parametrize("modulated", [False, True])
def test_kpconv_deformable(cuda, modulated):
    from d3feat_b200 import convolution_ops as co
    rng = np.random.default_rng(8)
    K, Cin, Cout = 15, 32, 32
    q, s, idx, f, Kp, W = make_case(rng, 600, 600, 48, Cin, Cout, extent=0.1)
    offsets = (rng.normal(size=(600, K, 3)) * 0.03).astype(np.float32)
    mods = rng.uniform(0.5, 1.5, (600, K)).astype(np.float32) if modulated else None
    for infl in ("linear", "constant", "gaussian"):
        out = co.KPConv_deform_ops(t(q, cuda), t(s, cuda), t(idx, cuda), t(f, cuda), t(Kp, cuda), t(offsets, cuda),
                                   t(mods, cuda) if modulated else None, t(W, cuda), 0.1, infl, "sum").cpu().numpy()
        ref = ok.kpconv_deform_ops(q, s, idx, f, Kp, offsets, mods, W, 0.1, infl, "sum", dtype=np.float64)
        assert rel_err(out, ref) < RTOL, infl


@pytest.mark.parametrize("N,Cin,Cout", [(3000, 64, 32), (3000, 32, 128), (645, 1024, 256), (195, 512, 2048), (7, 5, 3)])
def test_unary_convolution_and_epilogues(cuda, N, Cin, Cout):
    from d3feat_b200 import convolution_ops as co
    rng = np.random.default_rng(N + Cin)
    x = rng.normal(size=(N, Cin)).astype(np.float32)
    w = (rng.normal(size=(Cin, Cout)) * np.sqrt(2.0 / Cout)).astype(np.float32)
    out = co.unary_convolution(t(x, cuda), t(w, cuda)).cpu().numpy()
    ref = x.astype(np.float64) @ w.astype(np.float64)
    assert rel_err(out, ref) < RTOL
    scale = rng.uniform(0.5, 1.5, Cout).astype(np.float32)
    shift = rng.normal(size=Cout).astype(np.float32)
    res = rng.normal(size=(N, Cout)).astype(np.float32)
    out = co.unary_convolution(t(x, cuda), t(w, cuda), epilogue=(t(scale, cuda), t(shift, cuda), 0.2),
                               residual=t(res, cuda)).cpu().numpy()
    y = ref * scale + shift + res
    y = np.where(y > 0, y, 0.2 * y)
    assert rel_err(out, y) < RTOL


def test_pools_and_standalone_epilogue(cuda):
    from d3feat_b200 import network_blocks as nb
    from d3feat_b200.variables import ParamStore, use_params, variable_scope
    rng = np.random.default_rng(9)
    x = rng.normal(size=(900, 128)).astype(np.float32)
    inds = rng.integers(0, 901, (300, 17)).astype(np.int32)
    inds[5] = 900                                           # an all-shadow row -> column minima
    out = nb.ind_max_pool(t(x, cuda), t(inds, cuda)).cpu().numpy()
    assert np.array_equal(out, ok.ind_max_pool(x, inds))    # max / min are exact
    inds2 = inds.copy()
    inds2[5, 3] = 7                                         # every row has a real neighbour: the lazy column-min
    out = nb.ind_max_pool(t(x, cuda), t(inds2, cuda)).cpu().numpy()   # pass must not be needed, result unchanged
    assert np.array_equal(out, ok.ind_max_pool(x, inds2))
    out = nb.closest_pool(t(x, cuda), t(inds, cuda)).cpu().numpy()
    assert np.array_equal(out, ok.closest_pool(x, inds))
    bn = {"s/batch_normalization/gamma": rng.uniform(0.5, 1.5, 128), "s/batch_normalization/beta": rng.normal(size=128),
          "s/batch_normalization/moving_mean": rng.normal(size=128),
          "s/batch_normalization/moving_variance": rng.uniform(0.5, 2, 128)}
    store = ParamStore(bn, cuda)
    with use_params(store), variable_scope("s"):
        y = nb.leaky_relu(nb.batch_norm(t(x, cuda), True, 0.98, False)).cpu().numpy()
    ref = ok.leaky_relu(ok.batch_norm_inference(x.astype(np.float64), {k.split("/")[-1]: v for k, v in bn.items()}))
    assert rel_err(y, ref) < 1e-6
    with pytest.raises(NotImplementedError):
        with use_params(store), variable_scope("s"):
            nb.batch_norm(t(x, cuda), True, 0.98, True)


def _encoder_case(cuda, cfg, clouds, limits, seed=0, decoder=False):
    from d3feat_b200 import synth
    from d3feat_b200.encoder import KPFCNN
    P = np.concatenate(clouds, 0)
    L = np.array([c.shape[0] for c in clouds], np.int32)
    params = synth.make_params(cfg, seed)
    enc = KPFCNN(cfg, params, limits, device=cuda)
    out = enc(P, L, decoder=decoder)
    inputs = {k: [x.cpu().numpy() for x in v] for k, v in out["inputs"].items() if k != "features"}
    inputs["features"] = np.ones((P.shape[0], 1), np.float32)
    return P, L, params, out, inputs


def test_pyramid_matches_oracle_pyramid(cuda):
    """Every neighbour / pool / upsample matrix and every level's points, bit-exact, vs the oracle pyramid built
    with the C restatement (same canonical orders)."""
    from d3feat_b200 import synth
    cfg = synth.Config(architecture=synth.ARCH_ENCODER)
    clouds = [synth.room_fragment(20, 6000), synth.room_fragment(21, 5000)]
    limits = [35, 33, 34, 36, 30]
    P, L, params, out, inputs = _encoder_case(cuda, cfg, clouds, limits)
    ref = ok.descriptor_input_pyramid(cfg, P, L, limits, on.port_batch_neighbors, on.port_batch_subsampling)
    for l in range(5):
        assert np.array_equal(inputs["points"][l].view(np.uint32), ref["points"][l].view(np.uint32)), l
        assert np.array_equal(inputs["lengths"][l], ref["lengths"][l])
        for key in ("neighbors", "pools", "upsamples"):
            a, b = inputs[key][l], ref[key][l]
            if b.shape[0] == 0:
                assert a.shape[0] == 0
                continue
            Ns = {"neighbors": l, "pools": l, "upsamples": l + 1}[key]
            shadow = ref["points"][Ns].shape[0]
            # ours is always `limit` wide; the reference slice is min(max count, limit) wide: pad to compare
            if b.shape[1] < a.shape[1]:
                b = np.concatenate([b, np.full((b.shape[0], a.shape[1] - b.shape[1]), shadow, np.int32)], 1)
            assert np.array_equal(a, b), (key, l)


def test_encoder_matches_restatement_5_levels(cuda):
    from d3feat_b200 import synth
    cfg = synth.Config(architecture=synth.ARCH_ENCODER)
    clouds = [synth.room_fragment(30, 9000), synth.room_fragment(31, 7000)]
    P, L, params, out, inputs = _encoder_case(cuda, cfg, clouds, [35, 33, 34, 36, 30])
    F_ref, trace = ok.EncoderOracle(cfg, params, np.float64).encoder(inputs, return_all=True)
    assert [f.shape[1] for f in out["F"]] == [128, 256, 512, 1024, 2048]
    for l, (a, b) in enumerate(zip(out["F"], F_ref)):
        assert rel_err(a.cpu().numpy(), b) < RTOL, "level %d" % l


def test_encoder_with_decoder_descriptors(cuda):
    from d3feat_b200 import synth
    cfg = synth.Config()
    clouds = [synth.room_fragment(40, 6000)]
    P, L, params, out, inputs = _encoder_case(cuda, cfg, clouds, [35, 33, 34, 36, 30], decoder=True)
    orc = ok.EncoderOracle(cfg, params, np.float64)
    F_ref = orc.encoder(inputs)
    d_ref = orc.decoder(inputs, F_ref)
    d = out["descriptors"].cpu().numpy()
    assert d.shape == (6000, 32)
    assert np.allclose(np.linalg.norm(d, axis=1), 1.0, atol=1e-5)
    assert np.abs(d - d_ref).max() < RTOL          # unit-norm rows: absolute == relative to the row norm


def test_deformable_architecture_runs_and_matches(cuda):
    from d3feat_b200 import synth
    cfg = synth.Config(architecture=synth.ARCH_KITTI_DEFORM, first_subsampling_dl=0.3, first_features_dim=32)
    cloud = synth.lidar_scan(0, 9000)
    P, L, params, out, inputs = _encoder_case(cuda, cfg, [cloud], [40, 40, 40, 60, 40])
    F_ref = ok.EncoderOracle(cfg, params, np.float64).encoder(inputs)
    for l, (a, b) in enumerate(zip(out["F"], F_ref)):
        assert rel_err(a.cpu().numpy(), b) < RTOL, "level %d" % l


@pytest.mark.parametrize("Nq,Ns,H,Cout", [(6000, 6000, 40, 32), (4001, 9000, 37, 32), (20011, 20011, 45, 32),
                                          (3600, 3600, 8, 32)])
def test_kpconv_fused_kernel_matches_restatement_and_two_kernel_path(cuda, monkeypatch, Nq, Ns, H, Cout):
    """The persistent fused kernel of the Cin = 32 layers (kpconv_fused.cu: gather + correlation on mma.sync, contraction
    on wgmma out of a shared-memory B operand): vs the float64 restatement (1e-4) and vs the two-kernel path of the
    same library (both 3xTF32: agree far below the tolerance). Ragged tail tile (Nq % 48 != 0), strided queries
    (Nq != Ns), H not a multiple of 8, fused BN + LeakyReLU epilogue."""
    from d3feat_b200 import convolution_ops as co
    rng = np.random.default_rng(Nq + H)
    q, s, idx, f, Kp, W = make_case(rng, Nq, Ns, H, 32, Cout, extent=0.05)
    f[::5] = -np.abs(f[::5])                      # some supports do not count towards nn (:249-253)
    args = [t(x, cuda) for x in (q, s, idx, f, Kp, W)]
    scale = rng.uniform(0.5, 1.5, Cout).astype(np.float32)
    shift = rng.normal(size=Cout).astype(np.float32)
    epi = (t(scale, cuda), t(shift, cuda), 0.2)
    monkeypatch.setenv("D3F_FUSED_KPCONV", "1")
    co.packed_weight(args[5])                     # the one-time weight packing is not part of a call
    n0 = co._lib.launch_count()
    fused = co.KPConv_ops(*args, 0.05, "linear", "sum", epilogue=epi)
    fused_raw = co.KPConv_ops(*args, 0.05, "linear", "sum")
    launches_fused = co._lib.launch_count() - n0
    monkeypatch.setenv("D3F_FUSED_KPCONV", "0")
    n0 = co._lib.launch_count()
    two = co.KPConv_ops(*args, 0.05, "linear", "sum", epilogue=epi)
    assert launches_fused == 6      # per call: support packing, 8 KB-image weight packing, ONE persistent kernel
    ref = ok.kpconv_ops(q, s, idx, f, Kp, W, 0.05, "linear", "sum", dtype=np.float64)
    assert rel_err(fused_raw.cpu().numpy(), ref) < RTOL
    y = ref * scale + shift
    y = np.where(y > 0, y, 0.2 * y)
    assert rel_err(fused.cpu().numpy(), y) < RTOL
    assert rel_err(fused.cpu().numpy(), two.cpu().numpy()) < 2e-5
    # bit-reproducible (no atomics, fixed tile schedule)
    monkeypatch.setenv("D3F_FUSED_KPCONV", "1")
    assert torch.equal(co.KPConv_ops(*args, 0.05, "linear", "sum", epilogue=epi), fused)


@pytest.mark.parametrize("Cin,Cout,Nq,Ns,H", [(32, 32, 3000, 3000, 40), (64, 64, 900, 3000, 37), (128, 128, 700, 700, 40),
                                              (512, 512, 300, 300, 21)])
def test_kpconv_staged_stage1_variant(cuda, monkeypatch, Cin, Cout, Nq, Ns, H):
    """D3F_S1_STAGED=1: stage 1 with the gathered rows staged through shared memory (cp.async in the coalesced
    assignment, zero-filled shadow rows, swizzled conflict-free fragment reads, double-buffered per warp) -- same
    result as the default register-gather kernel (both 3xTF32; identical arithmetic per element) and within 1e-4 of
    the float64 restatement. H not a multiple of 8, strided queries, several channel passes (Cin = 512)."""
    from d3feat_b200 import convolution_ops as co
    rng = np.random.default_rng(Cin + H)
    extent = 0.06 if Ns >= 2000 else 0.12
    q, s, idx, f, Kp, W = make_case(rng, Nq, Ns, H, Cin, Cout, extent=extent)
    f[::7] = -np.abs(f[::7])
    args = [t(x, cuda) for x in (q, s, idx, f, Kp, W)]
    monkeypatch.setenv("D3F_S1_STAGED", "0")
    base = co.KPConv_ops(*args, extent, "linear", "sum")
    monkeypatch.setenv("D3F_S1_STAGED", "1")
    staged = co.KPConv_ops(*args, extent, "linear", "sum")
    ref = ok.kpconv_ops(q, s, idx, f, Kp, W, extent, "linear", "sum", dtype=np.float64)
    assert rel_err(staged.cpu().numpy(), ref) < RTOL
    assert torch.equal(staged, base)
