"""CPU: oracle/optim_np.py (the contract of d3f_momentum_clip_update and d3f_rank_mean) against a literal transcription
of TF 1.12's clip_by_norm and ApplyMomentum, the learning-rate decay against TF's float32 chain, and the argument checks
of the new entry points, which refuse before any CUDA call."""
import ctypes
import math

import numpy as np
import pytest
import torch

from oracle import optim_np as oo

F32 = np.float32


def tf_clip_by_norm(t, clip_norm, l2sum):
    """clip_ops.clip_by_norm (TF 1.12) for axes=None, line by line, in float32; l2sum = reduce_sum(t * t) is given
    (rounded to float32), because TF's fp32 sum has no stated order."""
    t = np.asarray(t, F32)
    l2sum = F32(l2sum)
    clip_norm = F32(clip_norm)                        # ops.convert_to_tensor(clip_norm, dtype=t.dtype)
    pred = l2sum > 0
    l2sum_safe = np.where(pred, l2sum, np.ones_like(l2sum))
    l2norm = np.where(pred, np.sqrt(l2sum_safe), l2sum)
    intermediate = t * clip_norm
    return intermediate / np.maximum(l2norm, clip_norm)


def tf_apply_momentum(var, accum, grad, lr, momentum):
    """training_ops ApplyMomentum, use_nesterov = False: accum = accum * momentum + grad; var -= accum * lr."""
    accum = np.asarray(accum, F32) * F32(momentum) + np.asarray(grad, F32)
    return np.asarray(var, F32) - accum * F32(lr), accum


def tf_step(var, accum, grad, lr, momentum, clip_norm, l2sum):
    """utils/trainer.py:129-156 for one tensor."""
    if clip_norm > 0:
        grad = tf_clip_by_norm(grad, clip_norm, l2sum)
    return tf_apply_momentum(var, accum, grad, lr, momentum)


def bits(a):
    return np.asarray(a, F32).view(np.uint32)


ULP_G = np.array([1013799911], np.uint32).view(F32)[0]      # 0.014487243...: fl32(fl32(g * 100) / 100) != g


def cases():
    rng = np.random.default_rng(0)
    big = (rng.normal(size=5000) * 10).astype(F32)           # norm ~700: clipped at 100
    small = (rng.normal(size=3000) * 0.1).astype(F32)        # norm ~5: not clipped
    return {
        "clip active": (big, 100.0),
        "clip inactive": (small, 100.0),
        "ulp below the threshold": (np.array([ULP_G, 0.5, -0.25], F32), 100.0),
        "zero gradient": (np.zeros(2049, F32), 100.0),
        "negative zero gradient": (-np.zeros(7, F32), 100.0),
        "clip_norm 0": (big, 0.0),
        "clip_norm negative": (big, -1.0),
        "1 element clipped": (np.array([-250.0], F32), 100.0),
        "1 element not clipped": (np.array([3.0], F32), 100.0),
        "1 element zero": (np.array([0.0], F32), 100.0),
        "2049 elements": ((rng.normal(size=2049) * 3).astype(F32), 100.0),
    }


@pytest.mark.parametrize("name", sorted(cases()))
def test_update_equals_tf_transcription(name):
    g, c = cases()[name]
    rng = np.random.default_rng(1)
    var = rng.normal(size=g.shape).astype(F32)
    accum = (rng.normal(size=g.shape) * 0.01).astype(F32)
    lr, m = 0.1, 0.98
    v1, a1 = oo.momentum_clip_update(var, accum, g, lr, m, c)
    v2, a2 = tf_step(var, accum, g, lr, m, c, oo.l2sum(g))
    assert np.array_equal(bits(v1), bits(v2)) and np.array_equal(bits(a1), bits(a2)), name
    assert np.array_equal(bits(oo.clip_by_norm(g, c)), bits(tf_clip_by_norm(g, c, oo.l2sum(g)) if c > 0 else g))


def test_clip_active_and_inactive_and_zero():
    cs = cases()
    big, c = cs["clip active"]
    out = oo.clip_by_norm(big, c)
    assert abs(float(np.sqrt((out.astype(np.float64) ** 2).sum())) - 100.0) < 1e-3
    assert np.array_equal(oo.clip_by_norm(*cs["1 element clipped"]), np.array([-100.0], F32))
    z = oo.clip_by_norm(*cs["zero gradient"])
    assert not z.any() and oo.clip_norm_max(cs["zero gradient"][0], 100.0) == F32(100)   # norm 0, no division by 0
    assert np.array_equal(bits(oo.clip_by_norm(*cs["negative zero gradient"])), bits(-np.zeros(7, F32)))
    for name in ("clip_norm 0", "clip_norm negative"):
        g, c = cs[name]
        assert np.array_equal(bits(oo.clip_by_norm(g, c)), bits(g))


def test_ulp_change_below_the_threshold():
    """Below the threshold TF still computes (g * c) / c: g = 0.014487243 (bits 0x3C6D5BE7) comes back one ulp lower,
    where torch.nn.utils.clip_grad_norm_ leaves it as it is."""
    g = np.array([ULP_G, 0.5, -0.25], F32)
    out = oo.clip_by_norm(g, 100.0)
    assert int(bits(out)[0]) == int(bits(g)[0]) - 1
    assert np.array_equal(out[1:], g[1:])
    t = torch.from_numpy(g.copy())
    t.grad = t.clone()
    torch.nn.utils.clip_grad_norm_([t], 100.0)
    assert np.array_equal(bits(t.grad.numpy()), bits(g))


def test_l2sum_block_order_and_accuracy():
    rng = np.random.default_rng(2)
    for n in (1, 2047, 2048, 2049, 6145):
        g = (rng.normal(size=n) * np.exp(rng.normal(size=n) * 3)).astype(F32)
        s = oo.l2sum(g)
        blocks = [math.fsum(float(v) * float(v) for v in g[i:i + 2048]) for i in range(0, n, 2048)]
        assert abs(s - math.fsum(blocks)) <= 1e-12 * s
        # the blocks themselves: sequential inside, then in block order
        g64 = g.astype(np.float64)
        want = 0.0
        for i in range(0, n, 2048):
            p = 0.0
            for v in g64[i:i + 2048]:
                p += v * v
            want += p
        assert s == want


def test_rank_mean_oracle():
    x = np.array([[1.0, -0.0, np.nan, 3.0, 1e30]], F32)
    assert np.array_equal(bits(oo.rank_mean(x)), bits(x[0]))          # R = 1: the input, -0.0 and NaN included
    rng = np.random.default_rng(3)
    x = rng.normal(size=(3, 1000)).astype(F32)
    want = np.array([F32((float(a) + float(b) + float(c)) / 3.0) for a, b, c in x.T], F32)
    assert np.array_equal(oo.rank_mean(x), want)


def test_learning_rate_matches_tf_float32_chain():
    from d3feat_b200 import synth, training as T
    cfg = synth.Config(**T.TRAINING_3DMATCH)
    assert cfg.lr_decays == {i: 0.1 ** (1 / 80) for i in range(1, 200)}        # training_3DMatch.py:107
    lr = F32(0.1)                                                             # tf.Variable(learning_rate): float32
    seen64 = 0.1
    differs = 0
    for epoch in range(201):
        got = T.learning_rate(cfg, epoch)
        assert got == float(lr) == float(oo.learning_rate(0.1, cfg.lr_decays, epoch)), epoch
        differs += got != float(F32(seen64))
        if epoch in cfg.lr_decays:                                            # end of epoch: assign(lr * decay)
            lr = F32(lr * F32(cfg.lr_decays[epoch]))
            seen64 *= cfg.lr_decays[epoch]
    assert differs > 0                                                        # the float32 chain is not fp64's
    assert abs(T.learning_rate(cfg, 81) / 0.01 - 1) < 1e-5                    # 80 decays: one tenth
    with pytest.raises(TypeError):
        cfg.lr_decays[5] = 0.5                              # shared by every Config: read-only
    assert T.TRAINING_KITTI["lr_decays"][5] == 0.1 ** (1 / 80)
    cfg.lr_decays = {}
    assert T.learning_rate(cfg, 150) == float(F32(0.1))


# ---------------------------------------------------------------------------------------------------- argument checks

def test_python_entry_points_refuse_wrong_arguments():
    from d3feat_b200 import distributed as D, training as T
    with pytest.raises(ValueError, match=r"MomentumClip: params\[0\] must be a float32 CUDA tensor"):
        T.MomentumClip([torch.zeros(3)], 0.1, 0.9, 100.0)
    with pytest.raises(ValueError, match=r"MomentumClip: params\[0\] must be a contiguous tensor"):
        T.MomentumClip([torch.zeros(4, 4).t()], 0.1, 0.9, 100.0)
    with pytest.raises(ValueError, match=r"momentum_clip_update: 1 vars, 2 accums and 1 grads"):
        T.momentum_clip_update([torch.zeros(3)], [torch.zeros(3)] * 2, [torch.zeros(3)], 0.1, 0.9, 1.0)
    with pytest.raises(ValueError, match=r"momentum_clip_update: var\[0\] must be a float32 CUDA tensor"):
        T.momentum_clip_update([torch.zeros(3)], [torch.zeros(3)], [torch.zeros(3)], 0.1, 0.9, 1.0)
    with pytest.raises(ValueError, match=r"rank_mean: x must be a float32 CUDA tensor of shape \[\*, \*\]"):
        D.rank_mean(torch.zeros(2, 3))
    with pytest.raises(ValueError, match=r"rank_mean: x must be a float32 CUDA tensor"):
        D.rank_mean(torch.zeros(3))
    with pytest.raises(ValueError, match=r"gather_step_stats: 2 values"):
        D.gather_step_stats([torch.zeros(()), torch.zeros(())])
    with pytest.raises(ValueError, match=r"reduce_gradients: params\[0\] must be a float32 CUDA tensor"):
        D.reduce_gradients([torch.zeros(3, dtype=torch.float64)])


def test_c_entry_points_refuse_before_any_cuda_call():
    from d3feat_b200 import build, _lib
    build.build()
    L = _lib.lib()
    fake = ctypes.c_void_p(256)
    assert L.d3f_momentum_clip_workspace_bytes(-1, 10) == 0
    assert L.d3f_momentum_clip_workspace_bytes(1025, 10) == 0
    assert L.d3f_momentum_clip_workspace_bytes(3, 4097) >= (3 + 3) * 8
    assert L.d3f_momentum_clip_update(fake, 1025, 10, 0.1, 0.9, 1.0, fake, 1 << 20, None) == -1
    assert b"T=1025" in L.d3f_last_error()
    assert L.d3f_momentum_clip_update(fake, 2, 10, float("nan"), 0.9, 1.0, fake, 1 << 20, None) == -1
    assert b"finite" in L.d3f_last_error()
    assert L.d3f_momentum_clip_update(None, 2, 10, 0.1, 0.9, 1.0, fake, 1 << 20, None) == -1
    assert L.d3f_momentum_clip_update(fake, 2, 10, 0.1, 0.9, 1.0, fake, 8, None) == -4
    assert L.d3f_momentum_clip_update(None, 0, 0, 0.1, 0.9, 1.0, None, 0, None) == 0          # nothing to do
    assert L.d3f_rank_mean(fake, 0, 10, fake, None) == -1
    assert b"R=0" in L.d3f_last_error()
    assert L.d3f_rank_mean(None, 2, 10, fake, None) == -1
    assert L.d3f_rank_mean(None, 2, 0, None, None) == 0
