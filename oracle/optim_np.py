"""numpy restatement of the training update (d3f_momentum_clip_update) and the rank mean (d3f_rank_mean);
d3feat_b200/training.py MomentumClip, d3feat_b200/distributed.py rank_mean.

This module is the contract. numpy rounds every float32 `* / + -` of two float32 arrays correctly and never fuses a
multiply with an add, and np.cumsum adds strictly left to right (np.sum would add pairwise), so csrc/optim.cu's
__fmul_rn / __fdiv_rn / __fadd_rn / __fsub_rn and its sequential fp64 sums reproduce these results bit for bit.

Per tensor (utils/trainer.py:116-156; TF 1.12 clip_ops.clip_by_norm and training_ops ApplyMomentum):
  l2sum = sum of g^2 in fp64 over fixed 2048-element blocks from element 0, each block summed sequentially, the block
          sums added in block order. TF sums g*g in fp32 in an unspecified order: the one deviation.
  norm  = fl32(sqrt(l2sum)), l2sum itself when not l2sum > 0 (TF's where(pred, sqrt(l2sum_safe), l2sum))
  M     = c if norm < c else norm             (Eigen's maximum: a NaN norm stays NaN)
  gc    = fl32(fl32(g * c) / M)               (c = fl32(clip_norm); clip_norm <= 0: gc = g, trainer.py:150-153)
  accum = fl32(fl32(accum * momentum) + gc)
  var   = fl32(var - fl32(accum * lr))
"""
import numpy as np

BLOCK = 2048
_F32 = np.float32


def sequential_sum(a):
    """a[0] + a[1] + ... in a's dtype, left to right (0 for an empty a)."""
    a = np.asarray(a)
    return np.cumsum(a)[-1] if a.size else a.dtype.type(0)


def l2sum(g):
    """The fp64 sum of squares of g in 2048-element blocks, each sequential, the blocks in order."""
    g = np.asarray(g, _F32).reshape(-1).astype(np.float64)
    if g.size == 0:
        return np.float64(0)
    nb = -(-g.size // BLOCK)
    sq = np.zeros(nb * BLOCK, np.float64)      # the zero padding of the last block adds exact zeros to a sum >= 0
    sq[:g.size] = g * g                        # exact: fp32 squares fit in fp64
    parts = np.cumsum(sq.reshape(nb, BLOCK), axis=1)[:, -1]
    return np.float64(sequential_sum(parts))


def clip_norm_max(g, clip_norm):
    """M = max(norm, c) of one gradient, in fp32."""
    s = l2sum(g)
    norm = _F32(np.sqrt(s)) if s > 0 else _F32(s)
    c = _F32(clip_norm)
    return c if norm < c else norm


def clip_by_norm(g, clip_norm):
    """tf.clip_by_norm(g, clip_norm) under the contract above (g returned as it is for clip_norm <= 0)."""
    g = np.asarray(g, _F32)
    if not clip_norm > 0:
        return g.copy()
    c = _F32(clip_norm)
    return (g * c) / clip_norm_max(g, clip_norm)


def momentum_clip_update(var, accum, grad, lr, momentum, clip_norm):
    """One update of one tensor: (new var, new accum), both float32 of var's shape."""
    gc = clip_by_norm(grad, clip_norm)
    a = np.asarray(accum, _F32) * _F32(momentum) + gc
    return np.asarray(var, _F32) - a * _F32(lr), a


def rank_mean(x):
    """x[R, P] float32 -> out[P] = fl32((x[0] + x[1] + ... + x[R-1]) / R), the sum in fp64 in rank order from x[0]."""
    x = np.asarray(x, _F32)
    s = x[0].astype(np.float64)
    for r in range(1, x.shape[0]):
        s = s + x[r].astype(np.float64)
    return (s / np.float64(x.shape[0])).astype(_F32)


def learning_rate(learning_rate, lr_decays, epoch):
    """The learning rate during epoch `epoch` (0-based) of utils/trainer.py:376-381: a float32 variable that starts at
    learning_rate and, at the end of every epoch e in lr_decays, becomes fl32(lr * fl32(lr_decays[e]))."""
    lr = _F32(learning_rate)
    for e in range(int(epoch)):
        if e in lr_decays:
            lr = lr * _F32(lr_decays[e])
    return lr
