"""Random keypoints of B stacked clouds in numpy: the contract of d3f_sample_keypoints (keypoints.sample_keypoints).

The testers' `-rand` arm draws np.random.choice(n_b, k) per cloud, with replacement (utils/tester.py:238-279,
geometric_registration/evaluate.py:45-54). Here every slot is its own counter-based draw, the splitmix64 and
multiply-shift of register_np.sample_index:

    c = (b << 32) | j,  z = splitmix64(seed + c * 0x9E3779B97F4A7C15),  index[b, j] = s_b + (((z >> 32) * n_b) >> 32)

(uint64, wrapping), where cloud b holds rows [s_b, s_b + n_b): the stack offsets of `lengths` cut at the row count n.
count[b] = k when n_b >= 1; an empty cloud has count 0 and index -1. The first c slots of a k-slot draw are the c-slot
draw with the same seed.
"""
import numpy as np

from .register_np import U, splitmix64

GOLDEN = 0x9E3779B97F4A7C15


def cloud_ranges(lengths, n):
    """(s [B], n_b [B]) int64: the stack offsets of `lengths` cut at n rows, as the kernels cut them."""
    start = np.concatenate([[0], np.cumsum(np.asarray(lengths, np.int64))])
    s = np.clip(start[:-1], 0, n)
    e = np.minimum(np.maximum(start[1:], s), n)
    return s, e - s


def sample_keypoints(lengths, k, seed, n):
    """(index [B,k] int32, count [B] int32) of k draws per cloud of a stack of n rows."""
    s, nb = cloud_ranges(lengths, n)
    B = len(s)
    b = np.repeat(np.arange(B, dtype=np.uint64), k).reshape(B, k)
    j = np.tile(np.arange(k, dtype=np.uint64), (B, 1))
    c = (b << U(32)) | j
    with np.errstate(over="ignore"):
        z = splitmix64(U(int(seed) & ((1 << 64) - 1)) + c * U(GOLDEN))
        off = ((z >> U(32)) * nb.astype(U)[:, None]) >> U(32)
    real = nb > 0
    index = np.where(real[:, None], s[:, None] + off.astype(np.int64), -1).astype(np.int32)
    count = np.where(real, k, 0).astype(np.int32)
    return index, count


def gather(index, rows):
    """rows[index] with zero rows where index is -1 (the padding of an empty cloud), rows [N, ...] float32."""
    rows = np.asarray(rows, np.float32)
    real = index >= 0
    out = rows[np.where(real, index, 0)]
    out[~real] = 0
    return out
