"""Mirror of kernels/kernel_points.py: the kernel-point dispositions a new run starts from, optimised on the GPU.

  kernel_point_optimization(radius, num_points, num_kernels, dimension, fixed, ratio)   :41-181
      (kernel_point_optimization_debug) -> (points [num_kernels, num_points, 3] * radius, saved_gradient_norms)
  load_kernels(radius, num_kpoints, num_kernels, dimension, fixed)                       :184-280
      -> [num_kernels, num_kpoints, 3], each the shared disposition rotated (and jittered)
  optimize(initial, fixed)                   the loop of :102-174 on the GPU (csrc/kernel_points.cu)

The optimiser runs the reference's loop in fp64 on the GPU, bit for bit as oracle/kernel_points_np.py restates it;
its one deviation is d^3 computed as d2 * sqrt(d2) instead of pow(d2, 3/2). The rest is host numpy in fp64:
  * the initial points (:76-91): rejection sampling of uniform points on [-1, 1)^3 inside |p|^2 < 0.5, the first
    num_kernels * num_points accepted in draw order, then the 'center' / 'verticals' fixing;
  * the rescale (:176-181): ratio / mean(|p|) over points 1..K-1 of every try, summed sequentially in (try, point)
    order; skipped when K = 1 (no such point);
  * the try load_kernels keeps (:214): argmin of the last row of saved_gradient_norms. That row is zero whenever the
    loop stopped before 10000 iterations, so, as in the reference, try 0 is kept then; the 100 tries still decide when
    the loop stops;
  * the rotations (:228-278): for 'verticals' about z by theta uniform on [0, 2 pi), cos and sin rounded to float32
    as the reference's float32 R holds them, without noise; otherwise u, v
    uniform on [-1, 1)^3 normalised with +1e-9, the pair redrawn while |u.v| > 0.99, Gram-Schmidt, w = u x v,
    R = [u v w] as columns, (radius * D) @ R + N(0, 0.01 radius). Callers cast the result to float32 (convolution_ops.py:145).

Random draws are counter-based splitmix64 (csrc/rng.cuh's function) of (seed, purpose, index): the same seed gives the
same bits on every rank, machine and run. numpy's global stream, which the reference draws from, is not reproduced.
Dispositions are cached per (num_kpoints, fixed, seed) in the process, as the reference caches one PLY file per
(num_kpoints, fixed) in its kernels/dispositions directory; `disposition=` takes a given [K, 3] one instead (for
example the points of a reference run's k_015_center.ply).

The reference fails on an empty maximum when no point moves (K = 1 with 'center', K <= 3 with 'verticals'); here no
iteration runs and the fixed points are returned (scaled when K > 1). dimension != 3 and an unknown `fixed` are
ValueErrors.
"""
import threading

import numpy as np
import torch

from . import _lib
from .trainer import GOLDEN, M64, splitmix64

FIXED = {"none": 0, "center": 1, "verticals": 2}     # include/d3feat_b200.h D3F_FIXED_*
MAX_ITER = 10000
NUM_TRIES = 100                                       # :187
MAX_POINTS = 6400                                     # tries * points the optimiser holds on chip

# the purpose of a draw: the top 16 bits of its counter
INITIAL, ROTATION_U, ROTATION_V, NOISE, THETA, KERNEL_SEED, WEIGHTS = range(7)


# ----------------------------------------------------------------------------------------------------
#  counter-based draws
# ----------------------------------------------------------------------------------------------------

def draw(seed, purpose, index):
    """uint64 draws splitmix64(seed + counter * golden), counter = (purpose << 48) | index, for an index array."""
    c = (np.uint64(purpose) << np.uint64(48)) | np.asarray(index, dtype=np.uint64)
    with np.errstate(over="ignore"):
        return splitmix64(np.uint64(int(seed) & M64) + c * np.uint64(GOLDEN))


def uniform(seed, purpose, index):
    """float64 on [0, 1): the top 53 bits of each draw."""
    return (draw(seed, purpose, index) >> np.uint64(11)).astype(np.float64) * 2.0 ** -53


def normal(seed, purpose, index):
    """Standard normals by Box-Muller from draws 2*index and 2*index + 1."""
    index = np.asarray(index, dtype=np.uint64) * np.uint64(2)
    u1 = 1.0 - uniform(seed, purpose, index)                  # (0, 1]
    u2 = uniform(seed, purpose, index + np.uint64(1))
    return np.sqrt(-2.0 * np.log(u1)) * np.cos(2.0 * np.pi * u2)


def sub_seed(seed, index):
    """The seed of one of several independent streams under `seed` (one per KPConv of a network, say)."""
    return int(draw(seed, KERNEL_SEED, index))


# ----------------------------------------------------------------------------------------------------
#  the optimiser
# ----------------------------------------------------------------------------------------------------

def _check(dimension, fixed):
    if dimension != 3:
        raise ValueError("Unsupported dimension of kernel : %r (only 3 is supported)" % (dimension,))
    if fixed not in FIXED:
        raise ValueError("fixed must be one of %s, got %r" % (tuple(FIXED), fixed))


def initial_points(num_points, num_kernels, seed, fixed):
    """:76-91 -- [num_kernels, num_points, 3]: the first num_kernels * num_points candidates (uniform on [-1, 1)^3,
    candidate i from draws 3i, 3i + 1, 3i + 2) with |p|^2 < 0.5, then fixed."""
    n = num_kernels * num_points
    got, start = [], 0
    while sum(len(g) for g in got) < n:
        m = 6 * n + 64                                     # about 18.5 % of the candidates are kept
        idx = (np.arange(start, start + m, dtype=np.uint64)[:, None] * np.uint64(3)) + np.arange(3, dtype=np.uint64)
        c = uniform(seed, INITIAL, idx) * 2 - 1
        sq = c * c
        got.append(c[((sq[:, 0] + sq[:, 1]) + sq[:, 2]) < 0.5])
        start += m
    return fix_points(np.concatenate(got, 0)[:n].reshape(num_kernels, num_points, 3), fixed)


def fix_points(p, fixed):
    """:85-91 on a copy of p [T, K, 3]."""
    p = np.array(p, dtype=np.float64)
    if fixed == "center":
        p[:, 0, :] *= 0
    if fixed == "verticals":
        p[:, :3, :] *= 0
        p[:, 1:2, -1] += 2 / 3                  # K < 3: the points that exist
        p[:, 2:3, -1] -= 2 / 3
    return p


def optimize(initial, fixed="center"):
    """The loop of :102-174 on the GPU from fixed initial points [T, K, 3] (any float array or tensor; computed in
    fp64 on the current CUDA device) -> (points [T, K, 3] before the rescale, saved_gradient_norms [10000, T],
    iterations: a device int32 scalar, the rows of saved_gradient_norms written). Enqueued on the current stream; no
    synchronisation. ValueError (before any launch) for T * K > 6400 or an unknown fixed."""
    if fixed not in FIXED:
        raise ValueError("optimize: fixed must be one of %s, got %r" % (tuple(FIXED), fixed))
    x = initial if torch.is_tensor(initial) else torch.as_tensor(np.asarray(initial, dtype=np.float64))
    if x.dim() != 3 or x.shape[2] != 3:
        raise ValueError("optimize: initial must be [T, K, 3], got %s" % (list(x.shape),))
    T, K = int(x.shape[0]), int(x.shape[1])
    if T < 1 or K < 1 or T * K > MAX_POINTS:
        raise ValueError("optimize: %d tries of %d points (need T, K >= 1 and T * K <= %d)" % (T, K, MAX_POINTS))
    dev = x.device if x.is_cuda else torch.device("cuda", torch.cuda.current_device())
    x = x.to(device=dev, dtype=torch.float64).contiguous()
    points = torch.empty_like(x)
    saved = torch.empty((MAX_ITER, T), dtype=torch.float64, device=dev)
    iters = torch.empty((), dtype=torch.int32, device=dev)
    _lib.check(_lib.lib().d3f_kernel_point_optimize(_lib.ptr(x), T, K, 3, FIXED[fixed], _lib.ptr(points),
                                                    _lib.ptr(saved), _lib.ptr(iters), _lib.stream()),
               "d3f_kernel_point_optimize")
    return points, saved, iters


def rescale(points, ratio=1.0):
    """:177-178 -- points * ratio / mean(r[:, 1:]), r = sqrt(((x*x + y*y) + z*z) + 1e-12), the mean's sum sequential
    in (try, point) order (np.cumsum). Unchanged for K = 1."""
    if points.shape[1] < 2:
        return points.copy()
    sq = points * points
    r = np.sqrt(((sq[..., 0] + sq[..., 1]) + sq[..., 2]) + 1e-12)[:, 1:]
    return points * (ratio / (np.cumsum(r.ravel())[-1] / r.size))


def kernel_point_optimization(radius, num_points, num_kernels=1, dimension=3, fixed="center", ratio=1.0, *, seed=0,
                              initial=None):
    """:41-181 -- (kernel points [num_kernels, num_points, 3] * radius, saved_gradient_norms [10000, num_kernels]),
    float64 numpy. `initial` replaces the draw of :76-83 (the points before the fixing)."""
    _check(dimension, fixed)
    if initial is None:
        p = initial_points(num_points, num_kernels, seed, fixed)
    else:
        p = fix_points(np.asarray(initial, dtype=np.float64).reshape(num_kernels, num_points, 3), fixed)
    points, saved, _ = optimize(p, fixed)
    return rescale(points.cpu().numpy(), ratio) * radius, saved.cpu().numpy()


# ----------------------------------------------------------------------------------------------------
#  load_kernels
# ----------------------------------------------------------------------------------------------------

_cache = {}
_cache_lock = threading.Lock()


def shared_disposition(num_kpoints, fixed="center", seed=0):
    """:203-218 -- the kept try of a 100-try optimisation at radius 1: [num_kpoints, 3] float64 (read-only), computed
    once per (num_kpoints, fixed, seed) in the process."""
    key = (int(num_kpoints), fixed, int(seed))
    with _cache_lock:
        hit = _cache.get(key)
        if hit is None:
            points, saved = kernel_point_optimization(1.0, num_kpoints, num_kernels=NUM_TRIES, fixed=fixed, seed=seed)
            hit = points[int(np.argmin(saved[-1, :]))]
            hit.setflags(write=False)
            _cache[key] = hit
    return hit


def _unit(x):
    sq = x * x
    return x / (np.sqrt((sq[:, 0] + sq[:, 1]) + sq[:, 2]) + 1e-9)[:, None]


def _dot(a, b):
    ab = a * b
    return (ab[:, 0] + ab[:, 1]) + ab[:, 2]


def rotation(seed, n):
    """:250-268 for kernel n -> (R [3, 3] with columns u, v, w, the number of (u, v) pairs drawn). Attempt a draws u
    and v from counters ((n << 20) | a) * 3 + 0..2."""
    for a in range(1 << 20):
        idx = np.uint64(((n << 20) | a) * 3) + np.arange(3, dtype=np.uint64)
        u = _unit(uniform(seed, ROTATION_U, idx)[None] * 2 - 1)
        v = _unit(uniform(seed, ROTATION_V, idx)[None] * 2 - 1)
        if not np.abs(_dot(u, v))[0] > 0.99:
            break
    v = _unit(v - _dot(u, v)[:, None] * u)
    w = np.stack([u[:, 1] * v[:, 2] - u[:, 2] * v[:, 1],
                  u[:, 2] * v[:, 0] - u[:, 0] * v[:, 2],
                  u[:, 0] * v[:, 1] - u[:, 1] * v[:, 0]], -1)
    return np.stack((u[0], v[0], w[0]), axis=-1), a + 1


def _rotate(d, R):
    """d [K, 3] @ R [3, 3], each output a sequential sum over the 3 inputs."""
    return (d[:, 0:1] * R[0] + d[:, 1:2] * R[1]) + d[:, 2:3] * R[2]


def load_kernels(radius, num_kpoints, num_kernels, dimension, fixed, *, seed=0, disposition=None):
    """:184-280 -- [num_kernels, num_kpoints, 3] float64: the disposition (computed, or given as [num_kpoints, 3] at
    radius 1) scaled by radius, rotated per kernel and, unless fixed is 'verticals', jittered by N(0, 0.01 radius)."""
    _check(dimension, fixed)
    if disposition is None:
        D = shared_disposition(num_kpoints, fixed, seed)
    else:
        D = np.asarray(disposition, dtype=np.float64)
        if D.shape != (num_kpoints, 3):
            raise ValueError("disposition must be [%d, 3], got %s" % (num_kpoints, list(D.shape)))
    d = radius * D
    out = np.empty((num_kernels, num_kpoints, 3))
    for n in range(num_kernels):
        if fixed == "verticals":
            theta = uniform(seed, THETA, np.arange(n, n + 1))[0] * 2 * np.pi
            c, s = np.float64(np.float32(np.cos(theta))), np.float64(np.float32(np.sin(theta)))   # R is float32 (:234)
            out[n] = _rotate(d, np.array([[c, s, 0.0], [-s, c, 0.0], [0.0, 0.0, 1.0]]))
        else:
            R, _ = rotation(seed, n)
            idx = np.uint64(n * num_kpoints * 3) + np.arange(num_kpoints * 3, dtype=np.uint64)
            out[n] = _rotate(d, R) + (radius * 0.01) * normal(seed, NOISE, idx).reshape(num_kpoints, 3)
    return out
