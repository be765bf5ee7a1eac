"""float64 numpy restatement of the kernel-point optimiser and of load_kernels (kernels/kernel_points.py:41-181 and
:184-280), the contract of csrc/kernel_points.cu and d3feat_b200/kernel_points.py.

It takes the initial points as input (the draw of :76-91 is the caller's), and it fixes every summation order, so the
kernel can be compared with it bit for bit:
  d2[i, j]  = ((dx*dx + dy*dy) + dz*dz), d = p_i - p_j                          :112 (np.sum over 3 is sequential)
  den[i, j] = d2 * sqrt(d2) + 1e-6                                              :113, with d2^(3/2) as d2 * sqrt(d2):
              the one deviation (neither numpy's nor CUDA's pow is correctly rounded)
  inter[j]  = sum over i = 0, 1, ..., K-1 in that order of (p_i - p_j) / den     :113-114 (np.sum over axis 1)
  g[j]      = inter[j] + 10 * p_j                                               :117-120
  norm[j]   = sqrt(((gx*gx + gy*gy) + gz*gz) + 1e-12)                           :129
Each operation is one IEEE fp64 operation, without fused multiply-add.

The reference fails on an empty maximum (K = 1 with 'center', K <= 3 with 'verticals': no point moves). Here no
iteration runs: the points stay as given and saved_gradient_norms stays zero.
"""
import numpy as np

MAX_ITER = 10000                 # :104
THRESH = 1e-5                    # :67
CLIP = 0.05                      # :70, clip = 0.05 * radius0
MOVING_FACTOR = 1e-2             # :63
MOVING_DECAY = 0.9995            # :64
FIXED = ("none", "center", "verticals")


def first_moving(fixed, K):
    """The first point the stop test looks at (:134-139): 1 for 'center', 3 for 'verticals', 0 for 'none'."""
    if fixed not in FIXED:
        raise ValueError("fixed must be one of %s, got %r" % (FIXED, fixed))
    return {"none": 0, "center": 1, "verticals": 3}[fixed]


def fix_points(points, fixed):
    """:85-91 on a copy of points [T, K, 3]."""
    p = np.array(points, dtype=np.float64, copy=True)
    if fixed == "center":
        p[:, 0, :] *= 0
    if fixed == "verticals":
        p[:, :3, :] *= 0
        p[:, 1:2, -1] += 2 * 1 / 3                  # K < 3: the points that exist
        p[:, 2:3, -1] -= 2 * 1 / 3
    return p


def gradients(p, fixed):
    """:109-129 for points p [T, K, 3] -> (gradients [T, K, 3], norms [T, K])."""
    K = p.shape[1]
    A = p[:, :, None, :]                     # A[t, i, j] = p_i   (:110)
    B = p[:, None, :, :]                     # B[t, i, j] = p_j   (:111)
    d = A - B
    sq = d * d
    d2 = (sq[..., 0] + sq[..., 1]) + sq[..., 2]
    den = d2 * np.sqrt(d2) + 1e-6
    q = d / den[..., None]
    inter = q[:, 0].copy()
    for i in range(1, K):
        inter = inter + q[:, i]
    g = inter + 10 * p
    if fixed == "verticals":
        g[:, 1:3, :-1] = 0                   # :122-123
    gg = g * g
    norms = np.sqrt(((gg[..., 0] + gg[..., 1]) + gg[..., 2]) + 1e-12)
    return g, norms


def optimize(initial, fixed="center"):
    """:102-174 from initial points [T, K, 3] (already fixed by :85-91) -> (points [T, K, 3] before the rescale of
    :176-178, saved_gradient_norms [10000, T], iterations: the number of rows of saved_gradient_norms written)."""
    p = np.array(initial, dtype=np.float64, copy=True)
    T, K, _ = p.shape
    m0 = first_moving(fixed, K)
    saved = np.zeros((MAX_ITER, T))
    if K <= m0:
        return p, saved, 0
    old = np.zeros((T, K))
    mf = MOVING_FACTOR
    for it in range(MAX_ITER):
        g, norms = gradients(p, fixed)
        saved[it, :] = np.max(norms, axis=1)                      # :130
        if np.max(np.abs(old[:, m0:] - norms[:, m0:])) < THRESH:  # :134-139
            return p, saved, it + 1
        old = norms                                               # :140
        moving = np.minimum(mf * norms, CLIP)                     # :146
        if fixed in ("center", "verticals"):
            moving[:, 0] = 0                                      # :149-152
        p = p - (moving[..., None] * g) / (norms + 1e-6)[..., None]   # :155
        mf *= MOVING_DECAY                                        # :174
    return p, saved, MAX_ITER


def rescale(points, ratio=1.0):
    """:177-178: points * (ratio / mean of |p| over every try's points 1..K-1), |p| = sqrt(((x*x + y*y) + z*z) + 1e-12)
    and the mean summed sequentially in (try, point) order. Unchanged when there is no such point (K = 1)."""
    p = np.asarray(points, dtype=np.float64)
    if p.shape[1] < 2:
        return p.copy()
    sq = p * p
    r = np.sqrt(((sq[..., 0] + sq[..., 1]) + sq[..., 2]) + 1e-12)[:, 1:]
    s = 0.0
    for x in r.ravel():
        s += x
    return p * (ratio / (s / r.size))


def kernel_point_optimization_debug(radius, initial, fixed="center", ratio=1.0):
    """:41-181 from given initial points [T, K, 3] (drawn by :76-83, not yet fixed) -> (points [T, K, 3] * radius,
    saved_gradient_norms [10000, T], iterations)."""
    p, saved, n = optimize(fix_points(initial, fixed), fixed)
    return rescale(p, ratio) * radius, saved, n


def best_try(saved_gradient_norms):
    """:214 -- argmin of the last row. That row is zero whenever the loop stopped before 10000 iterations, so the
    reference then keeps try 0."""
    return int(np.argmin(saved_gradient_norms[-1, :]))


def unit(x):
    """:255, :258, :264 -- x / (|x| + 1e-9), |x| = sqrt((x0*x0 + x1*x1) + x2*x2), per row."""
    x = np.asarray(x, dtype=np.float64)
    sq = x * x
    return x / (np.sqrt((sq[:, 0] + sq[:, 1]) + sq[:, 2]) + 1e-9)[:, None]


def dot(a, b):
    ab = a * b
    return (ab[:, 0] + ab[:, 1]) + ab[:, 2]


def rotation(u_draws, v_draws):
    """:250-268 for one kernel from its sequence of draws on [-1, 1)^3 (rows, in draw order): the first pair (u, v)
    with |u.v| <= 0.99 after normalisation, v made orthogonal to u and normalised, w = u x v, R = [u v w] as columns."""
    u, v = unit(u_draws), unit(v_draws)
    ok = np.nonzero(np.abs(dot(u, v)) <= 0.99)[0]
    if ok.size == 0:
        raise ValueError("no draw pair with |u.v| <= 0.99")
    u, v = u[ok[0]:ok[0] + 1], v[ok[0]:ok[0] + 1]
    v = unit(v - dot(u, v)[:, None] * u)
    w = np.stack([u[:, 1] * v[:, 2] - u[:, 2] * v[:, 1],
                  u[:, 2] * v[:, 0] - u[:, 0] * v[:, 2],
                  u[:, 0] * v[:, 1] - u[:, 1] * v[:, 0]], -1)
    return np.stack((u[0], v[0], w[0]), axis=-1)


def vertical_rotation(theta):
    """:232-239 -- rotation by theta about z, R[0, 1] = sin, R[1, 0] = -sin; R is float32 there (:234), so cos and sin
    are rounded to float32 (the matmul with the float64 kernel then runs in float64)."""
    c, s = float(np.float32(np.cos(theta))), float(np.float32(np.sin(theta)))
    return np.array([[c, s, 0.0], [-s, c, 0.0], [0.0, 0.0, 1.0]])


def rotate(disposition, radius, R, noise=None):
    """:241-245 / :270-278 -- (radius * disposition) @ R (+ noise), each output sum sequential over the 3 inputs."""
    d = radius * np.asarray(disposition, dtype=np.float64)
    out = (d[:, 0:1] * R[0] + d[:, 1:2] * R[1]) + d[:, 2:3] * R[2]
    return out if noise is None else out + noise
