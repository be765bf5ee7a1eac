"""numpy restatement of point-to-point ICP over stacked clouds (d3f_icp_pairs).

This module is the contract. Every step is a correctly rounded float64 `+ - * / sqrt`, in the order written here,
elementwise over the rows of one pair; sums are explicit loops in the blocked order below. No np.sum, `@` or linalg on
the contract path. The Horn solve is register_np.pose_from_moments and d^2 is register_np.residual2, shared with
RANSAC; the CUDA code (csrc/icp.cu, csrc/solver.cuh) performs the same operations with __dadd_rn / __dsub_rn /
__dmul_rn / __ddiv_rn / __dsqrt_rn, so it reproduces these results bit for bit. Points are fp32, widened exactly.

Clouds: `points` [N,3] stacked, cloud b holds rows [start[b], start[b+1]) of the lengths' exclusive scan, cut at the
row count min(rows, start[B]) (DESIGN.md section 2, "Rows and clouds"). A pair naming a cloud outside [0, B), or with
an empty source or target, keeps init with 0 correspondences and 0 iterations.

Pair p = (src, tgt), pose T_0 = init[p] (rows 0-2: R | t). Evaluation i of pose T_i = (R, t):
  * every source row s becomes q_a = ((R_a0 s_0 + R_a1 s_1) + R_a2 s_2) + t_a (residual2's order);
  * its correspondence is the target row j with the smallest d^2 = |q - t_j|^2 (residual2's order) among the rows with
    d^2 < tau^2 (strict, tau^2 = tau * tau), ties to the smaller row; a NaN d^2 never corresponds;
  * over the n corresponding rows, in ascending source row, in blocks of BLOCK consecutive source rows (counted from
    the cloud's first row) each summed sequentially from 0.0, then the block sums sequentially from 0.0 in ascending
    block order: the centroids cq = sum q / n, ct = sum t_j / n, then the centred cross-covariance
    H_ab = sum (q_a - cq_a)(t_b - ct_b), then sum d^2;
  * fitness = n / n_src, inlier_rmse = sqrt(sum d^2 / n), or 0 when n = 0 (Open3D's RegistrationResult);
  * the pair stops after evaluation i > 0 when |fitness_i - fitness_{i-1}| < relative_fitness and
    |rmse_i - rmse_{i-1}| < relative_rmse (Open3D's ICPConvergenceCriteria), when n < 3 (the pose is kept), or when
    i = max_iterations; otherwise U = Horn(q, t_j) and T_{i+1} = U T_i: R' = ((U_a0 R_0b + U_a1 R_1b) + U_a2 R_2b),
    t' = (((U_a0 t_0 + U_a1 t_1) + U_a2 t_2) + u_a). The pose is re-applied to the fp32 points every evaluation (Open3D
    transforms its double-precision copy in place: the one stated deviation).
Outputs, for the final pose: pose [P,4,4] (rows 0-2 of T, row 3 of init), fitness, inlier_rmse, n_correspondences and
iterations (the number of updates).

The nearest-row search proposes candidates with scipy's cKDTree (any row within the tree's nearest distance, widened
by 1e-9 relative, a superset of the rows that can tie under the contract's rounding); the choice among them is the
contract's d^2 and tie rule.
"""
import numpy as np

from . import register_np

BLOCK = 256
IDENTITY = [[1.0, 0.0, 0.0], [0.0, 1.0, 0.0], [0.0, 0.0, 1.0]]


def transform(R, t, s):
    """q_a = ((R_a0 s_0 + R_a1 s_1) + R_a2 s_2) + t_a, over the rows of s (3 coordinate arrays)."""
    return [((R[a][0] * s[0] + R[a][1] * s[1]) + R[a][2] * s[2]) + t[a] for a in range(3)]


def dist2(q, tt):
    """|q - t|^2 evaluated as register_np.residual2: q is the transformed point, so the pose is the identity (1 * q_a and
    0 * q_b are exact for finite q; non-finite q never reach here)."""
    return register_np.residual2(IDENTITY, [0.0, 0.0, 0.0], q, tt)


def corresponds(d2, tau2):
    return d2 < tau2


def pick_nearest(qi, row, d2):
    """Index into the candidate arrays of each query's correspondence: the smallest d^2, ties to the smaller row."""
    order = np.lexsort((row, d2, qi))
    first = np.ones(len(order), bool)
    first[1:] = qi[order][1:] != qi[order][:-1]
    return order[first]


def blocked_sum(x, use):
    """Sums of the rows of x [m, n] where use [n]: blocks of BLOCK consecutive rows each summed sequentially from 0.0,
    then the block sums sequentially from 0.0 in ascending block order. Returns [m]."""
    m, n = x.shape
    nb = -(-n // BLOCK)
    X = np.zeros((m, nb * BLOCK))
    U = np.zeros(nb * BLOCK, bool)
    X[:, :n], U[:n] = x, use
    X, U = X.reshape(m, nb, BLOCK), U.reshape(nb, BLOCK)
    acc = np.zeros((m, nb))
    for i in range(BLOCK):
        acc = np.where(U[:, i], acc + X[:, :, i], acc)
    total = np.zeros(m)
    for k in range(nb):
        total = total + acc[:, k]
    return total


def next_queries(s, R, t, U, q_prev):
    """The queries of the next evaluation: the new pose applied to the fp32 source points."""
    return transform(R, t, s)


def converged(fit, prev_fit, rmse, prev_rmse, relative_fitness, relative_rmse):
    return abs(fit - prev_fit) < relative_fitness and abs(rmse - prev_rmse) < relative_rmse


def correspond(q, tgt, tgt_lo, tau2, tree):
    """(j [n] global target row or -1, d2 [n]) of the queries q (3 arrays). tree: (cKDTree over the finite target rows,
    their rows), or None."""
    n = q[0].shape[0]
    j, d2 = np.full(n, -1, np.int64), np.zeros(n)
    fin = np.isfinite(q[0]) & np.isfinite(q[1]) & np.isfinite(q[2])
    if tree is None or not fin.any():
        return j, d2
    tree, tree_rows = tree
    live = np.nonzero(fin)[0]
    Q = np.stack([q[a][live] for a in range(3)], 1)
    tau = float(np.sqrt(tau2))
    d1, _ = tree.query(Q, k=1, distance_upper_bound=tau * (1 + 1e-9) + 1e-300)
    has = np.isfinite(d1)
    live, Q, d1 = live[has], Q[has], d1[has]
    if len(live) == 0:
        return j, d2
    cands = tree.query_ball_point(Q, r=d1 * (1 + 1e-9) + 1e-300, return_sorted=False)
    cnt = np.fromiter((len(c) for c in cands), np.int64, len(cands))
    local = np.fromiter((x for c in cands for x in c), np.int64, int(cnt.sum()))
    qi = np.repeat(np.arange(len(live)), cnt)
    rows = tree_rows[local]
    dd = dist2([Q[qi, a] for a in range(3)], [tgt[rows, a] for a in range(3)])
    ok = corresponds(dd, tau2)
    qi, rows, dd = qi[ok], rows[ok], dd[ok]
    pick = pick_nearest(qi, rows, dd)
    j[live[qi[pick]]] = rows[pick] + tgt_lo
    d2[live[qi[pick]]] = dd[pick]
    return j, d2


def _target_tree(tgt):
    from scipy.spatial import cKDTree
    fin = np.isfinite(tgt).all(1)
    if not fin.any():
        return None
    return cKDTree(tgt[fin]), np.nonzero(fin)[0]


def _pose(init):
    return [[float(init[a, b]) for b in range(3)] for a in range(3)], [float(init[a, 3]) for a in range(3)]


def icp_pair(points, src_lo, n_src, tgt_lo, n_tgt, init, tau2, I, relative_fitness, relative_rmse):
    """(R, t, fitness, inlier_rmse, n, iterations) of one pair with real clouds."""
    s = [points[src_lo:src_lo + n_src, a].astype(np.float64) for a in range(3)]
    tgt = points[tgt_lo:tgt_lo + n_tgt].astype(np.float64)
    tree = _target_tree(tgt)
    R, t = _pose(init)
    q = transform(R, t, s)
    prev = None
    for i in range(I + 1):
        j, d2 = correspond(q, tgt, tgt_lo, tau2, tree)
        use = j >= 0
        n = int(use.sum())
        tj = [np.where(use, points[np.maximum(j, 0), a].astype(np.float64), 0.0) for a in range(3)]
        m = float(n)
        sums = blocked_sum(np.stack(q + tj + [d2]), use)
        fit = m / float(n_src)
        rmse = float(np.sqrt(sums[6] / m)) if n > 0 else 0.0
        stop = (prev is not None and converged(fit, prev[0], rmse, prev[1], relative_fitness, relative_rmse)) \
            or i == I or n < 3
        if stop:
            return R, t, fit, rmse, n, i
        cq, ct = [sums[a] / m for a in range(3)], [sums[3 + a] / m for a in range(3)]
        ds, dt = [q[a] - cq[a] for a in range(3)], [tj[b] - ct[b] for b in range(3)]
        H = blocked_sum(np.stack([ds[a] * dt[b] for a in range(3) for b in range(3)]), use)
        with np.errstate(all="ignore"):
            Ru, tu = register_np.pose_from_moments([np.array([x]) for x in cq], [np.array([x]) for x in ct],
                                                   [[np.array([H[3 * a + b]]) for b in range(3)] for a in range(3)])
        Ru = [[float(Ru[a][b][0]) for b in range(3)] for a in range(3)]
        tu = [float(tu[a][0]) for a in range(3)]
        R = [[(Ru[a][0] * R[0][b] + Ru[a][1] * R[1][b]) + Ru[a][2] * R[2][b] for b in range(3)] for a in range(3)]
        t = [((Ru[a][0] * t[0] + Ru[a][1] * t[1]) + Ru[a][2] * t[2]) + tu[a] for a in range(3)]
        q = next_queries(s, R, t, (Ru, tu), q)
        prev = (fit, rmse)
    raise AssertionError("unreachable")


def cloud_ranges(lengths, N, rows=None):
    """(lo [B], n [B]) of every cloud: the lengths' exclusive scan cut at min(rows, start[B])."""
    lengths = np.asarray(lengths, np.int64)
    start = np.concatenate([[0], np.cumsum(lengths)])
    n_rows = N if rows is None else min(max(int(rows), 0), N)
    n_rows = min(n_rows, max(int(start[-1]), 0))
    lo = np.clip(start[:-1], 0, n_rows)
    hi = np.clip(start[1:], 0, n_rows)
    return lo, np.maximum(hi - lo, 0)


def icp(points, lengths, pairs, init, *, distance, max_iterations=30, relative_fitness=1e-6, relative_rmse=1e-6,
        rows=None):
    """dict(pose [P,4,4] float64, fitness, inlier_rmse [P] float64, n_correspondences, iterations [P] int32).
    points [N,3] float32, lengths [B], pairs [P,2], init [P,4,4] float64, rows: the row count (default N)."""
    points = np.asarray(points, np.float32).reshape(-1, 3)
    N = points.shape[0]
    lo, n = cloud_ranges(lengths, N, rows)
    B = len(lo)
    pairs = np.asarray(pairs, np.int64).reshape(-1, 2)
    P = pairs.shape[0]
    init = np.asarray(init, np.float64).reshape(P, 4, 4)
    tau2 = float(distance) * float(distance)
    out = dict(pose=init.copy(), fitness=np.zeros(P), inlier_rmse=np.zeros(P), n_correspondences=np.zeros(P, np.int32),
               iterations=np.zeros(P, np.int32))
    with np.errstate(all="ignore"):
        for p, (src, tgt) in enumerate(pairs):
            if not (0 <= src < B and 0 <= tgt < B) or n[src] == 0 or n[tgt] == 0:
                continue
            R, t, fit, rmse, nc, it = icp_pair(points, int(lo[src]), int(n[src]), int(lo[tgt]), int(n[tgt]), init[p],
                                               tau2, int(max_iterations), float(relative_fitness),
                                               float(relative_rmse))
            out["pose"][p, :3, :3] = R
            out["pose"][p, :3, 3] = t
            out["fitness"][p], out["inlier_rmse"][p] = fit, rmse
            out["n_correspondences"][p], out["iterations"][p] = nc, it
    return out
