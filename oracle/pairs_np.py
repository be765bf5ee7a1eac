"""numpy restatement of the training-pair ops (d3f_pair_correspondences_*, d3f_sample_correspondences,
d3f_augment_pairs; d3feat_b200/training_data.py).

This module is the contract. Every step is a correctly rounded float64 `+ - *` in the order written here, elementwise;
points are fp32, widened exactly. csrc/correspond.cu performs the same operations with __dadd_rn / __dsub_rn /
__dmul_rn, so it reproduces these results bit for bit. The one exception is the fp64 cos / sin of the rotation angle:
the GPU's are not correctly rounded, so R is compared bit for bit only where `ambiguous_rotation` is False, and the
points are compared given the GPU's own R.

Clouds: `points` [N,3] stacked, cloud b holds rows [start[b], start[b+1]) of the lengths' exclusive scan, cut at the row
count (icp_np.cloud_ranges). pairs [P,2] = (anchor cloud, positive cloud); a pair naming a cloud outside [0, B) has no
rows on either side. trans [P,4,4] maps anchor points onto the positive.

Correspondences of pair p: anchor row s becomes q_a = ((R_a0 s_0 + R_a1 s_1) + R_a2 s_2) + t_a (icp_np.transform);
d^2 = ((e_0^2 + e_1^2) + e_2^2), e_a = q_a - t_a, against every positive row t (icp_np.dist2); tau2 = tau * tau.
  mode "radius": every positive row with d^2 < tau2 (strict), KITTI's get_matching_indices (nanoflann's radius test on
  Open3D's squared radius); mode "nearest": the positive row with the smallest d^2 < tau2, ties to the smaller row
  (cal_overlap.py's BFMatcher with distance < voxel size). A non-finite q matches nothing. rows are cloud-local
  (anchor row, positive row), ascending per pair; overlap = count / anchor rows (0 for an empty anchor).

Counters: draw(seed, p, i, slot) = splitmix64(seed + c * GOLDEN), c = (p << 36) | (i << 4) | slot (uint64, wrapping);
u = (z >> 11) * 2^-53. The SLOT_* constants below name each purpose; side 0 is the anchor, 1 the positive.

Sampling of pair p with n candidates: valid = n >= max(min_count, 1) and, without replacement, n >= k. With
replacement draw m is ((z >> 32) * n) >> 32 of draw(seed, p, m, SLOT_DRAW) (RANSAC's index map); without, candidate c
gets key draw(seed, p, c, SLOT_KEY) >> 32 and the sample is the k candidates with the smallest (key, c), in that order.
anc = the anchor row, pos = the positive row + the anchor's length; -1 for an invalid pair.

Augmentation of side s of pair p, each fp32 row x widened to fp64 (cloud-local row i):
  x_a = x_a + u(SLOT_NOISE + 3 s + a, i) * noise                                (np.random.rand, not Gaussian)
  for each rotation r < num_axis: theta = (u(SLOT_ANGLE + s, r) * 2) * pi, axis = floor(u(SLOT_AXIS + s, 0) * 3) for
    num_axis 1 and r for 3; R = float32 [[c, -s, -s], [s, c, -s], [s, s, c]] of fp64 cos / sin, row and column `axis`
    those of the identity (the reference's rotate); x_j = ((x_0 R_0j + x_1 R_1j) + x_2 R_2j)   (p @ R, row vectors)
  KITTI (scale_shift): x_a = scale * x_a + shift_a, scale = lo + (hi - lo) u(SLOT_SCALE, 0) per pair,
    shift_a = -r + (r - -r) u(SLOT_SHIFT + s, a) per cloud (np.random.uniform's low + (high - low) u)
  then one rounding to fp32. KITTI's generator runs this chain on Open3D's fp64 points. 3DMatch's rounds to fp32 after
  the noise and multiplies by R in fp32 BLAS: a deviation of a few fp32 ulp, far below the noise amplitude.
backup points: fp32 of q = trans s for the anchor, the point itself for the positive.
"""
import numpy as np

from . import icp_np

GOLDEN = 0x9E3779B97F4A7C15
M64 = (1 << 64) - 1
SLOT_NOISE, SLOT_ANGLE, SLOT_AXIS, SLOT_SCALE, SLOT_SHIFT, SLOT_DRAW, SLOT_KEY = 0, 6, 8, 10, 11, 13, 14
MODES = ("radius", "nearest")


def splitmix64(z):
    z = np.asarray(z, np.uint64)
    with np.errstate(over="ignore"):
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        return z ^ (z >> np.uint64(31))


def draw(seed, p, i, slot):
    """z of counters (p, i, slot); p and i broadcast."""
    p = np.asarray(p, np.uint64)
    i = np.asarray(i, np.uint64)
    c = (p << np.uint64(36)) | (i << np.uint64(4)) | np.uint64(slot)
    with np.errstate(over="ignore"):
        return splitmix64(np.uint64(seed & M64) + c * np.uint64(GOLDEN))


def uniform(seed, p, i, slot):
    return (draw(seed, p, i, slot) >> np.uint64(11)).astype(np.float64) * 2.0 ** -53


def draw_index(z, n):
    """((z >> 32) * n) >> 32 (uint64)."""
    with np.errstate(over="ignore"):
        return ((np.asarray(z, np.uint64) >> np.uint64(32)) * np.uint64(n)) >> np.uint64(32)


def _pair_ranges(lengths, N, pairs):
    lo, n = icp_np.cloud_ranges(lengths, N)
    B = len(lo)
    pairs = np.asarray(pairs, np.int64).reshape(-1, 2)
    out = []
    for a, b in pairs:
        if 0 <= a < B and 0 <= b < B:
            out.append((int(lo[a]), int(n[a]), int(lo[b]), int(n[b])))
        else:
            out.append((0, 0, 0, 0))
    return out


def _candidates(q, tgt, tau, exhaustive):
    """(query index, target row) pairs that include every pair with d^2 < tau^2."""
    n_a, n_p = q.shape[0], tgt.shape[0]
    fin = np.isfinite(q).all(1)
    if exhaustive:
        qi, tj = np.nonzero(np.broadcast_to(fin[:, None], (n_a, n_p)))
        return qi, tj
    from scipy.spatial import cKDTree
    tf = np.nonzero(np.isfinite(tgt).all(1))[0]
    live = np.nonzero(fin)[0]
    if len(tf) == 0 or len(live) == 0:
        return np.zeros(0, np.int64), np.zeros(0, np.int64)
    tree = cKDTree(tgt[tf])
    lists = tree.query_ball_point(q[live], r=tau * (1 + 1e-6), return_sorted=False)
    cnt = np.fromiter((len(c) for c in lists), np.int64, len(lists))
    qi = np.repeat(live, cnt)
    tj = tf[np.fromiter((x for c in lists for x in c), np.int64, int(cnt.sum()))]
    return qi, tj


def correspondences(points, lengths, pairs, trans, distance, mode, exhaustive=None):
    """dict(offset [P+1] int64, rows [M,2] int32, count [P] int32, overlap [P] float64). exhaustive: test every (anchor,
    positive) pair (True), or take candidates from a cKDTree at tau (1 + 1e-6) (False; None: by size)."""
    assert mode in MODES
    points = np.asarray(points, np.float32).reshape(-1, 3)
    trans = np.asarray(trans, np.float64).reshape(-1, 4, 4)
    tau = float(distance)
    tau2 = tau * tau
    ranges = _pair_ranges(lengths, points.shape[0], pairs)
    rows, count, overlap = [], [], []
    with np.errstate(all="ignore"):
        for p, (a_lo, n_a, p_lo, n_p) in enumerate(ranges):
            s = points[a_lo:a_lo + n_a].astype(np.float64)
            tgt = points[p_lo:p_lo + n_p].astype(np.float64)
            R = [[float(trans[p, i, j]) for j in range(3)] for i in range(3)]
            t = [float(trans[p, i, 3]) for i in range(3)]
            q = np.stack(icp_np.transform(R, t, [s[:, 0], s[:, 1], s[:, 2]]), 1) if n_a else np.zeros((0, 3))
            ex = exhaustive if exhaustive is not None else n_a * n_p <= 4_000_000
            qi, tj = _candidates(q, tgt, tau, ex) if n_a and n_p else (np.zeros(0, np.int64),) * 2
            d2 = icp_np.dist2([q[qi, a] for a in range(3)], [tgt[tj, a] for a in range(3)])
            ok = d2 < tau2
            qi, tj, d2 = qi[ok], tj[ok], d2[ok]
            if mode == "nearest" and len(qi):
                pick = icp_np.pick_nearest(qi, tj, d2)
                qi, tj = qi[pick], tj[pick]
            order = np.lexsort((tj, qi))
            r = np.stack([qi[order], tj[order]], 1).astype(np.int32) if len(qi) else np.zeros((0, 2), np.int32)
            rows.append(r)
            count.append(len(r))
            overlap.append(len(r) / n_a if n_a else 0.0)
    offset = np.concatenate([[0], np.cumsum(count)]).astype(np.int64)
    return dict(offset=offset, rows=np.concatenate(rows) if rows else np.zeros((0, 2), np.int32),
                count=np.asarray(count, np.int32), overlap=np.asarray(overlap, np.float64))


def sample(offset, rows, anchor_len, k, replace, min_count, seed):
    """(anc [P,k] int32, pos [P,k] int32, valid [P] bool)."""
    offset = np.asarray(offset, np.int64)
    rows = np.asarray(rows, np.int64).reshape(-1, 2)
    P = len(offset) - 1
    anc, pos = np.full((P, k), -1, np.int32), np.full((P, k), -1, np.int32)
    valid = np.zeros(P, bool)
    for p in range(P):
        lo, hi = int(offset[p]), int(offset[p + 1])
        n = hi - lo
        ok = n >= max(min_count, 1) and (replace or n >= k)
        valid[p] = ok
        if not ok:
            continue
        if replace:
            c = draw_index(draw(seed, p, np.arange(k), SLOT_DRAW), n).astype(np.int64)
        else:
            cand = np.arange(n)
            key = draw(seed, p, cand, SLOT_KEY) >> np.uint64(32)
            c = np.lexsort((cand, key))[:k]
        anc[p] = rows[lo + c, 0]
        pos[p] = rows[lo + c, 1] + int(anchor_len[p])
    return anc, pos, valid


def rotation(theta, axis):
    """The reference's rotate() matrix for one angle and axis: float32 [3,3]."""
    c, s = np.cos(theta), np.sin(theta)
    R = np.array([[c, -s, -s], [s, c, -s], [s, s, c]], dtype=np.float32)
    R[:, axis] = 0
    R[axis, :] = 0
    R[axis, axis] = 1
    return R


def rotation_draws(seed, p, side, num_axis):
    """[(theta, axis)] of the rotations of one cloud."""
    out = []
    for r in range(num_axis):
        theta = (float(uniform(seed, p, r, SLOT_ANGLE + side)) * 2.0) * np.pi
        axis = int(float(uniform(seed, p, 0, SLOT_AXIS + side)) * 3.0) if num_axis == 1 else r
        out.append((theta, axis))
    return out


def ambiguous_rotation(theta, ulps=8):
    """Whether fp32(cos) or fp32(sin) of theta could change under an fp64 error of `ulps` ulp."""
    for f in (np.cos, np.sin):
        v = f(theta)
        d = ulps * np.spacing(abs(v))
        if np.float32(v - d) != np.float32(v + d):
            return True
    return False


def augment(points, lengths, pairs, trans, seed, noise, num_axis, scale=None, shift_range=None, R=None):
    """dict(points, backup_points [T,3] float32, lengths [P,2] int32, row_offset [P+1] int64, R [2P,num_axis,3,3]
    float32, scale [P], shift [2P,3] float64, ambiguous [2P] bool). scale = (lo, hi) and shift_range select KITTI's
    scale and shift. R: use these matrices (the GPU's) instead of the drawn ones."""
    points = np.asarray(points, np.float32).reshape(-1, 3)
    trans = np.asarray(trans, np.float64).reshape(-1, 4, 4)
    ranges = _pair_ranges(lengths, points.shape[0], pairs)
    P = len(ranges)
    kitti = scale is not None
    Rs = np.zeros((2 * P, num_axis, 3, 3), np.float32)
    amb = np.zeros(2 * P, bool)
    sc = np.ones(P)
    sh = np.zeros((2 * P, 3))
    out, backup, lens = [], [], np.zeros((P, 2), np.int32)
    for p, (a_lo, n_a, p_lo, n_p) in enumerate(ranges):
        lens[p] = (n_a, n_p)
        if kitti:
            lo, hi = float(scale[0]), float(scale[1])
            sc[p] = lo + (hi - lo) * float(uniform(seed, p, 0, SLOT_SCALE))
        for side, (c_lo, n) in enumerate(((a_lo, n_a), (p_lo, n_p))):
            for r, (theta, axis) in enumerate(rotation_draws(seed, p, side, num_axis)):
                Rs[2 * p + side, r] = rotation(theta, axis)
                amb[2 * p + side] |= ambiguous_rotation(theta)
            if kitti:
                rr = float(shift_range)
                for a in range(3):
                    sh[2 * p + side, a] = -rr + (rr - -rr) * float(uniform(seed, p, a, SLOT_SHIFT + side))
            Ruse = Rs[2 * p + side] if R is None else np.asarray(R, np.float32)[2 * p + side]
            x = points[c_lo:c_lo + n].astype(np.float64)
            i = np.arange(n)
            y = [x[:, a] + uniform(seed, p, i, SLOT_NOISE + 3 * side + a) * float(noise) for a in range(3)]
            for r in range(num_axis):
                M = Ruse[r].astype(np.float64)
                y = [(y[0] * M[0, j] + y[1] * M[1, j]) + y[2] * M[2, j] for j in range(3)]
            if kitti:
                y = [sc[p] * y[a] + sh[2 * p + side, a] for a in range(3)]
            out.append(np.stack(y, 1).astype(np.float32) if n else np.zeros((0, 3), np.float32))
            if side == 0 and n:
                Rt = [[float(trans[p, a, b]) for b in range(3)] for a in range(3)]
                t = [float(trans[p, a, 3]) for a in range(3)]
                backup.append(np.stack(icp_np.transform(Rt, t, [x[:, 0], x[:, 1], x[:, 2]]), 1).astype(np.float32))
            else:
                backup.append(x.astype(np.float32).reshape(-1, 3))
    row_offset = np.concatenate([[0], np.cumsum(lens.sum(1))]).astype(np.int64)
    cat = (lambda L: np.concatenate(L) if L else np.zeros((0, 3), np.float32))
    return dict(points=cat(out), backup_points=cat(backup), lengths=lens, row_offset=row_offset, R=Rs, scale=sc,
                shift=sh, ambiguous=amb)
