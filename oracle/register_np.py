"""numpy restatement of RANSAC registration of cloud pairs from keypoint correspondences (d3f_register_pairs).

This module is the contract. Every step is a correctly rounded float64 `+ - * / sqrt`, in the order written here,
elementwise over "lanes" (hypotheses, or pairs); sums are explicit loops in ascending index. No np.sum, `@` or linalg
on the contract path. The CUDA code performs the same operations with __dadd_rn / __dsub_rn / __dmul_rn / __ddiv_rn /
__dsqrt_rn, so it reproduces these results bit for bit. Inputs are fp32 points, widened to float64 exactly.

For pair p = (src, tgt) with n_c = clamp(n_corr[p], 0, L) real correspondence rows (source slot, target slot):
  * a pair naming a cloud outside [0, B), or a real row naming a slot outside [0, clamp(count[b], 0, k)), registers
    nothing (identity pose, 0 inliers, hypothesis -1, 0 validated); neither is ever read. So does a pair with n_c < n.
  * hypothesis h in [0, T) samples idx_m (m < n) by counter-based splitmix64 (sample_index); a sample with a repeated
    index is rejected; the edge-length checker, a Horn pose of the sample and the distance checker follow
    (Open3D's CorrespondenceCheckerBasedOnEdgeLength / OnDistance). Only the first V validated hypotheses in
    ascending h are scored.
  * a row is an inlier if d^2 = |R s + t - t'|^2 < tau^2 (strict). The best hypothesis has the most inliers, then the
    smaller sequential sum of inlier d^2, then the smaller h. Its pose is refit once over its inliers in ascending row
    order (a best hypothesis without inliers keeps its own pose).

Horn's quaternion method (J. Opt. Soc. Am. A 4(4), 1987): centroids (sequential sums, one division), the centred
cross-covariance H[a][b] = sum (s_a - cs_a)(t_b - ct_b), the 4x4 symmetric N, cyclic Jacobi with a fixed number of
sweeps, the eigenvector of the largest diagonal entry (ties to the lowest index), normalised, to R. A unit quaternion
always gives a proper rotation.
"""
import numpy as np

SWEEPS = 6
PIVOTS = ((0, 1), (0, 2), (0, 3), (1, 2), (1, 3), (2, 3))
LANES = 1 << 18          # hypotheses evaluated per numpy pass; the result does not depend on it

U = np.uint64


def splitmix64(z):
    """The splitmix64 finaliser (uint64, wrapping)."""
    z = (z ^ (z >> U(30))) * U(0xBF58476D1CE4E5B9)
    z = (z ^ (z >> U(27))) * U(0x94D049BB133111EB)
    return z ^ (z >> U(31))


def sample_index(p, h, m, n_c, seed):
    """idx_m of hypothesis h of pair p: c = ((p << 32) | h) * 8 + m, z = splitmix64(seed + c * golden),
    idx = ((z >> 32) * n_c) >> 32 -- all uint64, wrapping. p, h, n_c: int arrays."""
    c = ((p.astype(U) << U(32)) | h.astype(U)) * U(8) + U(m)
    z = splitmix64(U(seed) + c * U(0x9E3779B97F4A7C15))
    return (((z >> U(32)) * n_c.astype(U)) >> U(32)).astype(np.int64)


def length(a, b):
    d = [a[i] - b[i] for i in range(3)]
    return np.sqrt((d[0] * d[0] + d[1] * d[1]) + d[2] * d[2])


def edge_ok(S, T, ratio):
    """Open3D's edge-length checker over every a < b of the sample: fails if ls < ratio * lt or lt < ratio * ls."""
    ok = np.ones(S[0][0].shape, bool)
    for a in range(len(S)):
        for b in range(a + 1, len(S)):
            ls, lt = length(S[a], S[b]), length(T[a], T[b])
            ok &= ~((ls < ratio * lt) | (lt < ratio * ls))
    return ok


def residual2(R, t, s, tt):
    """d^2 = |R s + t - t'|^2: e_a = (((R_a0 s_0 + R_a1 s_1) + R_a2 s_2) + t_a) - t'_a, d^2 = (e_0^2 + e_1^2) + e_2^2."""
    e = [(((R[a][0] * s[0] + R[a][1] * s[1]) + R[a][2] * s[2]) + t[a]) - tt[a] for a in range(3)]
    return (e[0] * e[0] + e[1] * e[1]) + e[2] * e[2]


def pose_from_moments(cs, ct, H):
    """Horn: N from the cross-covariance, cyclic Jacobi, the quaternion of the largest eigenvalue, R and t."""
    (Sxx, Sxy, Sxz), (Syx, Syy, Syz), (Szx, Szy, Szz) = H
    a = [[(Sxx + Syy) + Szz, Syz - Szy, Szx - Sxz, Sxy - Syx],
         [None, (Sxx - Syy) - Szz, Sxy + Syx, Szx + Sxz],
         [None, None, (Syy - Sxx) - Szz, Syz + Szy],
         [None, None, None, (Szz - Sxx) - Syy]]
    for i in range(4):
        for j in range(i):
            a[i][j] = a[j][i]
    one, zero = np.ones_like(a[0][0]), np.zeros_like(a[0][0])
    v = [[one if i == j else zero for j in range(4)] for i in range(4)]
    for _ in range(SWEEPS):
        for p, q in PIVOTS:
            apq = a[p][q]
            rot = apq != 0.0                    # the exact-zero skip rule: an exactly zero pivot is left alone
            theta = (a[q][q] - a[p][p]) / (2.0 * apq)
            t = np.where(theta >= 0.0, 1.0, -1.0) / (np.abs(theta) + np.sqrt(theta * theta + 1.0))
            c = 1.0 / np.sqrt(t * t + 1.0)
            s = t * c
            tap = t * apq
            new = {(p, p): a[p][p] - tap, (q, q): a[q][q] + tap, (p, q): zero}
            for r in range(4):
                if r != p and r != q:
                    new[(r, p)] = c * a[r][p] - s * a[r][q]
                    new[(r, q)] = s * a[r][p] + c * a[r][q]
            for (i, j), x in new.items():
                a[i][j] = a[j][i] = np.where(rot, x, a[i][j])
            for r in range(4):
                vp = c * v[r][p] - s * v[r][q]
                vq = s * v[r][p] + c * v[r][q]
                v[r][p], v[r][q] = np.where(rot, vp, v[r][p]), np.where(rot, vq, v[r][q])
    best, dbest = np.zeros(one.shape, np.int64), a[0][0]
    for i in range(1, 4):                       # largest diagonal entry, ties to the lowest index
        take = a[i][i] > dbest
        best, dbest = np.where(take, i, best), np.where(take, a[i][i], dbest)
    q = [np.choose(best, [v[r][0], v[r][1], v[r][2], v[r][3]]) for r in range(4)]
    nrm = np.sqrt(((q[0] * q[0] + q[1] * q[1]) + q[2] * q[2]) + q[3] * q[3])
    w, x, y, z = (qi / nrm for qi in q)
    R = [[((w * w + x * x) - y * y) - z * z, 2.0 * (x * y - w * z), 2.0 * (x * z + w * y)],
         [2.0 * (x * y + w * z), ((w * w - x * x) + y * y) - z * z, 2.0 * (y * z - w * x)],
         [2.0 * (x * z - w * y), 2.0 * (y * z + w * x), ((w * w - x * x) - y * y) + z * z]]
    t = [ct[i] - ((R[i][0] * cs[0] + R[i][1] * cs[1]) + R[i][2] * cs[2]) for i in range(3)]
    return R, t


def horn(rows, m):
    """Pose t' ~ R s + t over `rows` = [(s, t', use)] in order (s, t': 3 coordinate arrays over lanes; use: bool array
    of the lanes whose sums take the row, None for all). m: rows used per lane (float64 array)."""
    with np.errstate(all="ignore"):       # NaN / inf points and exactly-zero pivots are part of the contract
        return _horn(rows, m)


def _horn(rows, m):
    zero = np.zeros(np.shape(m))
    ss, st = [zero] * 3, [zero] * 3
    for s, tt, use in rows:
        for i in range(3):
            ss[i] = ss[i] + s[i] if use is None else np.where(use, ss[i] + s[i], ss[i])
            st[i] = st[i] + tt[i] if use is None else np.where(use, st[i] + tt[i], st[i])
    cs, ct = [x / m for x in ss], [x / m for x in st]
    H = [[zero] * 3 for _ in range(3)]
    for s, tt, use in rows:
        ds, dt = [s[i] - cs[i] for i in range(3)], [tt[i] - ct[i] for i in range(3)]
        for i in range(3):
            for j in range(3):
                H[i][j] = H[i][j] + ds[i] * dt[j] if use is None else np.where(use, H[i][j] + ds[i] * dt[j], H[i][j])
    return pose_from_moments(cs, ct, H)


def is_inlier(d2, tau2):
    return d2 < tau2


def first_validated(hs, V):
    """hs: validated hypotheses in ascending h (at least the first V of them). The scored ones: the first V."""
    return hs[:V]


def pick_best(cnt, sums, hs):
    """Index of the best scored hypothesis: most inliers, then the smaller sum of inlier d^2, then the smaller h."""
    return int(np.lexsort((hs, sums, -cnt))[0])


def refit(R, t, rows, m):
    """The result pose: Horn over the inlier rows in ascending order; a lane without inliers keeps (R, t)."""
    R2, t2 = horn(rows, np.maximum(m, 1.0))
    keep = m == 0
    return [[np.where(keep, R[i][j], R2[i][j]) for j in range(3)] for i in range(3)], \
           [np.where(keep, t[i], t2[i]) for i in range(3)]


class _Rows:
    """The real correspondence rows of every active pair, concatenated: coordinates S[i], T[i] (float64)."""

    def __init__(self, points, corr, pairs, n_c, active):
        self.off = {}
        s, t, off = [], [], 0
        for p in active:
            src, tgt = pairs[p]
            self.off[p] = off
            s.append(points[src, corr[p, :n_c[p], 0]])
            t.append(points[tgt, corr[p, :n_c[p], 1]])
            off += n_c[p]
        s = np.concatenate(s).astype(np.float64) if s else np.zeros((0, 3))
        t = np.concatenate(t).astype(np.float64) if t else np.zeros((0, 3))
        self.S, self.T = [s[:, i] for i in range(3)], [t[:, i] for i in range(3)]

    def at(self, row):
        return [x[row] for x in self.S], [x[row] for x in self.T]


def hypotheses(rows, pp, hh, off, nc, n, tau2, ratio, seed):
    """Validation flag and sample pose of hypotheses (pp[e], hh[e]); off / nc: each lane's row offset and n_c."""
    idx = [sample_index(pp, hh, m, nc, seed) for m in range(n)]
    ok = np.ones(pp.shape, bool)
    for a in range(n):
        for b in range(a + 1, n):
            ok &= idx[a] != idx[b]
    smp = [rows.at(off + idx[m]) for m in range(n)]
    S, T = [s for s, _ in smp], [t for _, t in smp]
    ok &= edge_ok(S, T, ratio)
    R, t = horn([(S[m], T[m], None) for m in range(n)], np.full(pp.shape, float(n)))
    for m in range(n):
        ok &= residual2(R, t, S[m], T[m]) <= tau2
    return ok, R, t


def register(points, count, corr, n_corr, pairs, *, distance=0.05, ransac_n=3, edge_ratio=0.9, max_iterations=50000,
             max_validation=1000, seed=0):
    """dict(pose [P,4,4] float64, n_inliers, hypothesis, n_validated [P] int32) of every pair.
    points [B,k,3] float32, count [B], corr [P,L,2] (source slot, target slot), n_corr [P], pairs [P,2]."""
    points = np.asarray(points, np.float32)
    B, k, _ = points.shape
    pairs = np.asarray(pairs, np.int64).reshape(-1, 2)
    P = pairs.shape[0]
    corr = np.asarray(corr, np.int64).reshape(P, -1, 2)
    L = corr.shape[1]
    n_c = np.clip(np.asarray(n_corr, np.int64), 0, L)
    cnt = np.clip(np.asarray(count, np.int64), 0, k)
    n, T, V = int(ransac_n), int(max_iterations), int(max_validation)
    tau2, ratio = float(distance) * float(distance), float(edge_ratio)
    out = dict(pose=np.tile(np.eye(4), (P, 1, 1)), n_inliers=np.zeros(P, np.int32),
               hypothesis=np.full(P, -1, np.int32), n_validated=np.zeros(P, np.int32))
    active = []
    for p, (src, tgt) in enumerate(pairs):
        if not (0 <= src < B and 0 <= tgt < B):
            continue
        c = corr[p, :n_c[p]]
        if ((c[:, 0] < 0) | (c[:, 0] >= cnt[src]) | (c[:, 1] < 0) | (c[:, 1] >= cnt[tgt])).any():
            continue
        if n_c[p] >= n:
            active.append(p)
    with np.errstate(all="ignore"):
        rows = _Rows(points, corr, pairs, n_c, active)
        # hypotheses in ascending h, a round at a time, until every pair has V validated or h reaches T
        valid = {p: [] for p in active}
        live, h0 = list(active), 0
        while live and h0 < T:
            h1 = min(T, h0 + max(32, LANES // len(live)))
            hh = np.tile(np.arange(h0, h1, dtype=np.int64), len(live))
            pp = np.repeat(np.array(live, np.int64), h1 - h0)
            off = np.array([rows.off[p] for p in live], np.int64).repeat(h1 - h0)
            ok, _, _ = hypotheses(rows, pp, hh, off, n_c[pp], n, tau2, ratio, seed)
            ok = ok.reshape(len(live), h1 - h0)
            for i, p in enumerate(live):
                valid[p].extend((h0 + np.nonzero(ok[i])[0]).tolist())
            live = [p for p in live if len(valid[p]) < V]
            h0 = h1
        sel = {p: np.asarray(first_validated(np.asarray(valid[p], np.int64), V), np.int64) for p in active}
        scored = [p for p in active if len(sel[p])]
        for p in active:
            out["n_validated"][p] = len(sel[p])
        if not scored:
            return out
        # score every selected hypothesis over the pair's rows in ascending order
        pp = np.concatenate([np.full(len(sel[p]), p) for p in scored])
        hh = np.concatenate([sel[p] for p in scored])
        off = np.array([rows.off[p] for p in pp.tolist()])
        nc = n_c[pp]
        _, R, t = hypotheses(rows, pp, hh, off, nc, n, tau2, ratio, seed)
        inl_n, sums = np.zeros(pp.shape, np.int64), np.zeros(pp.shape)
        for r in range(int(nc.max())):
            real = r < nc
            s, tt = rows.at(off + np.minimum(r, nc - 1))
            d2 = residual2(R, t, s, tt)
            inl = real & is_inlier(d2, tau2)
            inl_n += inl
            sums = np.where(inl, sums + d2, sums)
        best = []
        for p in scored:
            e = np.nonzero(pp == p)[0]
            best.append(e[pick_best(inl_n[e], sums[e], hh[e])])
        best = np.array(best)
        # refit each pair's best over its inliers, rows ascending
        Rb = [[x[best] for x in Ri] for Ri in R]
        tb = [x[best] for x in t]
        offb, ncb = off[best], nc[best]
        rws, m = [], np.zeros(len(best))
        for r in range(int(ncb.max())):
            s, tt = rows.at(offb + np.minimum(r, ncb - 1))
            use = (r < ncb) & is_inlier(residual2(Rb, tb, s, tt), tau2)
            m = m + use
            rws.append((s, tt, use))
        Rf, tf = refit(Rb, tb, rws, m)
        for i, p in enumerate(scored):
            out["pose"][p, :3, :3] = [[Rf[a][b][i] for b in range(3)] for a in range(3)]
            out["pose"][p, :3, 3] = [tf[a][i] for a in range(3)]
            out["n_inliers"][p] = inl_n[best[i]]
            out["hypothesis"][p] = hh[best[i]]
    return out
