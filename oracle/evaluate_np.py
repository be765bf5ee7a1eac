"""numpy restatement of the ground-truth metrics of matched and registered cloud pairs (d3f_evaluate_pairs).

This module is the contract. Every step is one correctly rounded float64 `+ - * / sqrt` in the order written here,
elementwise over pairs or slots; sums are explicit sequential loops. No np.sum, `@` or linalg on the contract path, so
no BLAS and no fused multiply-add. The CUDA code (csrc/evaluation.cu) performs the same operations with __dadd_rn /
__dsub_rn / __dmul_rn / __ddiv_rn / __dsqrt_rn and reproduces every value bit for bit, except rre_deg and its sum:
they go through acos, which is not correctly rounded on the GPU, and agree within a few ulp.

Conventions. The truth G of pair p = (src, tgt) maps source points onto the target, t ~ R s + t, like
Registration.pose. Keypoints are the KeypointSet layout: cloud b's real slots are [0, n_b), n_b = clamp(count[b], 0, k),
in ascending score order, so its top n are the slots [max(0, n_b - n), n_b); slots at or past n_b are never read. A
source keypoint s (fp32, widened exactly) becomes q_a = ((G_a0 s_0 + G_a1 s_1) + G_a2 s_2) + t_a, and its squared
distance to a target keypoint t is d^2 = (e_0^2 + e_1^2) + e_2^2 with e = q - t: register_np.residual2. Every distance
test is d^2 < tau^2 (strict), tau^2 = tau * tau in fp64. The reference compares sqrt(d^2) < tau; the two differ only
at rounding ties.

A pair is evaluated (valid) when flags[p] bit 0 is set and both cloud ids lie in [0, B). For an evaluated pair:
  * FMR (geometric_registration/evaluate.py:67-82, :207): n_match_inliers counts the match rows m < clamp(n_matches[p],
    0, L) whose (source slot, target slot) are both real and have d^2 < tau_fmr^2 (a row naming a slot that is not
    real is a match that is not an inlier); inlier_ratio = n_match_inliers / n_matches, 0 when there are no matches
    (the reference fails on an empty list: this value is ours); fmr_hit = inlier_ratio > fmr_ratio.
  * repeatability (repeatability/evaluate_3dmatch_our.py:30-41): at level n_r, a target slot among the top n_r is
    repeated when no source slot among the top n_r gives a NaN d^2 and the smallest d^2 is < tau_rep^2 (numpy's
    min(axis=0) < tau, NaN included; no source slot: not repeated). repeatability = n_repeated / n_r (n_r, not the
    count, as in the reference).
  * pose metrics of every pose set s (utils/tester.py:326-342): rte = sqrt((d_0^2 + d_1^2) + d_2^2), d = t - t_G;
    tr = (c_0 + c_1) + c_2 with c_i = ((R_0i G_0i + R_1i G_1i) + R_2i G_2i) = tr(R^T R_G); c = (tr - 1) / 2 clamped to
    [-1, 1] (the one stated deviation: unclamped, a pose equal to G can give 1 + eps and a NaN); rre_deg =
    acos(c) * (180 / pi). success = rte < rte_max and c > cos(rre_max) (cos(rre_max_deg * (pi / 180)) on the host).
    A non-finite entry in rows 0-2 of G or of the pose makes rte, rre_deg and rmse2 NaN: a miss in every pose test.
  * registration recall (3dmatch/evaluate.m, mrEvaluateRegistration.m), when flags bit 1 is set and info is given:
    E = G inv(pose) with inv(pose) = [R^T | -R^T t], each entry ((x_0 y_0 + x_1 y_1) + x_2 y_2) (+ t_G);
    q_0 = 0.5 sqrt(((1 + E_00) + E_11) + E_22), q_v = -(E_21 - E_12, E_02 - E_20, E_10 - E_01) / (4 q_0) (dcm2quat);
    er = [t_E; -q_v]; v_j = sum_i er_i info_ij, rmse2 = (sum_j v_j er_j) / info_00 (sums sequential from 0.0);
    recall_hit = rmse2 <= err2 (a NaN is a miss, as in MATLAB).
A pair that is not evaluated reads nothing and has valid 0, zeros, and NaN rte / rre_deg / rmse2.

Totals, summed over pairs in pair order, sequentially from 0.0, into one float64 vector (counts are exact):
  [0] evaluated pairs, [1] FMR hits, [2] sum inlier_ratio, [3] sum n_match_inliers, [4 + r] sum repeatability at
  level r, then per pose set s at 4 + R + 7 s: successes, sum rte over rte < rte_max, that count, sum rre_deg over
  c > cos(rre_max), that count, recall hits, recall pairs.
"""
import math

import numpy as np

from . import register_np

MAX_LEVELS = 14          # 4 + 14 + 7 * 2 = 32 totals: one lane each in the CUDA totals warp
RAD2DEG = 180.0 / math.pi
CHUNK = 512              # source ranks per numpy pass in repeatability; the result does not depend on it


def n_totals(R, S):
    return 4 + R + 7 * S


def within(d2, tau2):
    return d2 < tau2


def repeat_divisor(n_r, n_target):
    """The divisor of n_repeated at level n_r: n_r itself, as in the reference."""
    return float(n_r)


def clamp_cos(c):
    return np.where(c > 1.0, 1.0, np.where(c < -1.0, -1.0, c))


def accumulate(values):
    """Sequential sum from 0.0 in the given (pair) order."""
    acc = 0.0
    for v in values:
        acc = acc + float(v)
    return acc


def transform(G, s):
    """q_a = ((G_a0 s_0 + G_a1 s_1) + G_a2 s_2) + t_a over the rows of s [n,3] (fp64)."""
    return [((G[a, 0] * s[:, 0] + G[a, 1] * s[:, 1]) + G[a, 2] * s[:, 2]) + G[a, 3] for a in range(3)]


def dist2(q, t):
    e = [q[a] - t[..., a] for a in range(3)]
    return (e[0] * e[0] + e[1] * e[1]) + e[2] * e[2]


def fmr_pair(G, src, tgt, ns, nt, rows, tau2):
    """n_match_inliers of one pair: rows [m,2] (source slot, target slot)."""
    if len(rows) == 0:
        return 0
    i, j = rows[:, 0], rows[:, 1]
    real = (i >= 0) & (i < ns) & (j >= 0) & (j < nt)
    s = src[np.where(real, i, 0)].astype(np.float64)
    t = tgt[np.where(real, j, 0)].astype(np.float64)
    return int((real & within(dist2(transform(G, s), t), tau2)).sum())


def repeat_pair(G, src, tgt, ns, nt, levels, tau2):
    """n_repeated [R] of one pair: source ranks walked from the top in chunks, a running min d^2 and NaN flag per
    target slot, hits recorded at each level boundary."""
    R = len(levels)
    out = np.zeros(R, np.int64)
    if R == 0 or nt == 0:
        return out
    n_max = levels[-1]
    t0 = max(0, nt - n_max)
    T = tgt[t0:nt].astype(np.float64)                    # target slots t0 .. nt-1
    mn = np.full(nt - t0, np.inf)
    nan = np.zeros(nt - t0, bool)
    done = 0
    for r, n_r in enumerate(levels):
        b = min(n_r, ns)
        while done < b:
            m1 = min(b, done + CHUNK)
            slots = ns - 1 - np.arange(done, m1)         # ranks done .. m1-1, from the highest score down
            q = transform(G, src[slots].astype(np.float64))
            d2 = dist2([x[:, None] for x in q], T[None, :, :])
            nan |= np.isnan(d2).any(axis=0)
            with np.errstate(invalid="ignore"):
                mn = np.minimum(mn, np.where(np.isnan(d2), np.inf, d2).min(axis=0))
            done = m1
        in_top = np.arange(t0, nt) >= nt - n_r
        if ns > 0:
            out[r] = int((in_top & ~nan & within(mn, tau2)).sum())
    return out


def pose_metrics(G, T, cos_max, rte_max):
    """(rte, c, rre_deg) of poses T [P,4,4] against G [P,4,4], elementwise over pairs."""
    with np.errstate(all="ignore"):
        d = [T[:, a, 3] - G[:, a, 3] for a in range(3)]
        rte = np.sqrt((d[0] * d[0] + d[1] * d[1]) + d[2] * d[2])
        col = [((T[:, 0, i] * G[:, 0, i] + T[:, 1, i] * G[:, 1, i]) + T[:, 2, i] * G[:, 2, i]) for i in range(3)]
        tr = (col[0] + col[1]) + col[2]
        c = clamp_cos((tr - 1.0) / 2.0)
        fin = finite_poses(G, T)
        rte = np.where(fin, rte, np.nan)
        c = np.where(fin, c, np.nan)
        rre = np.arccos(c) * RAD2DEG
    return rte, c, rre


def finite_poses(G, T):
    return np.isfinite(G[:, :3, :]).all(axis=(1, 2)) & np.isfinite(T[:, :3, :]).all(axis=(1, 2))


def choi_error(G, T, info):
    """Choi's registration error p of poses T against G with information matrices info [P,6,6]."""
    with np.errstate(all="ignore"):
        R, t = T[:, :3, :3], T[:, :3, 3]
        ti = [-((R[:, 0, a] * t[:, 0] + R[:, 1, a] * t[:, 1]) + R[:, 2, a] * t[:, 2]) for a in range(3)]
        E = [[(G[:, a, 0] * R[:, b, 0] + G[:, a, 1] * R[:, b, 1]) + G[:, a, 2] * R[:, b, 2] for b in range(3)]
             for a in range(3)]
        tE = [((G[:, a, 0] * ti[0] + G[:, a, 1] * ti[1]) + G[:, a, 2] * ti[2]) + G[:, a, 3] for a in range(3)]
        q0 = 0.5 * np.sqrt(((1.0 + E[0][0]) + E[1][1]) + E[2][2])
        d = 4.0 * q0
        qv = [-(E[2][1] - E[1][2]) / d, -(E[0][2] - E[2][0]) / d, -(E[1][0] - E[0][1]) / d]
        er = tE + [-x for x in qv]
        v = []
        for j in range(6):
            acc = np.zeros(len(q0))
            for i in range(6):
                acc = acc + er[i] * info[:, i, j]
            v.append(acc)
        num = np.zeros(len(q0))
        for j in range(6):
            num = num + v[j] * er[j]
        return num / info[:, 0, 0]


def evaluate(points, count, matches, n_matches, pairs, pose_gt, info, flags, poses=(), *, levels,
             fmr_distance=0.10, fmr_ratio=0.05, repeat_distance=0.10, err2=0.04, rte_max=2.0, rre_max_deg=5.0):
    """dict of per-pair fields and `totals`. points [B,k,3] float32, count [B], matches [P,L,2], n_matches [P],
    pairs [P,2], pose_gt [P,4,4] float64, info [P,6,6] float64 or None, flags [P], poses: 0-2 arrays [P,4,4],
    levels: ascending ints in [1, k]."""
    points = np.asarray(points, np.float32)
    B, k, _ = points.shape
    pairs = np.asarray(pairs, np.int64).reshape(-1, 2)
    P = pairs.shape[0]
    matches = np.asarray(matches, np.int64).reshape(P, -1, 2)
    L = matches.shape[1]
    n_m = np.clip(np.asarray(n_matches, np.int64).reshape(P), 0, L)
    cnt = np.clip(np.asarray(count, np.int64).reshape(B), 0, k)
    G = np.asarray(pose_gt, np.float64).reshape(P, 4, 4)
    flags = np.asarray(flags, np.int64).reshape(P)
    info = None if info is None else np.asarray(info, np.float64).reshape(P, 6, 6)
    poses = [np.asarray(T, np.float64).reshape(P, 4, 4) for T in poses]
    levels = [int(n) for n in levels]
    R, S = len(levels), len(poses)
    tau_f2 = float(fmr_distance) * float(fmr_distance)
    tau_r2 = float(repeat_distance) * float(repeat_distance)
    cos_max = math.cos(float(rre_max_deg) * (math.pi / 180.0))
    ok = ((flags & 1) != 0) & (pairs[:, 0] >= 0) & (pairs[:, 0] < B) & (pairs[:, 1] >= 0) & (pairs[:, 1] < B)
    out = dict(valid=ok.astype(np.int32), n_match_inliers=np.zeros(P, np.int32), inlier_ratio=np.zeros(P),
               fmr_hit=np.zeros(P, np.int32), n_repeated=np.zeros((P, R), np.int32), repeatability=np.zeros((P, R)),
               rte=np.full((S, P), np.nan), rre_deg=np.full((S, P), np.nan), rmse2=np.full((S, P), np.nan),
               success=np.zeros((S, P), np.int32), recall_hit=np.zeros((S, P), np.int32))
    with np.errstate(all="ignore"):
        for p in np.nonzero(ok)[0]:
            src, tgt = pairs[p]
            ns, nt = int(cnt[src]), int(cnt[tgt])
            nin = fmr_pair(G[p], points[src], points[tgt], ns, nt, matches[p, :n_m[p]], tau_f2)
            out["n_match_inliers"][p] = nin
            ratio = float(nin) / float(n_m[p]) if n_m[p] > 0 else 0.0
            out["inlier_ratio"][p] = ratio
            out["fmr_hit"][p] = ratio > fmr_ratio
            rep = repeat_pair(G[p], points[src], points[tgt], ns, nt, levels, tau_r2)
            out["n_repeated"][p] = rep
            out["repeatability"][p] = [float(rep[r]) / repeat_divisor(levels[r], nt) for r in range(R)]
    recall_pair = ok & ((flags & 2) != 0) & (info is not None)
    rte_ok, rre_ok = np.zeros((S, P), bool), np.zeros((S, P), bool)
    for s, T in enumerate(poses):
        rte, c, rre = pose_metrics(G, T, cos_max, rte_max)
        rte_ok[s], rre_ok[s] = ok & (rte < rte_max), ok & (c > cos_max)
        out["rte"][s] = np.where(ok, rte, np.nan)
        out["rre_deg"][s] = np.where(ok, rre, np.nan)
        out["success"][s] = rte_ok[s] & rre_ok[s]
        if info is not None:
            e = np.where(finite_poses(G, T), choi_error(G, T, info), np.nan)
            out["rmse2"][s] = np.where(recall_pair, e, np.nan)
            with np.errstate(invalid="ignore"):
                out["recall_hit"][s] = recall_pair & (e <= err2)
    idx = np.nonzero(ok)[0]
    totals = [accumulate(np.ones(len(idx))), accumulate(out["fmr_hit"][idx]), accumulate(out["inlier_ratio"][idx]),
              accumulate(out["n_match_inliers"][idx])]
    totals += [accumulate(out["repeatability"][idx, r]) for r in range(R)]
    for s in range(S):
        a, b = np.nonzero(rte_ok[s])[0], np.nonzero(rre_ok[s])[0]
        totals += [accumulate(out["success"][s, idx]), accumulate(out["rte"][s, a]), float(len(a)),
                   accumulate(out["rre_deg"][s, b]), float(len(b)), accumulate(out["recall_hit"][s, idx]),
                   float(recall_pair.sum())]
    out["totals"] = np.array(totals, np.float64)
    return out
