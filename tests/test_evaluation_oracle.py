"""Ground-truth metrics contract (oracle/evaluate_np.py) on the CPU: agreement with direct restatements of the reference
formulas, known answers, the emulated bugs it rejects, the 3DMatch gt.log / gt.info readers, and the argument checks
of evaluation.evaluate_pairs, GraphPipeline(evaluate=...) and d3f_evaluate_pairs that run before any device work."""
import ctypes as C
import os

import numpy as np
import pytest

from oracle import evaluate_np

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
LOG, INFO = os.path.join(GOLDEN, "hotel3_gt.log"), os.path.join(GOLDEN, "hotel3_gt.info")
FIELDS = ("valid", "n_match_inliers", "inlier_ratio", "fmr_hit", "n_repeated", "repeatability", "rte", "rmse2",
          "success", "recall_hit", "totals")


def mismatches(got, want, fields=FIELDS):
    bad = []
    for f in fields:
        g, w = np.asarray(got[f]), np.asarray(want[f])
        if g.dtype == np.float64:
            g, w = g.view(np.int64), w.view(np.int64)
        if g.shape != w.shape or not np.array_equal(g, w):
            bad.append(f)
    return bad


def rotation(axis, deg):
    axis = np.asarray(axis, float)
    axis = axis / np.linalg.norm(axis)
    th = np.deg2rad(deg)
    K = np.array([[0, -axis[2], axis[1]], [axis[2], 0, -axis[0]], [-axis[1], axis[0], 0]])
    return np.eye(3) + np.sin(th) * K + (1 - np.cos(th)) * K @ K


def rigid(R, t):
    T = np.eye(4)
    T[:3, :3], T[:3, 3] = R, t
    return T


def random_pose(rng, deg=30.0, shift=1.0):
    return rigid(rotation(rng.normal(size=3), rng.uniform(0, deg)), rng.uniform(-shift, shift, 3))


def scene(rng, P=6, B=4, k=64, noise=0.05, overlap=0.7):
    """B clouds of k keypoints: cloud b+1's first slots are cloud b's moved by a random pose plus noise. Pairs (b, b+1)
    with that pose as truth, identity matches on the overlapping slots, and random RANSAC-like poses near it."""
    pts = np.zeros((B, k, 3), np.float32)
    pts[0] = rng.uniform(0, 2, (k, 3))
    G = []
    for b in range(1, B):
        T = random_pose(rng)
        moved = pts[b - 1] @ T[:3, :3].T + T[:3, 3] + rng.normal(scale=noise, size=(k, 3))
        m = int(k * overlap)
        pts[b, :m] = moved[:m]
        pts[b, m:] = rng.uniform(-1, 3, (k - m, 3))
        G.append(T)
    pairs = [(b, b + 1) for b in range(B - 1)]
    pairs = (pairs * (P // len(pairs) + 1))[:P]
    G = np.stack([G[s] for s, _ in pairs])
    matches = np.full((P, k, 2), -1, np.int64)
    n_m = np.zeros(P, np.int64)
    for p in range(P):
        n = int(rng.integers(1, k + 1))
        idx = np.sort(rng.choice(k, n, replace=False))
        matches[p, :n] = np.stack([idx, idx], 1)
        n_m[p] = n
    est = np.stack([rigid(rotation(rng.normal(size=3), rng.uniform(0, 8)), rng.normal(scale=1.0, size=3)) @ g
                    for g in G])
    return pts, np.full(B, k), matches, n_m, np.array(pairs), G, est


def fixture_info(P):
    from d3feat_b200 import io_utils
    _, info = io_utils.load_info(INFO)
    return info[np.arange(P) % len(info)]


# ---- 1. agreement with the reference's own formulas ------------------------------------------------------------

def reference_metrics(pts, matches, n_m, pairs, G, est, info, levels, tau_f=0.1, tau_r=0.1):
    """The reference's per-pair numpy: evaluate.py's inlier ratio, cdist repeatability, tester.py's rte / rre and a
    numpy mrEvaluateRegistration -- with the truth applied as the reference does (T_log = inv(G) moves the target)."""
    from scipy.spatial.distance import cdist
    out = dict(ratio=[], rep=[], rte=[], rre=[], p=[])
    for p, (s, t) in enumerate(pairs):
        T_log = np.linalg.inv(G[p])
        corr = matches[p, :n_m[p]]
        frag1 = pts[s][corr[:, 0]].astype(np.float64)
        frag2 = pts[t][corr[:, 1]].astype(np.float64) @ T_log[:3, :3].T + T_log[:3, 3]
        distance = np.sqrt(np.sum(np.power(frag1 - frag2, 2), axis=1))
        out["ratio"].append(np.sum(distance < tau_f) / len(distance))
        rep = []
        for n in levels:
            src = pts[s][-n:].astype(np.float64)
            tgt = pts[t][-n:].astype(np.float64) @ T_log[:3, :3].T + T_log[:3, 3]
            rep.append(np.sum(cdist(src, tgt).min(axis=0) < tau_r) * 1.0 / n)
        out["rep"].append(rep)
        T = est[p]
        out["rte"].append(np.linalg.norm(T[:3, 3] - G[p][:3, 3]))
        out["rre"].append(np.arccos((np.trace(T[:3, :3].transpose() @ G[p][:3, :3]) - 1) / 2) * 180 / np.pi)
        E = np.linalg.inv(T_log) @ np.linalg.inv(T)             # gt.trans ^ -1 * result.trans, result = inv(pose)
        D = E[:3, :3]
        q = np.zeros(4)
        q[0] = 0.5 * np.sqrt(1 + D[0, 0] + D[1, 1] + D[2, 2])
        q[1] = -(D[2, 1] - D[1, 2]) / (4 * q[0])
        q[2] = -(D[0, 2] - D[2, 0]) / (4 * q[0])
        q[3] = -(D[1, 0] - D[0, 1]) / (4 * q[0])
        er = np.concatenate([E[:3, 3], -q[1:]])
        out["p"].append(er @ info[p] @ er / info[p][0, 0])
    return {k: np.array(v) for k, v in out.items()}


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_oracle_agrees_with_the_reference_formulas(seed):
    rng = np.random.default_rng(seed)
    pts, cnt, matches, n_m, pairs, G, est = scene(rng, P=9, k=80)
    info = fixture_info(len(pairs))
    levels = [4, 8, 16, 32, 64, 80]
    got = evaluate_np.evaluate(pts, cnt, matches, n_m, pairs, G, info, np.full(len(pairs), 3), [est], levels=levels)
    ref = reference_metrics(pts, matches, n_m, pairs, G, est, info, levels)
    assert (got["valid"] == 1).all()
    assert np.abs(got["inlier_ratio"] - ref["ratio"]).max() < 1e-9
    assert np.abs(got["repeatability"] - ref["rep"]).max() < 1e-9
    assert np.abs(got["rte"][0] - ref["rte"]).max() < 1e-9
    assert np.abs(got["rre_deg"][0] - ref["rre"]).max() < 1e-9
    assert np.abs(got["rmse2"][0] - ref["p"]).max() < 1e-9 * max(1.0, np.abs(ref["p"]).max())
    assert 0 < got["inlier_ratio"].max() and got["repeatability"].max() > 0
    t = got["totals"]
    assert len(t) == evaluate_np.n_totals(len(levels), 1)
    assert t[0] == len(pairs) and t[1] == (ref["ratio"] > 0.05).sum()
    assert abs(t[2] - ref["ratio"].sum()) < 1e-9
    assert t[4 + len(levels) + 6] == len(pairs)
    assert t[4 + len(levels) + 5] == (ref["p"] <= 0.04).sum()
    kitti = (ref["rte"] < 2) & (ref["rre"] < 5)
    assert t[4 + len(levels)] == kitti.sum()


# ---- 2. known answers -----------------------------------------------------------------------------------------

def exact_case(inverted=False, k=48):
    rng = np.random.default_rng(11)
    src = rng.uniform(0, 3, (k, 3)).astype(np.float32)
    G = random_pose(rng, 40, 2.0)
    tgt = (src.astype(np.float64) @ G[:3, :3].T + G[:3, 3]).astype(np.float32)
    pts = np.stack([src, tgt])
    matches = np.stack([np.arange(k)] * 2, 1)[None]
    truth = np.linalg.inv(G) if inverted else G
    info = fixture_info(1)
    return evaluate_np.evaluate(pts, [k, k], matches, [k], [(0, 1)], truth[None], info, [3], [G[None]],
                                levels=[4, 8, 16, 32, 48])


def test_oracle_known_answers_and_the_inverted_truth():
    got = exact_case()
    assert got["inlier_ratio"][0] == 1.0 and got["fmr_hit"][0] == 1
    assert (got["repeatability"][0] == 1.0).all()
    assert got["rte"][0, 0] == 0.0 and got["rre_deg"][0, 0] < 1e-6 and abs(got["rmse2"][0, 0]) < 1e-20
    assert got["success"][0, 0] == 1 and got["recall_hit"][0, 0] == 1
    bad = exact_case(inverted=True)
    assert bad["fmr_hit"][0] == 0 and bad["inlier_ratio"][0] < 0.1
    assert bad["repeatability"][0, -1] < 0.5
    assert bad["success"][0, 0] == 0 and bad["recall_hit"][0, 0] == 0


def test_oracle_pairs_that_are_not_evaluated():
    rng = np.random.default_rng(3)
    pts, cnt, matches, n_m, pairs, G, est = scene(rng, P=5)
    pairs[1] = (-1, 1)
    pairs[2] = (0, 4)
    G[4] = np.nan
    flags = np.array([1, 3, 3, 0, 3])
    got = evaluate_np.evaluate(pts, cnt, matches, n_m, pairs, G, fixture_info(5), flags, [est, est], levels=[4, 64])
    assert got["valid"].tolist() == [1, 0, 0, 0, 1]
    for p in (1, 2, 3):
        assert got["n_match_inliers"][p] == 0 and (got["repeatability"][p] == 0).all()
        assert np.isnan(got["rte"][:, p]).all() and np.isnan(got["rmse2"][:, p]).all()
    # a NaN truth is evaluated and misses every test
    assert got["n_match_inliers"][4] == 0 and (got["n_repeated"][4] == 0).all()
    assert np.isnan(got["rte"][:, 4]).all() and got["success"][:, 4].sum() == 0 and got["recall_hit"][:, 4].sum() == 0
    assert got["totals"][0] == 2 and got["totals"][4 + 2 + 6] == 1       # pair 0 has flags 1: no recall pair


# ---- 3. emulated bugs ----------------------------------------------------------------------------------------------

def tie_case():
    """Targets exactly at tau = 0.25 from their sources (exact in fp32 and fp64), three target keypoints."""
    src = np.array([[0, 0, 0], [1, 0, 0], [2, 0, 0], [3, 0, 0]], np.float32)
    tgt = np.zeros((4, 3), np.float32)
    tgt[:3] = src[1:] + np.float32([0.25, 0, 0])
    return np.stack([src, tgt]), [4, 3], np.array([[[1, 0], [2, 1], [3, 2], [-1, -1]]]), [3]


def unclamped_rotation():
    rng = np.random.default_rng(0)
    for _ in range(10000):
        T = random_pose(rng, 180.0)
        col = [((T[0, i] * T[0, i] + T[1, i] * T[1, i]) + T[2, i] * T[2, i]) for i in range(3)]
        if ((col[0] + col[1]) + col[2] - 1.0) / 2.0 > 1.0:
            return T
    raise AssertionError("no rotation with c > 1 found")


def _reversed(values):
    acc = 0.0
    for v in list(values)[::-1]:
        acc = acc + float(v)
    return acc


@pytest.mark.parametrize("bug", ["truth_inverted", "inlier_le", "divide_by_count", "consecutive_recall",
                                 "unclamped_cos", "totals_out_of_order"])
def test_oracle_rejects_emulated_bugs(monkeypatch, bug):
    from d3feat_b200 import io_utils
    kw = dict(levels=[4, 8])
    if bug == "truth_inverted":
        a, b = exact_case(), exact_case(inverted=True)
        assert mismatches(a, b)
        return
    if bug in ("inlier_le", "divide_by_count"):
        pts, cnt, matches, n_m = tie_case()
        args = (pts, cnt, matches, n_m, [(0, 1)], np.eye(4)[None], None, [1])
        kw = dict(levels=[4], fmr_distance=0.25, repeat_distance=0.25 if bug == "inlier_le" else 0.5)
    elif bug == "consecutive_recall":
        ids, _ = io_utils.load_log(LOG)
        pairs = ids[:, :2]
        est = np.tile(np.eye(4), (len(pairs), 1, 1))
        pts = np.zeros((37, 4, 3), np.float32)
        args = lambda: (pts, np.full(37, 4), np.full((len(pairs), 4, 2), -1), np.zeros(len(pairs)), pairs,  # noqa
                        *io_utils.truth_for_pairs(io_utils.load_log(LOG), io_utils.load_info(INFO), pairs), [est])
    elif bug == "unclamped_cos":
        T = unclamped_rotation()
        pts = np.zeros((2, 4, 3), np.float32)
        args = (pts, [4, 4], np.full((1, 4, 2), -1), [0], [(0, 1)], T[None], None, [1], [T[None]])
    else:
        rng = np.random.default_rng(5)
        pts, cnt, matches, n_m, pairs, G, est = scene(rng, P=40, k=64)
        args = (pts, cnt, matches, n_m, pairs, G, fixture_info(40), np.full(40, 3), [est])
    call = (lambda: evaluate_np.evaluate(*args(), **kw)) if callable(args) else \
        (lambda: evaluate_np.evaluate(*args, **kw))
    want = call()
    target, name, fn = {"inlier_le": (evaluate_np, "within", lambda d2, tau2: d2 <= tau2),
                        "divide_by_count": (evaluate_np, "repeat_divisor", lambda n_r, nt: float(min(n_r, nt))),
                        "consecutive_recall": (io_utils, "counts_for_recall", lambda i, j: j - i >= 1),
                        "unclamped_cos": (evaluate_np, "clamp_cos", lambda c: c),
                        "totals_out_of_order": (evaluate_np, "accumulate", _reversed)}[bug]
    monkeypatch.setattr(target, name, fn)
    got = call()
    assert mismatches(got, want), bug


# ---- 4. gt.log / gt.info readers ------------------------------------------------------------------------------------

def test_load_log_and_info_of_the_fixture():
    from d3feat_b200 import io_utils
    ids, T = io_utils.load_log(LOG)
    iids, info = io_utils.load_info(INFO)
    assert T.shape == (54, 4, 4) and info.shape == (54, 6, 6)
    assert (ids[:, 2] == 37).all() and np.array_equal(ids, iids)
    assert ids[0].tolist() == [0, 1, 37] and ids[1].tolist() == [0, 12, 37] and ids[-1].tolist() == [35, 36, 37]
    assert abs(T[0, 0, 0] - 0.968286) < 1e-12 and abs(T[0, 2, 3] + 0.12249969) < 1e-12
    assert np.abs(T[:, :3, :3] @ T[:, :3, :3].transpose(0, 2, 1) - np.eye(3)).max() < 1e-5
    assert (T[:, 3] == [0, 0, 0, 1]).all()
    assert np.abs(info - info.transpose(0, 2, 1)).max() == 0 and info[0, 0, 0] == 5000 and (info[:, 0, 0] > 0).all()


def test_truth_for_pairs_flags_and_inverse():
    from d3feat_b200 import io_utils
    log, info = io_utils.load_log(LOG), io_utils.load_info(INFO)
    pairs = [(0, 1), (0, 12), (2, 3), (1, 0), (5, 30)]
    gt = io_utils.truth_for_pairs(log, info, pairs)
    assert gt.flags.tolist() == [1, 3, 1, 0, 0]
    assert np.abs(gt.pose[1] @ log[1][1] - np.eye(4)).max() < 1e-12
    assert (gt.pose[3] == np.eye(4)).all() and (gt.info[0] == 0).all() and (gt.info[1] == info[1][1]).all()
    all_pairs = log[0][:, :2]
    flags = io_utils.truth_for_pairs(log, info, all_pairs).flags
    assert (flags & 1).all() and ((flags & 2) != 0).tolist() == (all_pairs[:, 1] - all_pairs[:, 0] > 1).tolist()
    assert (io_utils.truth_for_pairs(log, None, all_pairs).flags == 1).all()


def test_summary_of_totals():
    from d3feat_b200.evaluation import summary
    t = np.array([10, 8, 6.0, 400, 5.0, 2.5] + [6, 3.0, 7, 14.0, 6, 5, 8], np.float64)
    s = summary(t, (4, 8), ("ransac",))
    assert s["n_pairs"] == 10 and s["fmr"] == 0.8 and s["avg_inliers"] == 50.0 and s["avg_inlier_ratio"] == 0.75
    assert s["repeatability"] == {4: 0.5, 8: 0.25}
    assert s["ransac"]["success_rate"] == 0.6 and s["ransac"]["rte"] == 3.0 / 7 and s["ransac"]["rre_deg"] == 14.0 / 6
    assert s["ransac"]["registration_recall"] == 5 / 8
    with pytest.raises(ValueError, match="totals"):
        summary(t, (4,), ("ransac",))


# ---- 5. argument checks before any device work ---------------------------------------------------------------------

def test_evaluate_options_checked():
    from d3feat_b200.evaluation import check_evaluate_options
    assert check_evaluate_options(250)[0] == (4, 8, 16, 32, 64, 128)
    assert check_evaluate_options(5000)[0] == (4, 8, 16, 32, 64, 128, 256, 512)
    assert check_evaluate_options(3)[0] == ()
    assert check_evaluate_options(5000, repeat_levels=[1, 5000])[0] == (1, 5000)
    for bad in (dict(repeat_levels=[8, 4]), dict(repeat_levels=[4, 4]), dict(repeat_levels=[0]),
                dict(repeat_levels=[251]), dict(repeat_levels=list(range(1, 16))), dict(repeat_levels=[4.0]),
                dict(repeat_levels=5), dict(fmr_distance=0), dict(repeat_distance=float("nan")),
                dict(fmr_ratio=1.0), dict(fmr_ratio=-0.1), dict(err2=0), dict(rte_max=float("inf")),
                dict(rre_max_deg=0), dict(rre_max_deg=181), dict(fmr_distance="x")):
        with pytest.raises(ValueError, match="evaluate_pairs"):
            check_evaluate_options(250, **bad)


def test_graph_pipeline_evaluate_checked_first():
    from d3feat_b200.encoder import GraphPipeline
    bbox = np.zeros(6, np.float32)
    with pytest.raises(ValueError, match="needs match_pairs"):
        GraphPipeline(None, [1024] * 5, 2, bbox, decoder=True, keypoints=250, evaluate={})
    for bad in ([("fmr_ratio", 0.1)], {"fmr": 0.1}, {"repeat_levels": [300]}, {"rte_max": -1}):
        with pytest.raises(ValueError, match="GraphPipeline"):
            GraphPipeline(None, [1024] * 5, 2, bbox, decoder=True, keypoints=250, match_pairs=[(0, 1)], evaluate=bad)


def test_check_truth():
    from d3feat_b200.evaluation import GroundTruth, check_truth
    pose = np.tile(np.eye(4), (3, 1, 1))
    check_truth(GroundTruth(pose, None, np.array([1, 3, 0])), 3)
    for bad in (pose, GroundTruth(pose[:2], None, np.ones(3)), GroundTruth(pose, np.zeros((3, 6)), np.ones(3)),
                GroundTruth(pose, None, np.ones(2))):
        with pytest.raises(ValueError, match="truth"):
            check_truth(bad, 3)
    nan = pose.copy()
    nan[1, 2, 3] = np.inf
    with pytest.raises(ValueError, match="pair 1 has truth with a non-finite pose"):
        check_truth(GroundTruth(nan, None, np.array([1, 1, 1])), 3)
    check_truth(GroundTruth(nan, None, np.array([1, 0, 1])), 3)   # an unflagged pair is never read


def test_evaluate_pairs_invalid_arguments_without_a_gpu():
    from d3feat_b200 import build
    from d3feat_b200._lib import SYMBOLS
    lib = C.CDLL(build.build())
    lib.d3f_last_error.restype = C.c_char_p
    for name in ("d3f_evaluate_pairs_workspace_bytes", "d3f_evaluate_pairs"):
        fn = getattr(lib, name)
        fn.restype, fn.argtypes = [(r, a) for n, r, a in SYMBOLS if n == name][0]
    assert lib.d3f_evaluate_pairs_workspace_bytes(0, 1) == 0
    assert lib.d3f_evaluate_pairs_workspace_bytes(10, 3) == 0
    assert lib.d3f_evaluate_pairs_workspace_bytes(10, 0) >= 40
    ws_ok = lib.d3f_evaluate_pairs_workspace_bytes(100, 2)
    assert ws_ok >= 800
    fake = C.c_void_p(256)          # never dereferenced: validation fails first
    poses = (C.c_void_p * 2)(256, 256)
    no_pose = (C.c_void_p * 2)(256, None)

    def call(B=4, k=250, L=250, P=100, S=2, levels=(4, 8, 16), fd=0.1, fr=0.05, rd=0.1, e2=0.04, rm=2.0, rr=5.0,
             ws=ws_ok, null=None, pp=poses):
        p = [None if i == null else fake for i in range(20)]
        lv = (C.c_int * max(1, len(levels)))(*levels)
        return lib.d3f_evaluate_pairs(p[0], p[1], B, k, p[2], p[3], L, p[4], P, p[5], None, p[6], pp, S, lv,
                                      len(levels), fd, fr, rd, e2, rm, rr, *p[7:18], p[18], p[19], ws, None)

    cases = [(dict(B=0), b"B=0"), (dict(B=1025), b"B=1025"), (dict(k=0), b"k=0"), (dict(L=0), b"L=0"),
             (dict(P=0), b"P=0"), (dict(P=1 << 20, k=5000), b"exceeds int32"), (dict(S=3), b"S=3"),
             (dict(S=-1), b"S=-1"), (dict(levels=tuple(range(1, 16))), b"R=15"), (dict(levels=(8, 4)), b"ascend"),
             (dict(levels=(4, 4)), b"ascend"), (dict(levels=(0,)), b"ascend"), (dict(levels=(251,)), b"ascend"),
             (dict(fd=0.0), b"fmr_distance"), (dict(rd=float("nan")), b"repeat_distance"),
             (dict(fr=1.0), b"fmr_ratio"), (dict(fr=-0.5), b"fmr_ratio"), (dict(e2=0.0), b"err2"),
             (dict(rm=float("inf")), b"rte_max"), (dict(rr=0.0), b"rre_max_deg"), (dict(rr=200.0), b"rre_max_deg"),
             (dict(pp=no_pose), b"poses[1]"), (dict(pp=None), b"null pointer")]
    cases += [(dict(null=i), b"null pointer") for i in range(20)]
    for kw, msg in cases:
        assert call(**kw) == -1, kw
        assert msg in lib.d3f_last_error(), (kw, lib.d3f_last_error())
    # the outputs of absent levels and pose sets may be NULL (the checks still stop at the workspace)
    assert call(levels=(), null=11, ws=0) == -4
    assert call(levels=(), null=12, ws=0) == -4
    assert call(S=0, null=13, ws=0) == -4
    assert call(ws=ws_ok - 1) == -4
    assert b"workspace" in lib.d3f_last_error()
