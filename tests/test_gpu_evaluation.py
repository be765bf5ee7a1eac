"""Ground-truth metrics on the GPU (d3f_evaluate_pairs, evaluation.evaluate_pairs, GraphPipeline(..., evaluate=...))
against the numpy restatement oracle/evaluate_np.py.

Every value is compared bit for bit (float64 as bit patterns, any NaN equal to any NaN), except rre_deg, which goes
through the GPU's acos (not correctly rounded): it must lie within RRE_ULP ulp of the oracle, and the totals' sums of
rre_deg within RRE_REL relative. Every decision, including which pairs enter those sums, is exact."""
import numpy as np
import pytest

from oracle import evaluate_np

RRE_ULP = 4
RRE_REL = 1e-13
EXACT = ("valid", "n_match_inliers", "inlier_ratio", "fmr_hit", "n_repeated", "repeatability", "rte", "rmse2",
         "success", "recall_hit")
OPTS = dict(fmr_distance=0.10, fmr_ratio=0.05, repeat_distance=0.10, err2=0.04, rte_max=2.0, rre_max_deg=5.0)


def t(a, dev):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def same_bits(g, w):
    g, w = np.asarray(g), np.asarray(w)
    if g.shape != w.shape:
        return False
    if g.dtype != np.float64:
        return np.array_equal(g, w)
    return bool(((g.view(np.int64) == w.view(np.int64)) | (np.isnan(g) & np.isnan(w))).all())


def rre_sum_lanes(R, S):
    return [4 + R + 7 * s + 3 for s in range(S)]


def mismatches(got, want, R, S):
    bad = [f for f in EXACT if not same_bits(got[f], want[f])]
    g, w = np.asarray(got["rre_deg"]), np.asarray(want["rre_deg"])
    nan_ok = np.array_equal(np.isnan(g), np.isnan(w))
    fin = ~np.isnan(w)
    if g.shape != w.shape or not nan_ok or (np.abs(g[fin].view(np.int64) - w[fin].view(np.int64)) > RRE_ULP).any():
        bad.append("rre_deg")
    gt, wt = np.asarray(got["totals"]), np.asarray(want["totals"])
    approx = rre_sum_lanes(R, S)
    exact = [i for i in range(len(wt)) if i not in approx]
    if gt.shape != wt.shape or not same_bits(gt[exact], wt[exact]) or \
            (np.abs(gt[approx] - wt[approx]) > RRE_REL * np.abs(wt[approx])).any():
        bad.append("totals")
    return bad


def raw(dev, pts, count, matches, n_matches, pairs, G, info, flags, poses, levels, **opt):
    """The entry point itself, on outputs filled with sentinels: every element must be written."""
    import torch
    from d3feat_b200 import _lib
    lib = _lib.lib()
    opt = {**OPTS, **opt}
    pts = np.asarray(pts, np.float32)
    B, k = pts.shape[:2]
    P, L, R, S = len(pairs), matches.shape[1], len(levels), len(poses)
    i32 = lambda a: t(np.asarray(a, np.int32), dev)          # noqa: E731
    f64 = lambda a: t(np.asarray(a, np.float64), dev)        # noqa: E731
    tp, tc, tm, tn, tq, tG, tf = (t(pts, dev), i32(count), i32(matches), i32(n_matches), i32(pairs), f64(G),
                                  i32(flags))
    ti = None if info is None else f64(info)
    tT = [f64(T) for T in poses]
    full = lambda shape, dt: torch.full(shape, 7, dtype=dt, device=dev)  # noqa: E731
    out = dict(valid=full((P,), torch.int32), n_match_inliers=full((P,), torch.int32),
               inlier_ratio=full((P,), torch.float64), fmr_hit=full((P,), torch.int32),
               n_repeated=full((P, R), torch.int32), repeatability=full((P, R), torch.float64),
               rte=full((S, P), torch.float64), rre_deg=full((S, P), torch.float64), rmse2=full((S, P), torch.float64),
               success=full((S, P), torch.int32), recall_hit=full((S, P), torch.int32),
               totals=full((4 + R + 7 * S,), torch.float64))
    ws = _lib.workspace(lib.d3f_evaluate_pairs_workspace_bytes(P, S), dev)
    pp = (_lib.C.c_void_p * 2)(*[x.data_ptr() for x in tT])
    lv = (_lib.C.c_int * max(1, R))(*levels)
    o = [_lib.ptr(out[f]) if out[f].numel() else None for f in
         ("valid", "n_match_inliers", "inlier_ratio", "fmr_hit", "n_repeated", "repeatability", "rte", "rre_deg",
          "rmse2", "success", "recall_hit", "totals")]
    _lib.check(lib.d3f_evaluate_pairs(_lib.ptr(tp), _lib.ptr(tc), B, k, _lib.ptr(tm), _lib.ptr(tn), L, _lib.ptr(tq), P,
                                      _lib.ptr(tG), _lib.ptr(ti), _lib.ptr(tf), pp, S, lv, R, opt["fmr_distance"],
                                      opt["fmr_ratio"], opt["repeat_distance"], opt["err2"], opt["rte_max"],
                                      opt["rre_max_deg"], *o, _lib.ptr(ws), ws.numel(), _lib.stream()),
               "d3f_evaluate_pairs")
    return {f: v.cpu().numpy() for f, v in out.items()}


def check(dev, pts, count, matches, n_matches, pairs, G, info, flags, poses, levels, **opt):
    got = raw(dev, pts, count, matches, n_matches, pairs, G, info, flags, poses, levels, **opt)
    want = evaluate_np.evaluate(pts, count, matches, n_matches, pairs, G, info, flags, poses, levels=levels,
                                **{**OPTS, **opt})
    assert mismatches(got, want, len(levels), len(poses)) == []
    return want


# ---- inputs -------------------------------------------------------------------------------------------------------

def rotation(axis, deg):
    axis = np.asarray(axis, float)
    axis = axis / np.linalg.norm(axis)
    th = np.deg2rad(deg)
    K = np.array([[0, -axis[2], axis[1]], [axis[2], 0, -axis[0]], [-axis[1], axis[0], 0]])
    return np.eye(3) + np.sin(th) * K + (1 - np.cos(th)) * K @ K


def rigid(R, tr):
    T = np.eye(4)
    T[:3, :3], T[:3, 3] = R, tr
    return T


def info_matrices(P):
    import os
    from d3feat_b200 import io_utils
    _, info = io_utils.load_info(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "hotel3_gt.info"))
    return info[np.arange(P) % len(info)]


def make_case(rng, k, counts, pairs, poison=np.nan, noise=0.03, extent=2.0):
    """Clouds b = T_b(base) with noise and a partial slot shuffle (slots past count[b] hold `poison`); truth of pair
    (a, b) = T_b inv(T_a); mutual-looking matches with wrong and out-of-range rows; two pose sets: perturbed truths
    (some KITTI successes, some failures) and the exact truth (the clamp)."""
    B = len(counts)
    base = rng.uniform(0, extent, (k, 3))
    Ts = [rigid(rotation(rng.normal(size=3), rng.uniform(0, 60)), rng.uniform(-2, 2, 3)) for _ in range(B)]
    pts = np.full((B, k, 3), poison, np.float32)
    perms = []
    for b in range(B):
        perm = np.arange(k)
        sw = rng.choice(k, size=(k // 3, 2))
        for x, y in sw:
            perm[x], perm[y] = perm[y], perm[x]
        perms.append(perm)
        c = min(max(int(counts[b]), 0), k)
        moved = base[perm] @ Ts[b][:3, :3].T + Ts[b][:3, 3] + rng.normal(scale=noise, size=(k, 3))
        pts[b, :c] = moved[:c]
    P = len(pairs)
    G = np.tile(np.eye(4), (P, 1, 1))
    L = k
    matches = np.full((P, L, 2), -1, np.int64)
    n_m = np.zeros(P, np.int64)
    for p, (a, b) in enumerate(pairs):
        if 0 <= a < B and 0 <= b < B:
            G[p] = Ts[b] @ np.linalg.inv(Ts[a])
            inv_b = np.argsort(perms[b])
            i = np.sort(rng.choice(k, size=int(rng.integers(0, k + 1)), replace=False))
            j = inv_b[perms[a][i]]
            wrong = rng.random(len(i)) < 0.3
            j = np.where(wrong, rng.integers(-1, k + 1, len(i)), j)
            matches[p, :len(i)] = np.stack([i, j], 1)
            n_m[p] = len(i)
    n_m[::7] += 5                       # past L: clamped
    n_m[3::11] = -4                     # negative: no matches
    est = np.stack([rigid(rotation(rng.normal(size=3), rng.uniform(0, 9)), rng.normal(scale=1.5, size=3)) @ g
                    for g in G])
    return pts, np.asarray(counts), matches, n_m, G, [est, G.copy()]


# ---- 1. k in {1, 250, 5000}, counts {0, 1, k - 1, k}, levels above and below the counts -----------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("k,levels", [(1, (1,)), (250, (1, 4, 64, 249, 250)), (250, (4, 8, 16, 32, 64, 128)),
                                      (5000, (4, 512, 4999, 5000))])
def test_evaluate_pairs_counts_and_levels(cuda, k, levels):
    rng = np.random.default_rng(k + len(levels))
    counts = [0, 1, max(k - 1, 0), k, k + 3, -2]
    B = len(counts)
    if k == 5000:
        pairs = [(2, 3), (3, 2), (3, 3), (1, 3), (3, 0), (4, 2), (-1, 3), (3, B)]
    else:
        pairs = [(a, b) for a in range(B) for b in range(B)] + [(-1, 0), (0, B)]
    pts, cnt, matches, n_m, G, poses = make_case(rng, k, counts, pairs)
    flags = rng.choice([0, 1, 3, 3], len(pairs))
    flags[:4] = 3
    want = check(cuda, pts, cnt, matches, n_m, pairs, G, info_matrices(len(pairs)), flags, poses, levels)
    assert want["n_repeated"].max() > 0 or k == 1
    if k > 1:
        assert want["fmr_hit"].any() and want["success"].any() and want["recall_hit"].any()
        assert (want["success"][0] == 0).sum() > (want["valid"] == 0).sum()


# ---- 2. NaN / inf keypoints, poisoned slots, bad pair ids, flags, no info, a NaN truth ------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("poison", [np.nan, np.inf, 1e3])
def test_evaluate_pairs_non_finite_inputs_and_bad_ids(cuda, poison):
    rng = np.random.default_rng(5)
    k = 96
    counts = [96, 90, 96, 50]
    pairs = [(0, 1), (1, 0), (0, 2), (2, 3), (3, 0), (-1, 1), (0, 4), (4, 4), (1, 2), (2, 1)]
    pts, cnt, matches, n_m, G, poses = make_case(rng, k, counts, pairs, poison=poison)
    pts[0, 5] = np.nan                  # NaN and inf in real slots
    pts[1, 80, 1] = np.inf
    pts[2, 95] = -np.inf
    G[8] = np.nan                       # device truth: evaluated, a miss in every test
    G[9, 0, 0] = np.inf
    poses[0][3, 1, 1] = np.inf          # a non-finite pose: NaN metrics
    flags = np.array([3, 3, 1, 3, 0, 3, 3, 1, 3, 3])
    info = info_matrices(len(pairs))
    for inf_ in (info, None):
        want = check(cuda, pts, cnt, matches, n_m, pairs, G, inf_, flags, poses, (4, 8, 32, 64, 90, 96))
        assert want["valid"].tolist() == [1, 1, 1, 1, 0, 0, 0, 0, 1, 1]
        assert want["n_match_inliers"][8:].sum() == 0 and want["n_repeated"][8:].sum() == 0
        assert want["success"][:, 8:].sum() == 0 and want["recall_hit"][:, 8:].sum() == 0
        assert np.isnan(want["rte"][:, 8:]).all() and np.isnan(want["rte"][0, 3])
    # poison past the count is never read: the same inputs with zeros there give the same bits
    pts0 = pts.copy()
    for b, c in enumerate(counts):
        pts0[b, c:] = 0
    a = raw(cuda, pts, cnt, matches, n_m, pairs, G, info, flags, poses, (4, 96))
    b = raw(cuda, pts0, cnt, matches, n_m, pairs, G, info, flags, poses, (4, 96))
    assert all(same_bits(a[f], b[f]) for f in a)


@pytest.mark.gpu
@pytest.mark.parametrize("S,R", [(0, 0), (1, 0), (0, 3), (2, 14)])
def test_evaluate_pairs_without_levels_or_poses(cuda, S, R):
    rng = np.random.default_rng(17)
    k = 64
    pairs = [(0, 1), (1, 2), (2, 0), (1, 1)]
    pts, cnt, matches, n_m, G, poses = make_case(rng, k, [64, 60, 33], pairs)
    levels = tuple(range(1, 64, 4))[:R] if R <= 3 else tuple(range(4, 4 + 4 * R, 4))
    check(cuda, pts, cnt, matches, n_m, pairs, G, info_matrices(4), [3, 1, 3, 3], poses[:S], levels)


# ---- 3. B = 1024 clouds, P = 4096 pairs: the sequential totals -------------------------------------------------------

@pytest.mark.gpu
def test_evaluate_pairs_many_clouds_and_pairs(cuda):
    rng = np.random.default_rng(1024)
    k, B, P = 32, 1024, 4096
    counts = rng.integers(0, k + 1, B)
    counts[::97] = k
    pairs = np.stack([rng.integers(-1, B + 1, P), rng.integers(0, B, P)], 1)
    pts, cnt, matches, n_m, G, poses = make_case(rng, k, counts, [tuple(p) for p in pairs], extent=1.0)
    flags = rng.choice([0, 1, 3], P)
    want = check(cuda, pts, cnt, matches, n_m, pairs, G, info_matrices(P), flags, poses, (4, 8, 16, 32))
    assert want["totals"][0] > 2000 and want["totals"][1] > 0


# ---- 4. the Python API and a captured graph replayed on rewritten inputs ----------------------------------------------

@pytest.mark.gpu
def test_evaluate_pairs_python_api_and_cuda_graph(cuda):
    import torch
    from d3feat_b200.evaluation import GroundTruth, evaluate_pairs
    from d3feat_b200.keypoints import KeypointSet
    from d3feat_b200.matching import Matches
    from d3feat_b200.registration import Refinement, Registration
    rng = np.random.default_rng(33)
    k = 250
    pairs = [(0, 1), (0, 2), (1, 2), (2, 1)]
    fields = ("valid", "n_match_inliers", "inlier_ratio", "fmr_hit", "n_repeated", "repeatability", "rte", "rre_deg",
              "rmse2", "success", "recall_hit", "totals")

    def inputs(seed):
        r = np.random.default_rng(seed)
        return make_case(r, k, [250, 249, 200], pairs)
    pts, cnt, matches, n_m, G, poses = inputs(1)
    info = info_matrices(4)
    flags = np.array([3, 3, 1, 3])
    tp, tc, tm, tn = t(pts, cuda), t(cnt.astype(np.int32), cuda), t(matches.astype(np.int32), cuda), \
        t(n_m.astype(np.int32), cuda)
    tG, tf, ti = t(G, cuda), t(flags.astype(np.int32), cuda), t(info, cuda)
    t0, t1 = t(poses[0], cuda), t(poses[1], cuda)
    kp = KeypointSet(None, tc, tp, None, None)
    m = Matches(None, None, None, None, tm, tn)
    reg, ref = Registration(t0, None, None, None, None), Refinement(t1, None, None, None, None)

    def as_np(ev):
        return {f: getattr(ev, f).cpu().numpy() for f in fields}

    def want_of(pts, cnt, matches, n_m, G, flags, poses, levels, **kw):
        return evaluate_np.evaluate(pts, cnt, matches, n_m, pairs, G, info, flags, poses, levels=levels, **{**OPTS, **kw})
    # host truth and the default levels (4 .. 128 at k = 250)
    ev = evaluate_pairs(kp, m, pairs, GroundTruth(G, info, flags), reg, ref)
    assert mismatches(as_np(ev), want_of(pts, cnt, matches, n_m, G, flags, poses, (4, 8, 16, 32, 64, 128)), 6, 2) == []
    ev = evaluate_pairs(kp, m, pairs, GroundTruth(tG, None, tf), reg, None, repeat_distance=0.5, repeat_levels=[250])
    want = evaluate_np.evaluate(pts, cnt, matches, n_m, pairs, G, None, flags, poses[:1], levels=(250,),
                                **{**OPTS, "repeat_distance": 0.5})
    assert mismatches(as_np(ev), want, 1, 1) == []
    bad = G.copy()
    bad[1, 0, 3] = np.nan
    with pytest.raises(ValueError, match="non-finite"):
        evaluate_pairs(kp, m, pairs, GroundTruth(bad, info, flags), reg, ref)
    with pytest.raises(ValueError, match="outside"):
        evaluate_pairs(kp, m, [(0, 3)] * 4, GroundTruth(G, info, flags), reg, ref)
    # a captured graph replayed on inputs rewritten in place
    truth = GroundTruth(tG, ti, tf)
    tq = t(np.array(pairs, np.int32), cuda)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        evaluate_pairs(kp, m, tq, truth, reg, ref)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        ev = evaluate_pairs(kp, m, tq, truth, reg, ref)
    for trial in range(3):
        pts, cnt, matches, n_m, G, poses = inputs(10 + trial)
        flags = np.array([[3, 3, 1, 3], [1, 0, 3, 3], [0, 3, 3, 1]][trial])
        for dst, src in ((tp, pts), (tc, cnt.astype(np.int32)), (tm, matches.astype(np.int32)),
                         (tn, n_m.astype(np.int32)), (tG, G), (tf, flags.astype(np.int32)), (t0, poses[0]),
                         (t1, poses[1])):
            dst.copy_(t(src, cuda))
        g.replay()
        torch.cuda.synchronize()
        want = want_of(pts, cnt, matches, n_m, G, flags, poses, (4, 8, 16, 32, 64, 128))
        assert mismatches(as_np(ev), want, 6, 2) == [], trial


# ---- 5. GraphPipeline(..., register, icp, evaluate) over two encoder streams ----------------------------------------

LIMITS = [35, 33, 34, 36, 30]


def moved_copy(rng, pts, keep=0.85, noise=0.002, deg=3.0):
    T = rigid(rotation(rng.normal(size=3), deg), rng.uniform(-0.2, 0.2, 3))
    d = rng.normal(size=3)
    proj = pts @ d
    part = pts[proj <= np.quantile(proj, keep)]
    return (part @ T[:3, :3].T + T[:3, 3] + rng.normal(scale=noise, size=part.shape)).astype(np.float32), T


@pytest.mark.gpu
def test_graph_pipeline_evaluate_running_totals(cuda):
    """Seven batches of three clouds through one bucket on two encoder streams, each with its own truth (host or
    device, info or not, changing flags). Each step's evaluation equals the oracle on that step's keypoints, matches
    and poses; the running totals equal the step totals summed in step order, which a race between the overlapping
    encoders would break."""
    import torch
    from d3feat_b200 import synth
    from d3feat_b200.encoder import KPFCNN, EvaluatedDetections, GraphPipeline
    from d3feat_b200.evaluation import GroundTruth
    cfg = synth.Config(architecture=synth.ARCH_3DMATCH)
    enc = KPFCNN(cfg, synth.make_params(cfg, 5), LIMITS, device=cuda)
    rng = np.random.default_rng(21)
    pairs = [(0, 1), (0, 2), (1, 2)]
    info = info_matrices(3)
    batches = []
    for i, n in enumerate([9000, 8500, 9000, 7000, 8800, 8000, 9000]):
        base = synth.room_fragment(400 + i, n)
        c1, T1 = moved_copy(rng, base, keep=0.9)
        c2, T2 = moved_copy(rng, base, keep=0.8)
        G = np.stack([T1, T2, T2 @ np.linalg.inv(T1)])
        flags = np.array([[3, 3, 3], [1, 3, 0], [3, 1, 1]][i % 3], np.int32)
        truth = GroundTruth(G, info if i % 2 == 0 else None, flags)
        if i % 3 == 1:
            truth = GroundTruth(t(G, cuda), None if truth.info is None else t(info, cuda), t(flags, cuda))
        clouds = [base, c1, c2]
        batches.append((np.concatenate(clouds, 0), np.array([len(c) for c in clouds], np.int32), truth))
    reg = dict(distance=0.5, edge_ratio=0.5, ransac_n=4, max_iterations=2000, max_validation=200)
    ev_opts = dict(repeat_levels=[4, 16, 64, 250], rte_max=0.5, rre_max_deg=10.0)
    pipe = GraphPipeline.for_batch(enc, t(batches[0][0], cuda), t(batches[0][1], cuda), slack=1.2, decoder=True,
                                   keypoints=250, match_pairs=pairs, register=reg, icp=dict(distance=0.3),
                                   evaluate=ev_opts, encoder_streams=2)
    with pytest.raises(ValueError, match="truth"):
        pipe.prime(t(batches[0][0], cuda), t(batches[0][1], cuda))
    pipe.prime(t(batches[0][0], cuda), t(batches[0][1], cuda), truth=batches[0][2])
    steps = []
    for i in range(len(batches)):
        nxt = batches[i + 1] if i + 1 < len(batches) else None
        res, _ = pipe.step(t(nxt[0], cuda), t(nxt[1], cuda), next_truth=nxt[2]) if nxt else pipe.step()
        assert isinstance(res, EvaluatedDetections)
        kp, m, ev = res.keypoints, res.matches, res.evaluation
        steps.append(dict(points=kp.points.cpu().numpy(), count=kp.count.cpu().numpy(),
                          matches=m.matches.cpu().numpy(), n_matches=m.n_matches.cpu().numpy(),
                          poses=[res.registration.pose.cpu().numpy(), res.refinement.pose.cpu().numpy()],
                          ev={f: getattr(ev, f).cpu().numpy() for f in ev._fields}))
    pipe.check()
    running = pipe.evaluation_totals()
    acc = np.zeros_like(running)
    want_acc = np.zeros_like(running)
    for i, st in enumerate(steps):
        tr = batches[i][2]
        G = tr.pose.cpu().numpy() if hasattr(tr.pose, "cpu") else tr.pose
        inf_ = None if tr.info is None else info
        flags = tr.flags.cpu().numpy() if hasattr(tr.flags, "cpu") else tr.flags
        want = evaluate_np.evaluate(st["points"], st["count"], st["matches"], st["n_matches"], pairs, G, inf_, flags,
                                    st["poses"], levels=(4, 16, 64, 250),
                                    **{**OPTS, "rte_max": 0.5, "rre_max_deg": 10.0})
        assert mismatches(st["ev"], want, 4, 2) == [], i
        acc = acc + st["ev"]["totals"]
        want_acc = want_acc + want["totals"]
    assert same_bits(running, acc)
    approx = rre_sum_lanes(4, 2)
    exact = [j for j in range(len(acc)) if j not in approx]
    assert same_bits(running[exact], want_acc[exact])
    assert (np.abs(running[approx] - want_acc[approx]) <= RRE_REL * np.abs(want_acc[approx])).all()
    assert running[0] == sum(int((b[2].flags.cpu().numpy() if hasattr(b[2].flags, "cpu") else b[2].flags)
                                 .astype(bool).sum()) for b in batches)
    pipe.reset_evaluation()
    assert (pipe.evaluation_totals() == 0).all()
    torch.cuda.synchronize()


@pytest.mark.gpu
def test_graph_pipeline_evaluate_known_answer(cuda):
    """A cloud and a copy translated by an exactly representable offset register as a KITTI success against the
    translation as truth, and fail against its inverse: the source-to-target convention, end to end. The synthetic
    weights give uninformative descriptors, so the RANSAC pose is only near the truth (rte 0.045 m, rre 4.74 degrees
    on an H100); ICP over the two clouds brings it to the translation, and these thresholds are set from that run."""
    from d3feat_b200 import synth
    from d3feat_b200.encoder import KPFCNN, GraphPipeline
    from d3feat_b200.evaluation import GroundTruth, summary
    cfg = synth.Config(architecture=synth.ARCH_3DMATCH)
    enc = KPFCNN(cfg, synth.make_params(cfg, 7), LIMITS, device=cuda)
    a = np.round(synth.room_fragment(77, 8000) * 4096.0) / 4096.0
    off = np.array([1.5, 1.0, 0.0])
    b = a + off
    assert np.array_equal((a.astype(np.float32) + off.astype(np.float32)), b.astype(np.float32))
    pts = np.concatenate([a, b]).astype(np.float32)
    lens = np.array([len(a), len(b)], np.int32)
    G = rigid(np.eye(3), off)[None]
    pipe = GraphPipeline.for_batch(enc, t(pts, cuda), t(lens, cuda), slack=1.2, decoder=True, keypoints=250,
                                   match_pairs=[(0, 1)], register=dict(ransac_n=4, distance=0.05, max_iterations=5000),
                                   icp=dict(distance=0.3, max_iterations=100), evaluate={})
    flags = np.array([1], np.int32)
    pipe.prime(t(pts, cuda), t(lens, cuda), truth=GroundTruth(G, None, flags))
    fields = ("rte", "rre_deg", "success", "fmr_hit")
    r1, _ = pipe.step(t(pts, cuda), t(lens, cuda), next_truth=GroundTruth(np.linalg.inv(G[0])[None], None, flags))
    e1 = {f: getattr(r1.evaluation, f).cpu().numpy() for f in fields}
    r2, _ = pipe.step()
    e2 = {f: getattr(r2.evaluation, f).cpu().numpy() for f in fields}
    pipe.check()
    print("known answer: RANSAC rte %.3g m rre %.3g deg, ICP rte %.3g m rre %.3g deg; inverted truth: rte %.3g m" % (
        e1["rte"][0, 0], e1["rre_deg"][0, 0], e1["rte"][1, 0], e1["rre_deg"][1, 0], e2["rte"][0, 0]))
    assert (e1["success"][:, 0] == 1).all() and e1["fmr_hit"][0] == 1
    assert e1["rte"][0, 0] < 0.1 and e1["rte"][1, 0] < 0.01 and e1["rre_deg"][1, 0] < 0.5
    assert (e2["success"][:, 0] == 0).all() and e2["fmr_hit"][0] == 0 and (e2["rte"][:, 0] > 3.5).all()
    s = summary(pipe.evaluation_totals(), pipe.evaluate_levels, pipe.evaluate_pose_sets)
    assert s["n_pairs"] == 2 and s["fmr_hits"] == 1
    assert s["ransac"]["successes"] == 1 and s["icp"]["successes"] == 1
