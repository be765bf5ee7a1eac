"""Random keypoints (d3f_sample_keypoints, keypoints.sample_keypoints) and the keypoint sweep of
GraphPipeline(..., sweep=...) on the GPU.

* The sampler against oracle/keypoints_np.py, bit for bit: up to 1024 clouds with empty and one-point clouds, rows of
  no cloud, the static form with a device row count (eager and replayed from a CUDA graph), the prefix property.
* A 3DMatch-shaped scene batch (every i < j pair, with truth, register={}, evaluate={}): for every count, the score arm
  equals a separate pipeline built with keypoints=count -- keypoints, matches, poses, per-pair evaluation and running
  totals -- and the random arm equals the existing ops called on the oracle's prefix set.
* A KITTI-shaped pair with ICP over six steps (every slot captured, then replayed): every (arm, count) equals the eager
  chain of the existing ops on that step's network outputs. Two runs give the same bits; another seed other draws.
* A batch with a cloud wider than the scene bounds marks the pipeline, as tests/test_gpu_bucket_overflow.py checks for
  the single-count path: check() and evaluation_totals() raise, also after reset_evaluation()."""
import numpy as np
import pytest

from oracle import keypoints_np

LIMITS = [35, 33, 34, 36, 30]


def t(a, dev):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def same(a, b):
    """Bit-identical arrays (NaN payloads included)."""
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and a.dtype == b.dtype and a.tobytes() == b.tobytes()


def flat(entry):
    """{"stage.field": numpy} of a SweepEntry / result namedtuple (stages that did not run are left out)."""
    import torch
    out = {}
    for name in entry._fields:
        stage = getattr(entry, name)
        if stage is None or name == "sweep":
            continue
        if torch.is_tensor(stage):
            out[name] = stage.cpu().numpy()
            continue
        for f in stage._fields:
            x = getattr(stage, f)
            if x is not None:
                out["%s.%s" % (name, f)] = x.cpu().numpy()
    return out


def assert_same(got, want, what):
    assert set(got) == set(want), (what, sorted(set(got) ^ set(want)))
    bad = [f for f in got if not same(got[f], want[f])]
    assert bad == [], (what, bad)


# ---- 1. the sampler against the oracle ------------------------------------------------------------------------------

def stack_case(rng, B, tail=13, D=32):
    lens = rng.integers(0, 60, B).astype(np.int32)
    lens[rng.random(B) < 0.15] = 0
    lens[rng.random(B) < 0.15] = 1
    if B > 1:
        lens[0], lens[-1] = 0, 1
    N = int(lens.sum()) + tail                      # `tail` rows of no cloud
    pts = rng.normal(size=(N, 3)).astype(np.float32)
    desc = rng.normal(size=(N, D)).astype(np.float32)
    scores = rng.normal(size=(N, 1)).astype(np.float32)
    return lens, pts, desc, scores


def check_against_oracle(kp, lens, k, seed, n, pts, desc, scores):
    idx, cnt = keypoints_np.sample_keypoints(lens, k, seed, n)
    assert same(kp.index.cpu().numpy(), idx)
    assert same(kp.count.cpu().numpy(), cnt)
    for got, rows in ((kp.points, pts), (kp.descriptors, desc), (kp.scores, None if scores is None else scores[:, 0])):
        if rows is None:
            assert got is None
        else:
            assert same(got.cpu().numpy(), keypoints_np.gather(idx, rows))
    return idx


@pytest.mark.gpu
@pytest.mark.parametrize("B,k,D", [(1, 1, 32), (1, 5000, 32), (17, 250, 7), (1024, 37, 32)])
def test_sample_keypoints_matches_the_oracle(cuda, B, k, D):
    from d3feat_b200.keypoints import sample_keypoints
    rng = np.random.default_rng(B * 31 + k)
    lens, pts, desc, scores = stack_case(rng, B, D=D)
    for seed in (0, 9, (1 << 64) - 1):
        kp = sample_keypoints(t(lens, cuda), k, seed, points=t(pts, cuda), descriptors=t(desc, cuda),
                              scores=t(scores, cuda))
        idx = check_against_oracle(kp, lens, k, seed, len(pts), pts, desc, scores)
        assert (idx < int(lens.sum())).all()        # the rows of no cloud are never drawn
    # index and count alone, no rows to gather: the clouds are not cut
    kp = sample_keypoints(t(lens, cuda), k, 3)
    check_against_oracle(kp, lens, k, 3, 2 ** 31 - 1, None, None, None)


@pytest.mark.gpu
def test_sample_keypoints_prefix_and_seeds(cuda):
    from d3feat_b200.keypoints import sample_keypoints
    rng = np.random.default_rng(5)
    lens, pts, desc, scores = stack_case(rng, 64)
    args = dict(points=t(pts, cuda), descriptors=t(desc, cuda), scores=t(scores, cuda))
    big = flat(sample_keypoints(t(lens, cuda), 5000, 11, **args))
    again = flat(sample_keypoints(t(lens, cuda), 5000, 11, **args))
    assert_same(again, big, "repeat")
    for c in (2500, 1000, 500, 250, 1):
        small = flat(sample_keypoints(t(lens, cuda), c, 11, **args))
        for f, a in small.items():
            want = np.minimum(big[f], c) if f == "count" else big[f][:, :c]
            assert same(a, want), (c, f)
    other = sample_keypoints(t(lens, cuda), 5000, 12, **args).index.cpu().numpy()
    assert not np.array_equal(other, big["index"])


@pytest.mark.gpu
def test_sample_keypoints_static_rows_and_graph(cuda):
    """Capacity-sized inputs with the row count in device memory: clouds cut at the count, or rows of no cloud past the
    last one. The same call captured once and replayed with new lengths and counts follows them."""
    import torch
    from d3feat_b200.keypoints import sample_keypoints
    rng = np.random.default_rng(8)
    lens, pts, desc, scores = stack_case(rng, 40, tail=0)
    cap = len(pts) + 50
    pad = lambda a: np.concatenate([a, np.full((cap - len(a),) + a.shape[1:], np.nan, np.float32)])  # noqa: E731
    pts, desc, scores = pad(pts), pad(desc), pad(scores)
    tp, td, ts = t(pts, cuda), t(desc, cuda), t(scores, cuda)
    total = int(lens.sum())
    for n in (total + 30, total, total - 45, int(np.cumsum(lens)[20])):
        rows = torch.tensor([n], dtype=torch.int32, device=cuda)
        kp = sample_keypoints(t(lens, cuda), 300, 4, points=tp, descriptors=td, scores=ts, rows=rows)
        check_against_oracle(kp, lens, 300, 4, n, pts, desc, scores)
    tl = t(lens, cuda)
    rows = torch.tensor([total], dtype=torch.int32, device=cuda)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        sample_keypoints(tl, 300, 4, points=tp, descriptors=td, scores=ts, rows=rows)
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        kp = sample_keypoints(tl, 300, 4, points=tp, descriptors=td, scores=ts, rows=rows)
    for trial in range(3):
        new = rng.permutation(lens).astype(np.int32)
        n = total - 17 * trial
        tl.copy_(t(new, cuda))
        rows.fill_(n)
        g.replay()
        torch.cuda.synchronize()
        check_against_oracle(kp, new, 300, 4, n, pts, desc, scores)


# ---- 2. pipelines -----------------------------------------------------------------------------------------------------

def encoder(cuda, seed):
    from d3feat_b200 import synth
    from d3feat_b200.encoder import KPFCNN
    cfg = synth.Config(architecture=synth.ARCH_3DMATCH)
    return KPFCNN(cfg, synth.make_params(cfg, seed), LIMITS, device=cuda)


def scene(seed, n_clouds, n_points, keep=0.85):
    """A fragment and n_clouds - 1 partial moved copies of it, with the truth of every i < j pair (3DMatch flags:
    registration recall for j - i > 1), as (points, lengths, pairs, GroundTruth)."""
    from d3feat_b200 import synth
    from d3feat_b200.evaluation import GroundTruth
    from test_gpu_evaluation import info_matrices, moved_copy
    rng = np.random.default_rng(seed)
    base = synth.room_fragment(seed, n_points)
    clouds, Ts = [base], [np.eye(4)]
    for _ in range(n_clouds - 1):
        c, T = moved_copy(rng, base, keep=keep)
        clouds.append(c)
        Ts.append(T)
    pairs = [(a, b) for a in range(n_clouds) for b in range(a + 1, n_clouds)]
    G = np.stack([Ts[b] @ np.linalg.inv(Ts[a]) for a, b in pairs])
    flags = np.array([3 if b - a > 1 else 1 for a, b in pairs], np.int32)
    truth = GroundTruth(G, info_matrices(len(pairs)), flags)
    return (np.ascontiguousarray(np.concatenate(clouds, 0), np.float32),
            np.array([len(c) for c in clouds], np.int32), pairs, truth)


def run_steps(pipe, batches, on_step=None):
    """prime + one step per batch; returns the flattened result of every step (main result and every sweep entry).
    on_step(i, k, res) runs right after step i, while slot k still holds it."""
    import torch
    cuda = pipe.enc.device
    P, L, _, T = batches[0]
    pipe.prime(t(P, cuda), t(L, cuda), truth=T)
    out = []
    for i in range(len(batches)):
        k = pipe.pending
        nxt = batches[i + 1] if i + 1 < len(batches) else None
        res, _ = pipe.step(t(nxt[0], cuda), t(nxt[1], cuda), next_truth=nxt[3]) if nxt else pipe.step()
        torch.cuda.synchronize()
        snap = {"main": flat(res)}
        for key, e in getattr(res, "sweep", {}).items():
            snap[key] = flat(e)
        if on_step is not None:
            on_step(i, k, res)
        out.append(snap)
    pipe.drain()
    return out


def eager_entry(pipe, k, res, arm, c):
    """The existing ops on step k's network outputs: the arm's keypoints (select_keypoints, or the oracle's prefix
    set gathered on the host), then match_keypoints, register_pairs, icp_pairs and evaluate_pairs with the pipeline's
    options."""
    import torch
    from d3feat_b200.encoder import SweepEntry
    from d3feat_b200.evaluation import evaluate_pairs
    from d3feat_b200.keypoints import KeypointSet, select_keypoints
    from d3feat_b200.matching import match_keypoints
    from d3feat_b200.registration import icp_pairs, register_pairs
    inputs = pipe.out[k][0]
    pts, lens, rows = inputs["points"][0], inputs["lengths"][0], inputs["rows"][0]
    if arm == "score":
        kp = select_keypoints(res.scores, lens, c, points=pts, descriptors=res.descriptors, rows=rows)
    else:
        idx, cnt = keypoints_np.sample_keypoints(lens.cpu().numpy(), pipe.sweep_counts[0], pipe.sweep_seed,
                                                 int(rows.item()))
        idx, cnt = idx[:, :c], np.minimum(cnt, c)
        g = lambda x: t(keypoints_np.gather(idx, x.cpu().numpy()), pts.device)   # noqa: E731
        kp = KeypointSet(t(idx, pts.device), t(cnt, pts.device), g(pts), g(res.descriptors),
                         g(res.scores.reshape(-1)))
    m = match_keypoints(kp, pipe.match_pairs)
    reg = ref = ev = None
    if pipe.register is not None:
        reg = register_pairs(kp, m, pipe.match_pairs, **pipe.register)
        if pipe.icp is not None:
            ref = icp_pairs(pts, lens, pipe.match_pairs, reg.pose, rows=rows, bbox=pipe.bbox, **pipe.icp)
    if pipe.evaluate is not None:
        ev = evaluate_pairs(kp, m, pipe.match_pairs, pipe.truth[k], reg, ref, **pipe.evaluate)
    torch.cuda.synchronize()
    return flat(SweepEntry(kp, m, reg, ref, ev))


def check_eager(pipe, failures):
    """on_step callback: every sweep entry of the step against eager_entry."""
    def on_step(i, k, res):
        for (arm, c), e in res.sweep.items():
            got, want = flat(e), eager_entry(pipe, k, res, arm, c)
            bad = sorted(f for f in set(got) | set(want) if f not in got or f not in want or not same(got[f], want[f]))
            if bad:
                failures.append((i, arm, c, bad))
    return on_step


def stepwise_totals(snaps, arms, counts):
    acc = None
    for s in snaps:
        tot = np.stack([np.stack([s[(a, c)]["evaluation.totals"] for c in counts]) for a in arms])
        acc = tot if acc is None else acc + tot
    return acc


@pytest.fixture(scope="module")
def room_batches():
    """Two 3DMatch-shaped scene batches of five 6000-point fragments, every i < j pair with truth."""
    return [scene(300 + i, 5, 6000) for i in range(2)]


@pytest.mark.gpu
def test_score_arm_equals_separate_pipelines(cuda, room_batches):
    from d3feat_b200.encoder import GraphPipeline
    from d3feat_b200.evaluation import summary, sweep_summary
    enc = encoder(cuda, 3)
    P0, L0, pairs, _ = room_batches[0]
    counts, arms = (500, 250, 100), ("score", "random")
    pipe = GraphPipeline.for_batch(enc, t(P0, cuda), t(L0, cuda), slack=1.2, decoder=True, keypoints=500,
                                   match_pairs=pairs, register={}, evaluate={},
                                   sweep=dict(counts=counts, arms=arms, seed=7))
    assert pipe.evaluate_levels == (4, 8, 16, 32, 64)        # the default levels clipped to the smallest count
    failures = []
    snaps = run_steps(pipe, room_batches, check_eager(pipe, failures))
    assert failures == []
    pipe.check()
    totals = pipe.evaluation_totals()
    assert totals.shape == (2, 3, 4 + 5 + 7)
    assert same(totals, stepwise_totals(snaps, arms, counts))
    for i in range(len(room_batches)):                       # count == keypoints: the regular result itself
        assert_same({f: v for f, v in snaps[i]["main"].items() if f not in ("descriptors", "scores")},
                    snaps[i][("score", 500)], "main, step %d" % i)
    for j, c in enumerate(counts):
        sep = GraphPipeline.for_batch(enc, t(P0, cuda), t(L0, cuda), slack=1.2, decoder=True, keypoints=c,
                                      match_pairs=pairs, register={},
                                      evaluate=dict(repeat_levels=pipe.evaluate_levels))
        ref = run_steps(sep, room_batches)
        sep.check()
        for i in range(len(room_batches)):
            assert_same(snaps[i][("score", c)], {f: v for f, v in ref[i]["main"].items()
                                                 if f not in ("descriptors", "scores")}, "score %d, step %d" % (c, i))
            assert same(snaps[i]["main"]["descriptors"], ref[i]["main"]["descriptors"])
        assert same(totals[0, j], sep.evaluation_totals()), c
    rows = sweep_summary(totals, pipe.sweep_arms, pipe.sweep_counts, pipe.evaluate_levels, pipe.evaluate_pose_sets)
    assert [(r["arm"], r["count"]) for r in rows] == [(a, c) for a in arms for c in counts]
    assert repr(rows[4]) == repr(dict(arm="random", count=250,
                                      **summary(totals[1, 1], pipe.evaluate_levels, ("ransac",))))
    for r in rows:
        print("%-6s %4d  FMR %.3f  inlier ratio %.4f  RR %.3f" % (r["arm"], r["count"], r["fmr"], r["avg_inlier_ratio"],
                                                                r["ransac"]["registration_recall"]))


def kitti_batches(n, seed0=50):
    return [scene(seed0 + i, 2, 5000, keep=0.9) for i in range(n)]


def kitti_pipe(enc, batch, seed=0, arms=("score", "random")):
    from d3feat_b200.encoder import GraphPipeline
    P0, L0, pairs, _ = batch
    return GraphPipeline.for_batch(enc, t(P0, enc.device), t(L0, enc.device), slack=1.3, decoder=True, keypoints=250,
                                   match_pairs=pairs, register=dict(ransac_n=4, distance=0.3, max_iterations=3000),
                                   icp=dict(distance=0.3, max_iterations=30), evaluate=dict(repeat_distance=0.5),
                                   sweep=dict(counts=(250, 120, 40), arms=arms, seed=seed))


@pytest.mark.gpu
def test_kitti_pair_with_icp_replayed_steps_equal_eager_calls(cuda):
    """Six steps through the four slots (each captured once, two replayed): every entry equals the eager chain, the
    running totals the step totals summed in order; a second run gives the same bits and another seed other draws."""
    enc = encoder(cuda, 4)
    batches = kitti_batches(6)
    pipe = kitti_pipe(enc, batches[0])
    failures = []
    snaps = run_steps(pipe, batches, check_eager(pipe, failures))
    assert failures == []
    pipe.check()
    assert pipe.evaluate_pose_sets == ("ransac", "icp")
    totals = pipe.evaluation_totals()
    assert same(totals, stepwise_totals(snaps, pipe.sweep_arms, pipe.sweep_counts))
    again = kitti_pipe(enc, batches[0])
    snaps2 = run_steps(again, batches)
    for i in range(len(batches)):
        for key in snaps[i]:
            assert_same(snaps2[i][key], snaps[i][key], "second run, step %d, %s" % (i, key))
    assert same(again.evaluation_totals(), totals)
    other = kitti_pipe(enc, batches[0], seed=1)
    snaps3 = run_steps(other, batches[:2])
    for i in range(2):
        assert_same(snaps3[i][("score", 120)], snaps[i][("score", 120)], "score arm, other seed")
        assert not same(snaps3[i][("random", 250)]["keypoints.index"], snaps[i][("random", 250)]["keypoints.index"])


@pytest.mark.gpu
def test_sweep_pipeline_marks_an_overflowing_batch(cuda):
    """A cloud scaled 60 times about its mean is wider than the scene bounds: the slot's status bit 0 is set, every
    output of the step stays finite, and check() and evaluation_totals() raise from then on."""
    enc = encoder(cuda, 4)
    batches = kitti_batches(3, seed0=80)
    P, L, pairs, T = batches[1]
    c = P[L[0]:]
    m = c.mean(0)
    wide = np.concatenate([P[:L[0]], m + (c - m) * np.float32(60.0)]).astype(np.float32)
    feed = [batches[0], (wide, L, pairs, T), batches[2]]
    pipe = kitti_pipe(enc, batches[0], arms=("random", "score"))
    snaps = run_steps(pipe, feed)
    st = [int(buf.status.item()) for buf in pipe.slots]
    assert st[1] & 1 and st[0] == st[2] == st[3] == 0, st
    for key, e in snaps[1].items():
        for f in ("keypoints.points", "keypoints.descriptors", "registration.pose", "refinement.pose"):
            if f in e:
                assert np.isfinite(e[f]).all(), (key, f)
    for _ in range(2):
        with pytest.raises(RuntimeError, match="status"):
            pipe.check()
        with pytest.raises(RuntimeError, match="status"):
            pipe.evaluation_totals()
        pipe.reset_evaluation()
