"""Batches of up to 1024 clouds through the half of the pipeline after the input pyramid: the encoder and the decoder,
the detection scores, the keypoints, the matching of cloud pairs, RANSAC and ICP -- in the eager exact path, in the
static form, and replayed by the captured serving loop (GraphPipeline) -- against the float64 and exact oracles.

The batches are those of tests/test_gpu_many_clouds.py (clouds of 0, 1, 2, 31, 32, 33 and a few hundred points, runs of
empty clouds, lattice ties, exact copies, lengths summing short of or past the row count), plus one one-point cloud and
1024 one-point clouds, with every fourth cloud replaced by a rigidly moved copy of the cloud before it so that the pair
(b - 1, b) has a pose to find. With k = 64 keypoints, clouds of 120 points and more select and smaller ones are padded;
a one-point cloud gives a keypoint set of count 1 that goes on to matching and to a RANSAC sample of 3.

Checks, for every batch:
* every traced op of the encoder and the decoder on its own inputs, element by element against float64 (tests/_trace.py);
* the descriptors against the float64 l2 normalisation of the traced last unary, and every detection score of a row
  that belongs to a cloud against the oracle (the score of a row of no cloud is unspecified);
* the keypoints: exactly the argsort oracle applied to the GPU's own scores, no index naming a row of no cloud;
* matching, registration and ICP on those keypoints: bit for bit against oracle/match_np.py, register_np.py, icp_np.py.
The captured loop then returns the eager static run bit for bit, and a step with no points at all (n0 = 0) between two
non-empty batches returns empty keypoint sets, no matches, unregistered pairs and refinements that keep their init.

The CPU tests at the end show that the new batches change the oracles' results under emulated bugs of the chain."""
import functools

import numpy as np
import pytest
import torch

from oracle import icp_np, kpconv_np as ok, match_np

from _oracle import TOL, assert_close
from _trace import check_sampled_rows, record_ops
from test_gpu_icp import as_numpy as icp_numpy, mismatches as icp_mismatches, moved_copy
from test_gpu_keypoints import bits, check_gathered, oracle as keypoint_oracle
from test_gpu_many_clouds import LIMITS, batch, clip_lengths, poisoned, scene, tail_batch
from test_gpu_registration import as_numpy as reg_numpy, mismatches as reg_mismatches, oracle_from_matches

K = 64
RTOL = 1e-4
SAMPLED_ROWS = 400
# the synthetic weights give uninformative descriptors: checkers as loose as test_graph_pipeline_register's, and few
# hypotheses so that the numpy oracle stays fast on a thousand pairs
REGISTER = dict(distance=0.5, edge_ratio=0.5, ransac_n=3, max_iterations=200, max_validation=20)
ICP = dict(distance=0.1, max_iterations=5)
TAIL_JITTER = np.float32([0.01, 0.0, 0.0])

CASES = ["B17", "B33", "B300", "B1024", "B1024_lone", "B1_one_point", "B1024_one_point",
         "B33_sum_N-37", "B33_sum_N+0", "B33_sum_N+37"]
MATCH_FIELDS = ("nn_st", "sim_st", "nn_ts", "sim_ts", "matches", "n_matches")


# ---- batches ----------------------------------------------------------------------------------------------------------

def with_moved_copies(P, L, seed):
    """Cloud b = 3, 7, 11, ... replaced by test_gpu_icp.moved_copy of cloud b - 1 (80 % of it, rotated by 3-10 degrees,
    shifted by up to 0.2 m per axis, 2 mm of noise) where both are non-empty, so that the empty runs and the lone
    cloud stay. Rows past the last cloud stay; a cloud cut by the row count is left as it is, so the lengths still sum
    to the same excess over the row count."""
    rng = np.random.default_rng(seed)
    Lc = clip_lengths(L, len(P))
    start = np.concatenate([[0], np.cumsum(Lc)])
    clouds = [P[start[b]:start[b + 1]] for b in range(len(L))]
    L = np.array(L, np.int32, copy=True)
    for b in range(3, len(L), 4):
        if Lc[b] == L[b] > 0 and Lc[b - 1] > 0:
            clouds[b], _ = moved_copy(rng, clouds[b - 1], deg=rng.uniform(3.0, 10.0))
            L[b] = len(clouds[b])
    P = np.concatenate(clouds + [P[start[-1]:]], 0)
    return np.ascontiguousarray(P, np.float32), L


@functools.lru_cache(maxsize=None)
def serving_batch(case, variant=0):
    """(points, lengths) of a case. "B<n>_one_point": n one-point clouds, random rows of the scene. "B33_sum_N<e>":
    tail_batch(33, e); short of the row count, the rows of no cloud are the last cloud's rows moved by 1 cm, so that a
    search reaching them finds them before (not tied with) the real rows. Other cases: batch(case, variant)."""
    if case.endswith("one_point"):
        B = int(case.split("_")[0][1:])
        room, _ = scene()
        rng = np.random.default_rng(7 * B + variant)
        P, L = room[rng.choice(len(room), B, replace=False)], np.ones(B, np.int32)
    elif "_sum_N" in case:
        excess = int(case.split("_sum_N")[1])
        P, L = tail_batch(int(case.split("_")[0][1:]), excess)
        P = P.copy()
        if excess < 0:
            P[len(P) + excess:] += TAIL_JITTER
    else:
        P, L = batch(case, variant)
    return with_moved_copies(P, L, seed=len(L) * 100 + variant)


def pairs_for(L):
    """Every (b, b + 1) (among them every (b - 1, moved copy)), a few (b, b), and the largest cloud paired both ways
    with the last cloud and with the first empty, one-point and two-point cloud."""
    B = len(L)
    big = int(np.argmax(L))
    pairs = [(b, b + 1) for b in range(B - 1)] + [(b, b) for b in sorted({B // 3, (2 * B) // 3, big, B - 1})]
    pairs += [(big, B - 1), (B - 1, big)]
    for size in (0, 1, 2):
        hit = np.nonzero(np.asarray(L) == size)[0]
        if len(hit):
            pairs += [(int(hit[0]), big), (big, int(hit[0]))]
    return pairs


# ---- checks shared by the eager exact path and the static form -------------------------------------------------------

def t(a, dev):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def report(rep, what):
    worst = {}
    for op, _, _, r in rep:
        worst[op] = max(worst.get(op, 0.0), r)
    print("%s: largest |err|/mag per op: %s" % (what, ", ".join("%s %.3e" % kv for kv in sorted(worst.items()))))


def check_chain(tr, P, L, n, desc, scores, kp, m, reg, ref, pairs, what, seed=0):
    """Every traced op, the descriptors, the scores, the keypoints, the matches, the registration and the refinement
    of one batch against the oracles. P: the batch's host points (n rows below the device count), L its lengths.
    Returns the oracle's registration and refinement."""
    rep = check_sampled_rows(tr, SAMPLED_ROWS, np.random.default_rng(seed), RTOL, min_kpconv=10, what=what)
    report(rep, what)
    rec = tr.records[-1]
    assert rec["op"] == "detection_scores" and tr.records[-2]["op"] == "unary"
    assert rec["features"] is tr.records[-2]["out"]
    n_real = int(clip_lengths(L, n).sum())
    x = rec["features"][:n].cpu().numpy().astype(np.float64)
    unit = x / np.sqrt(np.maximum((x * x).sum(1, keepdims=True), 1e-10))
    assert_close(desc[:n].cpu().numpy(), unit, np.abs(unit), TOL, "%s l2_normalize" % what)
    nbr = rec["neighbors"][:n].cpu().numpy()
    assert nbr.min(initial=0) >= 0 and nbr.max(initial=0) <= n
    s = scores[:n].cpu().numpy().reshape(-1)
    want, mag, alt = ok.detection_scores(x, nbr, rec["lengths"].cpu().numpy(), magnitude=True)
    assert_close(s[:n_real, None], want[:n_real], mag[:n_real], TOL, "%s detection_scores (rows of a cloud)" % what,
                 alt=alt[:n_real])
    # keypoints: the argsort oracle on the GPU's own scores
    idx, cnt = keypoint_oracle(s, L, K, n=n)
    assert np.array_equal(kp.index.cpu().numpy(), idx), what
    assert np.array_equal(kp.count.cpu().numpy(), cnt), what
    assert idx.max(initial=-1) < n_real, "%s: a keypoint names a row of no cloud" % what
    check_gathered(kp, idx, P[:n], desc[:n].cpu().numpy(), s)
    # matching, RANSAC and ICP on those keypoints
    pairs = np.asarray(pairs, np.int32)
    want_m = match_np.match(kp.descriptors.cpu().numpy(), kp.count.cpu().numpy(), pairs)
    for f in MATCH_FIELDS:
        got = getattr(m, f).cpu().numpy()
        if got.dtype == np.float32:
            got, want_m[f] = bits(got), bits(want_m[f])
        assert np.array_equal(got, want_m[f]), "%s: matches.%s" % (what, f)
    want_r, n_corr = oracle_from_matches(kp, m, pairs, False, **REGISTER)
    assert reg_mismatches(reg_numpy(reg), want_r) == [], what
    assert np.array_equal(reg.n_correspondences.cpu().numpy(), n_corr), what
    want_i = icp_np.icp(P[:n], L, pairs, reg.pose.cpu().numpy(), **ICP)
    assert icp_mismatches(icp_numpy(ref), want_i) == [], what
    return want_r, want_i


def assert_reaches_every_stage(case, want_r, want_i):
    """The batch is not vacuous: a pair registers and an ICP pair iterates (not for one-point clouds, whose count-1
    keypoint sets only match)."""
    if case.endswith("one_point"):
        return
    assert (want_r["hypothesis"] >= 0).any(), case
    assert (want_i["iterations"] >= 1).any(), case


@pytest.fixture(scope="module")
def model(cuda):
    from d3feat_b200 import synth
    from d3feat_b200.encoder import KPFCNN
    cfg = synth.Config(architecture=synth.ARCH_3DMATCH)
    return KPFCNN(cfg, synth.make_params(cfg, 0), LIMITS, device=cuda)


# ---- the eager exact path ---------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES)
def test_exact_path_chain_matches_oracles(cuda, model, case):
    """KPFCNN(...)(P, L, num_keypoints=64) under the trace, then match_keypoints, register_pairs and icp_pairs on its
    keypoints and level-0 clouds."""
    from d3feat_b200.matching import match_keypoints
    from d3feat_b200.registration import icp_pairs, register_pairs
    P, L = serving_batch(case)
    pairs = pairs_for(L)
    with record_ops() as tr:
        out = model(P, L, num_keypoints=K)
        torch.cuda.synchronize()
    kp = out["keypoints"]
    m = match_keypoints(kp, pairs)
    reg = register_pairs(kp, m, pairs, **REGISTER)
    ref = icp_pairs(out["inputs"]["points"][0], L, pairs, reg.pose, **ICP)
    torch.cuda.synchronize()
    n = len(P)
    assert tuple(out["descriptors"].shape) == (n, 32)
    want_r, want_i = check_chain(tr, P, L, n, out["descriptors"], out["scores"], kp, m, reg, ref, pairs,
                                 "exact " + case)
    assert_reaches_every_stage(case, want_r, want_i)
    if case.endswith("one_point"):
        assert (kp.count.cpu().numpy() == 1).all()
        assert (m.n_matches.cpu().numpy() == 1).all() and (want_i["iterations"] == 0).all()


# ---- the static form and the captured serving loop --------------------------------------------------------------------

def static_run(model, pipe, P, L):
    """The static form of one batch on its own PyramidBuffers with the bucket's capacities (level-0 rows past n0
    poisoned), run eagerly under the trace: encoder, decoder, keypoints, matching, RANSAC and ICP as the serving loop
    runs them."""
    from d3feat_b200 import pyramid as pyr
    from d3feat_b200.keypoints import select_keypoints
    from d3feat_b200.matching import match_keypoints
    from d3feat_b200.registration import icp_pairs, register_pairs
    dev = model.device
    buf = pyr.PyramidBuffers(model.config, model.limits, pipe.caps, pipe.n_clouds, dev, bbox=pipe.bbox)
    n = len(P)
    pts0 = np.zeros((buf.caps[0], 3), np.float32)
    pts0[:n] = P
    buf.points0.copy_(t(poisoned(pts0, n), dev))
    buf.lengths0.copy_(t(L, dev))
    buf.n0.fill_(n)
    inputs = model.build_inputs_static(buf)
    with record_ops() as tr:
        F = model.encode(inputs)
        desc, scores = model.describe(inputs, F, with_scores=True)
        rows = inputs["rows"][0]
        kp = select_keypoints(scores, inputs["lengths"][0], K, points=inputs["points"][0], descriptors=desc, rows=rows)
        m = match_keypoints(kp, pipe.match_pairs)
        reg = register_pairs(kp, m, pipe.match_pairs, **REGISTER)
        ref = icp_pairs(inputs["points"][0], inputs["lengths"][0], pipe.match_pairs, reg.pose, rows=rows,
                        bbox=pipe.bbox, **ICP)
        torch.cuda.synchronize()
    assert int(inputs["status"].item()) == 0
    assert all(r.get("rows_q") is not None for r in tr.records)      # every op ran capacity-sized
    return tr, inputs, (desc, scores, kp, m, reg, ref)


def fields(res, n):
    """Every output of a step, cut to the device count n where the buffer is capacity-sized."""
    desc, scores, kp, m, reg, ref = res
    out = {"descriptors": desc[:n], "scores": scores[:n]}
    for group, nt in (("keypoints", kp), ("matches", m), ("registration", reg), ("refinement", ref)):
        for f in nt._fields:
            out["%s.%s" % (group, f)] = getattr(nt, f)
    return {k: v.clone() for k, v in out.items() if v is not None}


def same_bits(a, b):
    if a.shape != b.shape:
        return False
    view = torch.int64 if a.dtype == torch.float64 else torch.int32
    return torch.equal(a.view(view), b.view(view)) if a.is_floating_point() else torch.equal(a, b)


EMPTY = "empty"
LOOP_CASES = ["B17", "B33", "B300", "B1024", "B1_one_point", "B1024_one_point"]


def loop_batches(case):
    """Variants 0-3, a batch with no points at all (index 4: its slot was captured on variant 0), variant 4; for B33
    then the three tail batches."""
    got = [serving_batch(case, v) for v in range(4)] + [EMPTY, serving_batch(case, 4)]
    if case == "B33":
        got += [serving_batch("B33_sum_N%+d" % e) for e in (-37, 0, 37)]
    return got


@pytest.mark.gpu
@pytest.mark.parametrize("case", LOOP_CASES)
def test_serving_loop_matches_static_path(cuda, model, case):
    """One bucket from GraphPipeline.for_batch (decoder, 64 keypoints, pairs, RANSAC, ICP) stepped through batches of
    one B with different empty and one-point patterns. Every non-empty batch's static form, run eagerly, is checked
    against the oracles, and the graph step returns it bit for bit. The step with no points returns level counts 0,
    keypoint counts 0 (index -1), no matches, hypothesis -1 with the identity pose, and ICP keeps that init; the batch
    after it, loaded into a slot that held a larger batch, is still exact."""
    from d3feat_b200.encoder import GraphPipeline, RefinedDetections
    from test_gpu_kernel_variants import SPLITK, launched
    batches = loop_batches(case)
    real = [b for b in batches if b is not EMPTY]
    B = len(real[0][1])
    assert all(len(L) == B for _, L in real)
    assert len({(P.tobytes(), tuple(L)) for P, L in real}) == len(real)
    pairs = pairs_for(real[0][1])
    P0, L0 = max(real, key=lambda b: len(b[0]))
    pipe = GraphPipeline.for_batch(model, t(P0, cuda), t(L0, cuda), slack=1.5, margin=0.1, decoder=True, keypoints=K,
                                   match_pairs=pairs, register=REGISTER, icp=ICP)
    eager = []
    for i, b in enumerate(batches):
        if b is EMPTY:
            eager.append(None)
            continue
        P, L = b
        if i == 0 and case == "B1_one_point":
            # every level holds one row while the capacity is two 128-row tiles: the deep GEMMs take the split-K plan
            (tr, inputs, res), names = launched(lambda: static_run(model, pipe, P, L))
            assert inputs["counts"][:5].cpu().tolist() == [1] * 5
            assert any(SPLITK in name for name in names), sorted(names)
        else:
            tr, inputs, res = static_run(model, pipe, P, L)
        counts = inputs["counts"][:5].cpu().tolist()
        assert counts[0] == len(P) and all(c <= cap for c, cap in zip(counts, pipe.caps))
        want_r, want_i = check_chain(tr, P, L, len(P), *res, pairs, "static %s batch %d" % (case, i), seed=i)
        assert_reaches_every_stage(case, want_r, want_i)
        eager.append((counts, fields(res, len(P))))
        del tr
    dev_batches = [(t(np.zeros((0, 3), np.float32), cuda), t(np.zeros(B, np.int32), cuda)) if b is EMPTY
                   else (t(b[0], cuda), t(b[1], cuda)) for b in batches]
    pipe.prime(*dev_batches[0])
    got = []
    for i in range(len(batches)):
        nxt = dev_batches[i + 1] if i + 1 < len(batches) else None
        res, cnt = pipe.step(*nxt) if nxt else pipe.step()
        assert isinstance(res, RefinedDetections)
        n = 0 if batches[i] is EMPTY else len(batches[i][0])
        got.append((cnt[:5].cpu().tolist(), fields(res, n)))
    pipe.check()
    for i, ((cnt, res), want) in enumerate(zip(got, eager)):
        if want is None:
            assert cnt == [0] * 5, cnt
            P_ = len(pairs)
            assert (res["keypoints.count"] == 0).all() and (res["keypoints.index"] == -1).all()
            assert (res["matches.n_matches"] == 0).all()
            assert (res["registration.hypothesis"] == -1).all()
            eye = torch.eye(4, dtype=torch.float64, device=cuda).expand(P_, 4, 4)
            assert same_bits(res["registration.pose"], eye.contiguous())
            assert same_bits(res["refinement.pose"], eye.contiguous())
            assert (res["refinement.iterations"] == 0).all() and (res["refinement.n_correspondences"] == 0).all()
            continue
        assert cnt == want[0], (i, cnt, want[0])
        for name, a in want[1].items():
            assert same_bits(res[name], a), (case, i, name)


def test_loop_batches_are_distinct_and_fit_one_bucket():
    """The loop's batches differ in their empty and one-point patterns, and the empty step sits in a slot captured on a
    non-empty batch (the ring holds 4 slots)."""
    for case in LOOP_CASES:
        batches = loop_batches(case)
        assert batches.index(EMPTY) == 4 and len(batches) >= 6, case
        real = [b for b in batches if b is not EMPTY]
        assert len({(P.tobytes(), tuple(L)) for P, L in real}) == len(real), case
        if not case.endswith("one_point"):
            assert len(batches[5][0]) < len(batches[1][0]), case      # rows of the earlier batch left past n0


# ---- CPU: the batches catch chained bugs ------------------------------------------------------------------------------

def synthetic(P, seed):
    """Scores [N] and unit descriptors [N, 32] for a batch's rows."""
    rng = np.random.default_rng(seed)
    d = rng.normal(size=(len(P), 32))
    return rng.normal(size=len(P)).astype(np.float32), (d / np.linalg.norm(d, axis=1, keepdims=True)).astype(np.float32)


def gathered(idx, rows):
    out = rows[np.maximum(idx, 0)]
    out[idx < 0] = 0
    return out


def keypoint_sets(P, L, seed):
    s, desc = synthetic(P, seed)
    idx, cnt = keypoint_oracle(s, L, K, n=len(P))
    return s, desc, idx, cnt


def test_serving_batches_reach_every_stage_without_a_gpu():
    """The pairs of every case touch empty, one-point and two-point clouds and a moved copy; the tail cases cut or
    extend the last cloud; the one-point cases hold level counts of one."""
    for case in CASES:
        P, L = serving_batch(case)
        pairs = np.asarray(pairs_for(L))
        sizes = np.asarray(L)[pairs]
        if case == "B1_one_point":
            assert len(P) == 1 and list(L) == [1]
            continue
        if case.endswith("one_point"):
            assert len(L) == 1024 and (L == 1).all()
            continue
        if case != "B1024_lone":
            for size in (0, 1, 2):
                assert (sizes == size).any() or not (L == size).any(), (case, size)
            assert (sizes == 0).any() and ((sizes == 1).any() or (sizes == 2).any()), case
            assert any(b % 4 == 3 and L[b] > 0 for _, b in pairs), case
    assert int(serving_batch("B33_sum_N-37")[1].sum()) == len(serving_batch("B33_sum_N-37")[0]) - 37
    assert int(serving_batch("B33_sum_N+37")[1].sum()) == len(serving_batch("B33_sum_N+37")[0]) + 37


def _unclipped_keypoints(s, L, n):
    """The per-cloud windows of the sorted order taken at the lengths' own offsets: the last cloud's window reaches
    past the row count (positions past it read as -1)."""
    order = keypoint_oracle(s, L, None, n)
    order = np.concatenate([order, np.full(int(np.sum(L)), -1, np.int32)])
    ends = np.concatenate([[0], np.cumsum(L)])[1:]
    idx = np.full((len(L), K), -1, np.int32)
    cnt = np.zeros(len(L), np.int32)
    for b in range(len(L)):
        c = min(K, int(L[b]))
        idx[b, :c] = order[ends[b] - c:ends[b]]
        cnt[b] = c
    return idx, cnt


def test_chain_bug_keypoints_over_unclipped_lengths_is_caught():
    P, L = serving_batch("B33_sum_N+37")
    s, _, idx, cnt = keypoint_sets(P, L, 1)
    bug = _unclipped_keypoints(s, L, len(P))
    assert not (np.array_equal(bug[0], idx) and np.array_equal(bug[1], cnt))


def test_chain_bug_rows_of_no_cloud_in_the_last_cloud_is_caught():
    P, L = serving_batch("B33_sum_N-37")
    s, _, idx, cnt = keypoint_sets(P, L, 2)
    Lb = L.copy()
    Lb[-1] += 37                                        # the 37 rows of no cloud joined to cloud B - 1
    bug = keypoint_oracle(s, Lb, K, n=len(P))
    assert not np.array_equal(bug[0], idx)


@pytest.mark.parametrize("case", ["B17", "B33", "B300", "B1024"])
def test_chain_bug_matching_reads_k_slots_is_caught(case):
    """match_np on the keypoint sets of the batch, with every count read as k: the padding of a short cloud (zero
    descriptors, similarity 0) enters the nearest-neighbour search."""
    P, L = serving_batch(case)
    pairs = pairs_for(L)
    _, desc, idx, cnt = keypoint_sets(P, L, 3)
    kd = gathered(idx, desc)
    want = match_np.match(kd, cnt, pairs)
    bug = match_np.match(kd, np.full_like(cnt, K), pairs)
    assert ((cnt > 0) & (cnt < K)).any()
    assert any(not np.array_equal(want[f], bug[f]) for f in ("nn_st", "matches", "n_matches"))


def _register(P, L, seed, count_of=None):
    """register_np on the batch's keypoint sets (synthetic scores and descriptors) and their one-way matches.
    count_of: the bug's view of the keypoint sets (points, count, corr, n_corr) instead of the real one."""
    from oracle import register_np
    pairs = np.asarray(pairs_for(L), np.int64)
    _, desc, idx, cnt = keypoint_sets(P, L, seed)
    pts, kd = gathered(idx, P), gathered(idx, desc)
    m = match_np.match(kd, cnt, pairs)
    nn = m["nn_st"]
    corr = np.stack([np.broadcast_to(np.arange(K, dtype=np.int32), nn.shape), nn], 2)
    n_corr = (nn >= 0).sum(1)
    if count_of is not None:
        pts, cnt, corr, n_corr = count_of(pts, cnt, corr, n_corr, pairs)
    return register_np.register(pts, cnt, corr, n_corr, pairs, **REGISTER)


def _sample_wraps_short_clouds(pts, cnt, corr, n_corr, pairs):
    """A source cloud with fewer than ransac_n keypoints sampled anyway: its slots wrap around (slot j reads slot
    j mod count), so the sample repeats its points under distinct indices."""
    n = REGISTER["ransac_n"]
    pts, cnt, corr, n_corr = pts.copy(), cnt.copy(), corr.copy(), n_corr.copy()
    for b in np.nonzero((cnt > 0) & (cnt < n))[0]:
        c = int(cnt[b])
        pts[b, :n] = pts[b, np.arange(n) % c]
        cnt[b] = n
    for p, (src, tgt) in enumerate(pairs):
        if 0 < n_corr[p] < n and cnt[src] == n:
            corr[p, :n] = corr[p, np.arange(n) % n_corr[p]]
            corr[p, :n, 0] = np.arange(n)
            n_corr[p] = n
    return pts, cnt, corr, n_corr


@pytest.mark.parametrize("case", ["B33", "B300"])
def test_chain_bug_ransac_sample_from_a_short_cloud_is_caught(case):
    """The batches with a one-point cloud: its pair with the largest cloud registers nothing, but a sample wrapped
    around its one keypoint (three copies of one correspondence) passes both checkers."""
    P, L = serving_batch(case)
    want = _register(P, L, 4)
    bug = _register(P, L, 4, _sample_wraps_short_clouds)
    pairs = np.asarray(pairs_for(L))
    short = (np.asarray(L)[pairs[:, 0]] > 0) & (np.asarray(L)[pairs[:, 0]] < REGISTER["ransac_n"])
    assert short.any()
    assert (want["hypothesis"][short] == -1).all()
    assert (bug["hypothesis"][short] >= 0).any()


def test_chain_bug_icp_targets_include_rows_of_no_cloud_is_caught():
    """icp_np with the 37 rows of no cloud joined to the last cloud as targets (its sources unchanged): pairs whose
    target is the last cloud find the moved near-copies."""
    P, L = serving_batch("B33_sum_N-37")
    pairs = [p for p in pairs_for(L) if p[1] == len(L) - 1 and L[p[0]] > 0]
    assert pairs
    init = np.tile(np.eye(4), (len(pairs), 1, 1))
    want = icp_np.icp(P, L, pairs, init, **ICP)
    start = np.concatenate([[0], np.cumsum(L)])
    lo = int(start[-2])
    src = [P[start[a]:start[a + 1]] for a, _ in pairs]
    tgt_bug = P[lo:]                                    # the last cloud and the 37 rows after it
    Pb = np.concatenate(src + [tgt_bug], 0)
    Lb = [len(c) for c in src] + [len(tgt_bug)]
    bug = icp_np.icp(Pb, Lb, [(i, len(src)) for i in range(len(src))], init, **ICP)
    assert icp_mismatches(bug, want) != []
