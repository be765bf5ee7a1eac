"""Descriptor matching on the GPU (d3f_match_descriptors, matching.match_keypoints,
GraphPipeline(..., match_pairs=...)) against the numpy restatement oracle/match_np.py.

Every comparison is exact: nearest-neighbour indices, the mutual match list, the counts and the bits of every
similarity. The similarity is a sequential-channel fp32 sum with no FMA, so the sim comparison also fails if the
kernel's multiply and add were contracted."""
import ctypes as C

import numpy as np
import pytest

from oracle import match_np

KMAX_BATCH = 1024
FIELDS = ("nn_st", "sim_st", "nn_ts", "sim_ts", "matches", "n_matches")


def t(a, dev):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def as_numpy(m):
    return {f: getattr(m, f).cpu().numpy() for f in FIELDS}


def mismatches(got, want):
    """Fields of `got` that differ from `want`: integers exactly, similarities bit for bit."""
    bad = []
    for f in FIELDS:
        g, w = np.asarray(got[f]), np.asarray(want[f])
        if g.dtype == np.float32:
            g, w = g.view(np.uint32), w.view(np.uint32)
        if g.shape != w.shape or not np.array_equal(g, w):
            bad.append(f)
    return bad


def check(m, desc, count, pairs):
    want = match_np.match(desc, count, pairs)
    assert mismatches(as_numpy(m), want) == []
    return want


def all_ordered_pairs(B, extra=()):
    """every ordered pair (self pairs included), then `extra`"""
    p = [(i, j) for i in range(B) for j in range(B)] + list(extra)
    return np.array(p, np.int32)


def match_dev(desc, count, pairs, dev):
    from d3feat_b200.matching import match_keypoints
    return match_keypoints(t(desc, dev), t(pairs, dev), count=t(count, dev))


def unit_rows(rng, shape):
    d = rng.normal(size=shape).astype(np.float32)
    return (d / np.linalg.norm(d, axis=-1, keepdims=True)).astype(np.float32)


# ---- 1. counts {0, 1, k-1, k, ...}, every ordered pair, repeats and out-of-range ids -----------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("k", [1, 250, 5000])
def test_match_descriptors_against_oracle(cuda, k):
    rng = np.random.default_rng(k)
    B, D = 8, 32
    if k == 5000:       # keep the numpy oracle's k x k similarities few: three large clouds
        count = np.array([0, 1, k - 1, k, 40, 2, 130, k], np.int32)
    else:
        count = np.array([0, 1, max(k - 1, 0), k, k // 2, k, min(3, k), k], np.int32)
    desc = unit_rows(rng, (B, k, D))
    pairs = all_ordered_pairs(B, extra=[(3, 5), (3, 5), (2, 2), (-1, 3), (3, -1), (B, 0), (0, B), (-1, B)])
    want = check(match_dev(desc, count, pairs, cuda), desc, count, pairs)
    assert want["n_matches"][pairs.tolist().index([3, 5])] > 0
    assert (want["n_matches"][-5:] == 0).all()


# ---- 2. descriptor widths around the 32-channel chunk -------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("D", [1, 31, 33, 64])
def test_match_descriptors_widths(cuda, D):
    rng = np.random.default_rng(100 + D)
    k = 150
    count = np.array([150, 97, 64, 1], np.int32)
    desc = rng.normal(size=(4, k, D)).astype(np.float32)
    pairs = all_ordered_pairs(4)
    check(match_dev(desc, count, pairs, cuda), desc, count, pairs)


# ---- 3. exact ties, +-0, +-inf and NaN entries ---------------------------------------------------------------------

def quantised(rng, shape, special_rate=0.003):
    """multiples of 1/8 (many exactly tied similarities) with +-0.0, +-inf and NaNs of both signs mixed in"""
    d = (np.round(rng.normal(size=shape) * 2) / 8).astype(np.float32).view(np.uint32).copy()
    m = rng.random(shape)
    special = np.array([0x00000000, 0x80000000, 0x7f800000, 0xff800000, 0x7fc00000, 0xffc00000], np.uint32)
    sel = m < special_rate
    d[sel] = special[rng.integers(0, len(special), int(sel.sum()))]
    return d.view(np.float32)


@pytest.mark.gpu
@pytest.mark.parametrize("D", [4, 32])
def test_match_descriptors_ties_and_special_values(cuda, D):
    rng = np.random.default_rng(7 + D)
    k = 300
    count = np.array([300, 300, 211, 65], np.int32)
    # clouds 0 and 1 are finite (one NaN column would make every row's nearest neighbour a NaN), 2 and 3 are not
    desc = np.concatenate([quantised(rng, (2, k, D), special_rate=0), quantised(rng, (2, k, D), special_rate=0.01)])
    pairs = all_ordered_pairs(4)
    want = check(match_dev(desc, count, pairs, cuda), desc, count, pairs)
    s = match_np.similarity(desc[0], desc[1])
    best = s.max(axis=1, keepdims=True)
    assert ((s == best).sum(axis=1) > 1).mean() > 0.05, "the case should hold tied nearest neighbours"
    assert np.isnan(want["sim_st"]).any() and np.isnan(want["sim_ts"]).any()
    assert np.isinf(desc[2:]).any() and np.isnan(desc[2:]).any()


# ---- 4. padding poisoned with NaN; device counts above k and below 0 ---------------------------------------------

@pytest.mark.gpu
def test_match_descriptors_padding_and_count_clamp(cuda):
    import torch
    rng = np.random.default_rng(4)
    k, D = 200, 32
    count = np.array([k + 5, -3, 120, k, 0, 17], np.int32)
    desc = unit_rows(rng, (6, k, D))
    for b, c in enumerate(np.clip(count, 0, k)):
        desc[b, c:] = np.nan
    pairs = all_ordered_pairs(6)
    want = check(match_dev(desc, count, pairs, cuda), desc, count, pairs)
    assert not np.isnan(want["sim_st"]).any()
    # the raw entry point on sentinel-filled outputs: every element is written
    from d3feat_b200 import _lib
    lib = _lib.lib()
    P = len(pairs)
    out = [torch.full(s, 7, dtype=dt, device=cuda) for s, dt in (
        ((P, k), torch.int32), ((P, k), torch.float32), ((P, k), torch.int32), ((P, k), torch.float32),
        ((P, k, 2), torch.int32), ((P,), torch.int32))]
    ws = _lib.workspace(lib.d3f_match_descriptors_workspace_bytes(k, P), cuda)
    td, tc, tp = t(desc, cuda), t(count, cuda), t(pairs, cuda)
    _lib.check(lib.d3f_match_descriptors(_lib.ptr(td), _lib.ptr(tc), 6, k, D, _lib.ptr(tp), P,
                                         *[_lib.ptr(o) for o in out], _lib.ptr(ws), ws.numel(), _lib.stream()),
               "d3f_match_descriptors")
    assert mismatches({f: o.cpu().numpy() for f, o in zip(FIELDS, out)}, want) == []


# ---- 5. many clouds and pairs ---------------------------------------------------------------------------------------

@pytest.mark.gpu
def test_match_descriptors_many_clouds_and_pairs(cuda):
    rng = np.random.default_rng(5)
    B, k, D, P = KMAX_BATCH, 24, 32, 4096
    count = rng.integers(-2, k + 3, B).astype(np.int32)
    desc = rng.normal(size=(B, k, D)).astype(np.float32)
    pairs = rng.integers(0, B, (P, 2)).astype(np.int32)
    pairs[::97, 0] = -1
    pairs[::89, 1] = B
    check(match_dev(desc, count, pairs, cuda), desc, count, pairs)


# ---- 6. captured in a CUDA graph, inputs rewritten in place ------------------------------------------------------

@pytest.mark.gpu
def test_match_descriptors_in_a_cuda_graph(cuda):
    import torch
    from d3feat_b200.matching import match_keypoints
    rng = np.random.default_rng(6)
    B, k, D = 5, 250, 32
    pairs = all_ordered_pairs(B, extra=[(-1, 0)])
    desc = t(unit_rows(rng, (B, k, D)), cuda)
    count = t(np.array([250, 3, 0, 200, 249], np.int32), cuda)
    pr = t(pairs, cuda)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        match_keypoints(desc, pr, count=count)          # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        m = match_keypoints(desc, pr, count=count)
    for r in range(3):
        d_new = quantised(rng, (B, k, D)) if r == 1 else unit_rows(rng, (B, k, D))
        c_new = rng.integers(-1, k + 2, B).astype(np.int32)
        desc.copy_(t(d_new, cuda))
        count.copy_(t(c_new, cuda))
        g.replay()
        torch.cuda.synchronize()
        assert mismatches(as_numpy(m), match_np.match(d_new, c_new, pairs)) == [], r


# ---- 7. GraphPipeline(decoder=True, keypoints=250, match_pairs=every i < j) ---------------------------------------

LIMITS = [35, 33, 34, 36, 30]


@pytest.mark.gpu
def test_graph_pipeline_match_pairs(cuda):
    """Five batches of three clouds through one captured bucket. The matches are the oracle applied to the graph's own
    keypoint descriptors, and equal an eager match_keypoints of the same KeypointSet."""
    import torch
    from d3feat_b200 import synth
    from d3feat_b200.encoder import KPFCNN, GraphPipeline, MatchedDetections
    from d3feat_b200.keypoints import KeypointSet
    from d3feat_b200.matching import match_keypoints
    cfg = synth.Config(architecture=synth.ARCH_3DMATCH)
    enc = KPFCNN(cfg, synth.make_params(cfg, 5), LIMITS, device=cuda)
    batches = []
    for i, n in enumerate([9000, 8500, 9000, 7000, 8800]):
        clouds = [synth.room_fragment(300 + 3 * i + c, n - 400 * c) for c in range(3)]
        batches.append((np.concatenate(clouds, 0), np.array([c.shape[0] for c in clouds], np.int32)))
    pairs = [(i, j) for i in range(3) for j in range(i + 1, 3)]
    pipe = GraphPipeline.for_batch(enc, t(batches[0][0], cuda), t(batches[0][1], cuda), slack=1.2, decoder=True,
                                   keypoints=250, match_pairs=pairs)
    pipe.prime(t(batches[0][0], cuda), t(batches[0][1], cuda))
    got = []
    for i in range(len(batches)):
        nxt = batches[i + 1] if i + 1 < len(batches) else None
        res, _ = pipe.step(t(nxt[0], cuda), t(nxt[1], cuda)) if nxt else pipe.step()
        assert isinstance(res, MatchedDetections)
        got.append((KeypointSet(*[x.clone() for x in res.keypoints]), [x.clone() for x in res.matches]))
    pipe.check()
    for i, (kp, m) in enumerate(got):
        gm = {f: x.cpu().numpy() for f, x in zip(FIELDS, m)}
        want = match_np.match(kp.descriptors.cpu().numpy(), kp.count.cpu().numpy(), pairs)
        assert mismatches(gm, want) == [], i
        assert (want["n_matches"] > 0).all(), i
        assert mismatches(as_numpy(match_keypoints(kp, pairs)), gm) == [], i
    torch.cuda.synchronize()


# ---- CPU: argument validation, pipeline arguments, the oracle itself -------------------------------------------

def test_match_descriptors_invalid_arguments_without_a_gpu():
    from d3feat_b200 import build
    from d3feat_b200._lib import SYMBOLS
    lib = C.CDLL(build.build())
    lib.d3f_last_error.restype = C.c_char_p
    for name in ("d3f_match_descriptors_workspace_bytes", "d3f_match_descriptors"):
        fn = getattr(lib, name)
        fn.restype, fn.argtypes = [(r, a) for n, r, a in SYMBOLS if n == name][0]
    fake = C.c_void_p(256)          # never dereferenced: validation fails first
    ws_ok = lib.d3f_match_descriptors_workspace_bytes(250, 6)
    assert ws_ok >= 2 * 8 * 250 * 6
    assert lib.d3f_match_descriptors_workspace_bytes(0, 6) == 0
    assert lib.d3f_match_descriptors_workspace_bytes(65536, 65536) == 0

    def call(B=4, k=250, D=32, P=6, ws=ws_ok, null=None):
        ptrs = [None if i == null else fake for i in range(10)]
        return lib.d3f_match_descriptors(ptrs[0], ptrs[1], B, k, D, ptrs[2], P, *ptrs[3:9], ptrs[9], ws, None)

    cases = [(dict(B=0), b"B=0"), (dict(B=KMAX_BATCH + 1), b"B=1025"), (dict(k=0), b"k=0"), (dict(D=0), b"D=0"),
             (dict(P=0), b"P=0"), (dict(k=65536, P=65536), b"exceeds int32")]
    cases += [(dict(null=i), b"null pointer") for i in range(10)]
    for kw, msg in cases:
        assert call(**kw) == -1, kw
        assert msg in lib.d3f_last_error(), (kw, lib.d3f_last_error())
    assert call(ws=ws_ok - 1) == -4
    assert b"workspace" in lib.d3f_last_error()


def test_host_pairs_are_range_checked():
    from d3feat_b200.matching import host_pairs
    assert host_pairs([(0, 1), (1, 0)], 2).dtype == np.int32
    for bad in ([(0, 2)], [(-1, 0)], [], [(0, 1, 2)], [0, 1], [(0.0, 1.0)]):
        with pytest.raises(ValueError):
            host_pairs(bad, 2)


def test_graph_pipeline_match_pairs_checked_first():
    """match_pairs without keypoints, or naming a cloud outside [0, n_clouds), is refused before the pipeline touches
    the encoder or the device."""
    from d3feat_b200.encoder import GraphPipeline
    bbox = np.zeros(6, np.float32)
    with pytest.raises(ValueError, match="needs keypoints"):
        GraphPipeline(None, [1024] * 5, 2, bbox, decoder=True, match_pairs=[(0, 1)])
    for bad in ([(0, 2)], [(-1, 1)], []):
        with pytest.raises(ValueError, match="GraphPipeline"):
            GraphPipeline(None, [1024] * 5, 2, bbox, decoder=True, keypoints=250, match_pairs=bad)


def test_oracle_agrees_with_sqrt_argmin_on_unit_descriptors():
    """On unit descriptors the exact argmax of s is build_correspondence's argmin of sqrt(2 - 2s) wherever the float64
    best and second-best similarities of a row (a column) differ by more than 1e-5."""
    rng = np.random.default_rng(12)
    checked = 0
    for n, m in ((250, 250), (250, 180), (60, 250)):
        a, b = unit_rows(rng, (n, 32)), unit_rows(rng, (m, 32))
        s64 = a.astype(np.float64) @ b.astype(np.float64).T
        top_r, top_c = np.sort(s64, axis=1), np.sort(s64, axis=0)
        clear_r = top_r[:, -1] - top_r[:, -2] > 1e-5
        clear_c = top_c[-1, :] - top_c[-2, :] > 1e-5
        want = match_np.match(np.stack([np.pad(a, ((0, 250 - n), (0, 0))), np.pad(b, ((0, 250 - m), (0, 0)))]),
                              [n, m], [(0, 1)])
        nn_st, nn_ts, pairs = match_np.reference_correspondence(a, b)
        assert np.array_equal(want["nn_st"][0, :n][clear_r], nn_st[clear_r])
        assert np.array_equal(want["nn_ts"][0, :m][clear_c], nn_ts[clear_c])
        if clear_r.all() and clear_c.all():
            assert np.array_equal(want["matches"][0, :want["n_matches"][0]], pairs)
            checked += 1
        assert clear_r.mean() > 0.9 and clear_c.mean() > 0.9
    assert checked >= 1


def _fma_similarity(a, b):
    s = np.zeros((a.shape[0], b.shape[0]), np.float32)
    for c in range(a.shape[1]):
        s = (np.multiply.outer(a[:, c].astype(np.float64), b[:, c].astype(np.float64)) + s).astype(np.float32)
    return s


def _nearest_ties_to_largest(s):
    n, m = s.shape
    nn_st = (m - 1 - np.argmax(s[:, ::-1], axis=1)).astype(np.int32)
    nn_ts = (n - 1 - np.argmax(s[::-1, :], axis=0)).astype(np.int32)
    return nn_st, s[np.arange(n), nn_st], nn_ts, s[nn_ts, np.arange(m)]


def _mutual_by_target(nn_st, nn_ts):
    j = np.arange(len(nn_ts))
    keep = nn_st[nn_ts] == j
    return np.stack([nn_ts[keep], j[keep]], 1).astype(np.int32).reshape(-1, 2)


@pytest.mark.parametrize("bug", ["fma", "ties_to_largest", "count_ignored", "mutual_by_target"])
def test_oracle_rejects_emulated_bugs(monkeypatch, bug):
    rng = np.random.default_rng(13)
    k = 120
    desc = quantised(rng, (3, k, 32), special_rate=0) if bug == "ties_to_largest" else unit_rows(rng, (3, k, 32))
    count = np.array([k, 90, 61], np.int32)
    pairs = all_ordered_pairs(3)
    want = match_np.match(desc, count, pairs)
    assert mismatches(want, match_np.match(desc, count, pairs)) == []
    if bug == "count_ignored":
        got = match_np.match(desc, np.full(3, k, np.int32), pairs)
    else:
        name, fn = {"fma": ("similarity", _fma_similarity), "ties_to_largest": ("nearest", _nearest_ties_to_largest),
                    "mutual_by_target": ("mutual", _mutual_by_target)}[bug]
        monkeypatch.setattr(match_np, name, fn)
        got = match_np.match(desc, count, pairs)
    bad = mismatches(got, want)
    assert bad, bug
    if bug == "fma":
        assert "sim_st" in bad and "sim_ts" in bad
