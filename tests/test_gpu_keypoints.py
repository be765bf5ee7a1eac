"""Keypoint selection on the GPU (d3f_select_keypoints, keypoints.select_keypoints, KPFCNN(num_keypoints=...),
GraphPipeline(keypoints=...)) against numpy.

Oracle for cloud b: np.argsort(s_b, kind="stable")[-k:] + start_b (utils/tester.py:209-213, 281-290 select with an
argsort of the scores). Every comparison is exact: indices, counts and the gathered rows bit for bit."""
import ctypes as C

import numpy as np
import pytest

KMAX_BATCH = 1024
NAN_BITS = np.array([0x7fc00000, 0xffc00000, 0x7f800001, 0xffffffff], np.uint32)   # +qNaN, -qNaN, sNaN, -NaN payload


def make_scores(rng, n, quantum=0.125):
    """Quantised scores (many exact ties) with +-0.0, +-inf and NaNs of both signs mixed in."""
    s = (np.round(rng.normal(size=n) / quantum) * quantum).astype(np.float32).view(np.uint32).copy()
    m = rng.random(n)
    pick = rng.integers(0, 4, n)
    special = np.array([0x00000000, 0x80000000, 0x7f800000, 0xff800000], np.uint32)
    s[m < 0.05] = special[pick[m < 0.05]]
    sel = (m >= 0.05) & (m < 0.08)
    s[sel] = NAN_BITS[pick[sel]]
    return s.view(np.float32)


def oracle(s, lens, k=None, n=None):
    """(index [B,k], count [B]) or, k=None, the full order; clouds cut at n. Rows past the last cloud come last."""
    n = s.shape[0] if n is None else n
    start = np.minimum(np.concatenate([[0], np.cumsum(lens)]), n).astype(np.int64)
    parts = [np.argsort(s[start[b]:start[b + 1]], kind="stable") + start[b] for b in range(len(lens))]
    if k is None:
        parts.append(np.argsort(s[start[-1]:n], kind="stable") + start[-1])
        return np.concatenate(parts).astype(np.int32)
    idx = np.full((len(lens), k), -1, np.int32)
    cnt = np.zeros(len(lens), np.int32)
    for b, p in enumerate(parts):
        top = p[-k:]
        idx[b, :len(top)] = top
        cnt[b] = len(top)
    return idx, cnt


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def check_gathered(kp, index, points, desc, scores):
    """Gathered rows == fancy-indexed inputs, bit for bit; zero rows in the padding."""
    real = index >= 0
    safe = np.where(real, index, 0)
    for got, src in ((kp.points, points), (kp.descriptors, desc), (kp.scores, scores)):
        if src is None:
            assert got is None
            continue
        want = src[safe]
        want[~real] = 0
        assert np.array_equal(bits(got.cpu().numpy()), bits(want))


def t(a, dev):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


# ---- 1. op against the oracle -----------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("k", [1, 250, 5000])
def test_select_keypoints_matches_stable_argsort(cuda, k):
    from d3feat_b200.keypoints import select_keypoints
    rng = np.random.default_rng(k)
    lens = np.array([0, 1, k - 1, k, k + 1, 30000, 0, 60000, 7, k + 1, 1, 2], np.int32)
    N = int(lens.sum())
    s = make_scores(rng, N)
    P = rng.normal(size=(N, 3)).astype(np.float32)
    Dsc = rng.normal(size=(N, 32)).astype(np.float32)
    kp = select_keypoints(t(s, cuda), t(lens, cuda), k, points=t(P, cuda), descriptors=t(Dsc, cuda))
    idx, cnt = oracle(s, lens, k)
    got = kp.index.cpu().numpy()
    assert np.array_equal(kp.count.cpu().numpy(), cnt)
    assert np.array_equal(got, idx)
    assert (got[np.arange(k)[None, :] >= cnt[:, None]] == -1).all()
    check_gathered(kp, got, P, Dsc, s)
    order = select_keypoints(t(s[:, None], cuda), t(lens, cuda)).cpu().numpy()
    assert np.array_equal(order, oracle(s, lens))


@pytest.mark.gpu
def test_select_keypoints_order_of_special_values(cuda):
    """The order the contract names: NaNs of either sign above +inf, -0.0 tied with +0.0 (row order decides)."""
    from d3feat_b200.keypoints import select_keypoints
    s = np.array([np.nan, 1, 0, -0.0, -np.nan, np.inf, -np.inf, 0], np.float32)
    s[4] = NAN_BITS[1:2].view(np.float32)[0]
    want = np.array([6, 2, 3, 7, 1, 5, 0, 4], np.int32)
    assert np.array_equal(np.argsort(s, kind="stable"), want)
    got = select_keypoints(t(s, cuda), t(np.array([8], np.int32), cuda)).cpu().numpy()
    assert np.array_equal(got, want)


@pytest.mark.gpu
def test_select_keypoints_odd_descriptor_width_and_no_optional_inputs(cuda):
    from d3feat_b200.keypoints import select_keypoints
    rng = np.random.default_rng(3)
    lens = np.array([5, 0, 40, 3], np.int32)
    N = int(lens.sum())
    s = make_scores(rng, N)
    Dsc = rng.normal(size=(N, 37)).astype(np.float32)
    kp = select_keypoints(t(s, cuda), t(lens, cuda), 6, descriptors=t(Dsc, cuda))
    idx, cnt = oracle(s, lens, 6)
    assert np.array_equal(kp.index.cpu().numpy(), idx) and np.array_equal(kp.count.cpu().numpy(), cnt)
    check_gathered(kp, idx, None, Dsc, s)
    kp = select_keypoints(t(s, cuda), t(lens, cuda), 6)
    assert kp.points is None and kp.descriptors is None
    assert np.array_equal(kp.index.cpu().numpy(), idx)


# ---- 2. many clouds: the cloud id takes more than 8 key bits ----------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("B", [300, KMAX_BATCH])
def test_select_keypoints_many_clouds(cuda, B):
    from d3feat_b200.keypoints import select_keypoints
    rng = np.random.default_rng(B)
    lens = rng.integers(0, 60, B).astype(np.int32)
    N = int(lens.sum())
    s = make_scores(rng, N, quantum=0.5)
    P = rng.normal(size=(N, 3)).astype(np.float32)
    kp = select_keypoints(t(s, cuda), t(lens, cuda), 9, points=t(P, cuda))
    idx, cnt = oracle(s, lens, 9)
    assert np.array_equal(kp.index.cpu().numpy(), idx) and np.array_equal(kp.count.cpu().numpy(), cnt)
    check_gathered(kp, idx, P, None, s)
    assert np.array_equal(select_keypoints(t(s, cuda), t(lens, cuda)).cpu().numpy(), oracle(s, lens))


# ---- 3. device row counts: capacity-sized inputs, poisoned tails, sentinel-filled outputs -----------------------

def _call_raw(s, lens, k, P, Dsc, n, cap, dev):
    """d3f_select_keypoints on capacity-sized buffers with n in device memory; every output pre-filled with a
    sentinel. Returns the numpy outputs."""
    import torch
    from d3feat_b200 import _lib
    lib = _lib.lib()
    B, D = len(lens), Dsc.shape[1]
    order = torch.full((cap,), -7, dtype=torch.int32, device=dev)
    index = torch.full((B, k), -7, dtype=torch.int32, device=dev)
    count = torch.full((B,), -7, dtype=torch.int32, device=dev)
    op = torch.full((B, k, 3), 7.5, device=dev)
    od = torch.full((B, k, D), 7.5, device=dev)
    osc = torch.full((B, k), 7.5, device=dev)
    n_dev = torch.tensor([n], dtype=torch.int32, device=dev)
    ws = _lib.workspace(lib.d3f_select_keypoints_workspace_bytes(cap, B), dev)
    ts, tl, tp, td = t(s, dev), t(lens, dev), t(P, dev), t(Dsc, dev)
    _lib.check(lib.d3f_select_keypoints(_lib.ptr(ts), _lib.ptr(tl), B, cap, k, _lib.ptr(tp), _lib.ptr(td), D,
                                        _lib.ptr(order), _lib.ptr(index), _lib.ptr(count), _lib.ptr(op), _lib.ptr(od),
                                        _lib.ptr(osc), _lib.ptr(ws), ws.numel(), _lib.stream(), _lib.ptr(n_dev)),
               "d3f_select_keypoints")
    from d3feat_b200.keypoints import KeypointSet
    return order.cpu().numpy(), KeypointSet(index.cpu().numpy(), count.cpu().numpy(), op, od, osc)


@pytest.mark.gpu
@pytest.mark.parametrize("excess", [0, 700, -900])
def test_select_keypoints_device_row_count(cuda, excess):
    """excess = sum(lengths) - n: 0 (consistent), > 0 (the last clouds are cut at n), < 0 (rows past the last cloud
    belong to none and come last in the order). No row >= n is selected, read or written."""
    rng = np.random.default_rng(abs(excess) + 1)
    k = 250
    lens = np.array([3000, 0, 120, 4000, 2500], np.int32)
    n = int(lens.sum()) - excess
    cap = n + 1500
    s = make_scores(rng, cap)
    tail = np.arange(n, cap)
    s[tail] = np.where(tail % 2 == 0, np.float32(np.inf), NAN_BITS[0:1].view(np.float32)[0])
    P = rng.normal(size=(cap, 3)).astype(np.float32)
    Dsc = rng.normal(size=(cap, 32)).astype(np.float32)
    P[n:] = np.nan
    Dsc[n:] = np.nan
    order, kp = _call_raw(s, lens, k, P, Dsc, n, cap, cuda)
    idx, cnt = oracle(s, lens, k, n=n)
    assert np.array_equal(kp.index, idx) and np.array_equal(kp.count, cnt)
    assert kp.index.max() < n
    check_gathered(kp, kp.index, P, Dsc, s)
    assert np.array_equal(order[:n], oracle(s, lens, n=n))
    assert (order[n:] == -7).all()


# ---- 4. the tester's own call on tie-free scores ----------------------------------------------------------------

@pytest.mark.gpu
def test_select_keypoints_equals_io_utils_on_tie_free_scores(cuda):
    from d3feat_b200 import io_utils
    from d3feat_b200.keypoints import select_keypoints
    rng = np.random.default_rng(11)
    lens = np.array([5000, 250, 12000, 100], np.int32)
    N = int(lens.sum())
    s = ((rng.permutation(N) - N // 2) / 64.0).astype(np.float32)     # distinct, exactly representable
    assert np.unique(s).size == s.size
    k = 250
    kp = select_keypoints(t(s, cuda), t(lens, cuda), k)
    order = select_keypoints(t(s, cuda), t(lens, cuda)).cpu().numpy()
    index = kp.index.cpu().numpy()
    start = np.concatenate([[0], np.cumsum(lens)])
    for b in range(len(lens)):
        sb = s[start[b]:start[b + 1], None]
        top = io_utils.select_keypoints(sb, k) + start[b]
        assert np.array_equal(index[b, :len(top)], top)
        assert np.array_equal(order[start[b]:start[b + 1]], io_utils.select_keypoints(sb) + start[b])


# ---- 5. KPFCNN(num_keypoints=...) -------------------------------------------------------------------------------

LIMITS = [35, 33, 34, 36, 30]


@pytest.mark.gpu
def test_kpfcnn_num_keypoints(cuda):
    from d3feat_b200 import synth
    from d3feat_b200.encoder import KPFCNN
    cfg = synth.Config(architecture=synth.ARCH_3DMATCH)
    enc = KPFCNN(cfg, synth.make_params(cfg, 7), LIMITS, device=cuda)
    clouds = [synth.room_fragment(40 + i, n) for i, n in enumerate([9000, 7000, 8000])]
    P = np.concatenate(clouds, 0)
    L = np.array([c.shape[0] for c in clouds], np.int32)
    out = enc(P, L, num_keypoints=250)
    assert set(out) == {"inputs", "F", "descriptors", "scores", "keypoints"}
    kp = out["keypoints"]
    s = out["scores"].cpu().numpy().reshape(-1)
    idx, cnt = oracle(s, L, 250)
    assert np.array_equal(kp.index.cpu().numpy(), idx) and np.array_equal(kp.count.cpu().numpy(), cnt)
    check_gathered(kp, idx, out["inputs"]["points"][0].cpu().numpy(), out["descriptors"].cpu().numpy(), s)
    with pytest.raises(ValueError):
        enc(P, L, decoder=False, num_keypoints=250)


# ---- 6. GraphPipeline(decoder=True, keypoints=...) ---------------------------------------------------------------

def rel_err(a, b):
    a = np.asarray(a, np.float64)
    b = np.asarray(b, np.float64)
    return np.abs(a - b).max() / max(np.abs(b).max(), 1e-30)


@pytest.mark.gpu
def test_graph_pipeline_keypoints(cuda):
    """Five batches of different sizes through one captured bucket with the decoder, the detection scores and the
    keypoint selection inside the encoder graph. The dense descriptors and scores match the eager path (2e-5, as the
    encoder-only graph test); the keypoints are exactly the oracle applied to the graph's OWN scores."""
    import torch
    from d3feat_b200 import synth
    from d3feat_b200.encoder import KPFCNN, GraphPipeline, Detections
    cfg = synth.Config(architecture=synth.ARCH_3DMATCH)
    enc = KPFCNN(cfg, synth.make_params(cfg, 5), LIMITS, device=cuda)
    batches = []
    for i, n in enumerate([12000, 11000, 12000, 9500, 11800]):
        clouds = [synth.room_fragment(120 + 2 * i, n), synth.room_fragment(121 + 2 * i, n - 700)]
        batches.append((np.concatenate(clouds, 0), np.array([c.shape[0] for c in clouds], np.int32)))
    want = []
    for P, L in batches:
        o = enc(P, L)
        want.append((o["descriptors"].cpu().numpy(), o["scores"].cpu().numpy()))
    pipe = GraphPipeline.for_batch(enc, t(batches[0][0], cuda), t(batches[0][1], cuda), slack=1.2, decoder=True,
                                   keypoints=250)
    pipe.prime(t(batches[0][0], cuda), t(batches[0][1], cuda))
    got = []
    for i in range(len(batches)):
        nxt = batches[i + 1] if i + 1 < len(batches) else None
        res, counts = pipe.step(t(nxt[0], cuda), t(nxt[1], cuda)) if nxt else pipe.step()
        assert isinstance(res, Detections)
        kp = res.keypoints
        got.append((res.descriptors.clone(), res.scores.clone(), [x.clone() for x in kp], counts.clone()))
    pipe.check()
    for i, ((desc, scores, kp, counts), (wd, ws), (P, L)) in enumerate(zip(got, want, batches)):
        n = int(counts[0].item())
        assert n == P.shape[0] == wd.shape[0], i
        desc, scores = desc[:n].cpu().numpy(), scores[:n].cpu().numpy()
        assert rel_err(desc, wd) < 2e-5, i
        assert rel_err(scores, ws) < 2e-5, i
        index, count, kpts, kdesc, kscores = [x.cpu().numpy() for x in kp]
        idx, cnt = oracle(scores.reshape(-1), L, 250)
        assert np.array_equal(index, idx) and np.array_equal(count, cnt), i
        real = index >= 0
        assert real.all()
        assert np.array_equal(bits(kdesc), bits(desc[index])), i
        assert np.array_equal(bits(kscores), bits(scores.reshape(-1)[index])), i
        assert np.array_equal(bits(kpts), bits(P[index])), i
    torch.cuda.synchronize()


# ---- 7. CPU: argument validation before any CUDA call ------------------------------------------------------------

def test_select_keypoints_invalid_arguments_without_a_gpu():
    from d3feat_b200 import build
    lib = C.CDLL(build.build())
    lib.d3f_last_error.restype = C.c_char_p
    lib.d3f_select_keypoints_workspace_bytes.restype = C.c_size_t
    lib.d3f_select_keypoints_workspace_bytes.argtypes = [C.c_int, C.c_int]
    from d3feat_b200._lib import SYMBOLS
    fn = lib.d3f_select_keypoints
    fn.restype, fn.argtypes = [(r, a) for name, r, a in SYMBOLS if name == "d3f_select_keypoints"][0]
    fake = C.c_void_p(256)          # never dereferenced: validation fails first
    ws_ok = lib.d3f_select_keypoints_workspace_bytes(1000, 4)
    assert ws_ok > 0

    def call(B=4, N=1000, k=250, desc=None, D=0, order=None, index=fake, ws=ws_ok, pts=None, out_p=None):
        return fn(fake, fake, B, N, k, pts, desc, D, order, index, None, out_p, None, None, fake, ws, None, None)

    cases = [(dict(B=0), b"B=0"), (dict(B=KMAX_BATCH + 1), b"B=1025"), (dict(k=0), b"k=0"),
             (dict(desc=fake, D=0), b"D=0"), (dict(N=-1), b"bad shape"), (dict(index=None), b"no output"),
             (dict(out_p=fake), b"without points")]
    for kw, msg in cases:
        assert call(**kw) == -1, kw
        assert msg in lib.d3f_last_error(), (kw, lib.d3f_last_error())
    assert call(ws=ws_ok - 1) == -4
    assert b"workspace" in lib.d3f_last_error()
    assert call(k=0, index=None, order=fake, ws=0) == -4     # the full order needs no k


def test_graph_pipeline_keypoints_argument_checked_first():
    """keypoints without the decoder (or k < 1) is refused before the pipeline touches the encoder or the device."""
    from d3feat_b200.encoder import GraphPipeline
    with pytest.raises(ValueError, match="decoder=True"):
        GraphPipeline(None, [1024] * 5, 2, np.zeros(6, np.float32), keypoints=250)
    with pytest.raises(ValueError, match=">= 1"):
        GraphPipeline(None, [1024] * 5, 2, np.zeros(6, np.float32), decoder=True, keypoints=0)
