"""Keypoint detection on the GPU: per-cloud selection by detection score (d3f_select_keypoints), and the uniform
random keypoints it is compared against (d3f_sample_keypoints).

The reference selects keypoints on the host after every batch: the 3DMatch tester dumps each fragment's points,
descriptors and scores sorted by score and the evaluation keeps the last 250 rows (utils/tester.py:209-213,
geometric_registration/evaluate.py:45-50); the KITTI tester keeps the top 250 per cloud (utils/tester.py:281-290).
Here all clouds of a stack are ordered by one device sort, with no host round trip, so the selection can run inside
a captured CUDA graph (encoder.GraphPipeline(..., keypoints=k)).

Order: within each cloud, ascending score, ties by ascending row -- np.argsort(s_b, kind="stable") -- with every NaN
(either sign) above +inf and -0.0 equal to +0.0. The top k of cloud b are argsort(s_b, kind="stable")[-k:] + start_b.
This is deliberately not io_utils.select_keypoints' order: that function uses numpy's default argsort, whose tie order
depends on the numpy build; on tie-free scores the two agree.

sample_keypoints draws the testers' `-rand` arm in the same layout. Its draws are counter-based (splitmix64 of the
seed and the slot, rng.cuh), so numpy's random stream is not reproduced.
"""
from collections import namedtuple

import torch

from . import _lib

KeypointSet = namedtuple("KeypointSet", "index count points descriptors scores")
KeypointSet.__doc__ = """Fixed-shape keypoints of B clouds, k slots each (slots j >= count[b] hold index -1 and zeros).
    index [B,k] int32 global rows, count [B] int32 = min(k, len_b), points [B,k,3], descriptors [B,k,D] and scores
    [B,k] float32 (None when the matching input was not given). Slots are in ascending score order; sample_keypoints'
    slots are in draw order and its count is k, or 0 for an empty cloud."""


def select_keypoints(scores, lengths, k=None, points=None, descriptors=None, *, rows=None):
    """scores [N] or [N,1] (CUDA float32), lengths [B] stack lengths.

    k=None: the full order int32 [N] -- every row, clouds in stack order, ascending score within each (the 3DMatch
    tester's layout). k: a KeypointSet with the top min(k, len_b) rows of every cloud, gathered from `points` [N,3]
    and `descriptors` [N,D] when given.
    rows: optional device int32 scalar with the actual row count (the static pyramid's level-0 count); N is then the
    capacity of the inputs and no row at or past it is read (order[rows:] is left unwritten)."""
    op = "select_keypoints"
    s = _lib.tensor_arg(scores, op + ": scores", torch.float32).reshape(-1)
    dev = s.device
    lens = _lib.i32(lengths, dev)
    N, B = int(s.shape[0]), int(lens.shape[0])
    pts = _lib.tensor_arg(points, op + ": points", torch.float32, (N, 3), dev, optional=True)
    desc = _lib.tensor_arg(descriptors, op + ": descriptors", torch.float32, (N, None), dev, optional=True)
    rows = _lib.row_count_arg(rows, op + ": rows", dev)
    D = int(desc.shape[1]) if desc is not None else 0
    lib = _lib.lib()
    ws = _lib.workspace(lib.d3f_select_keypoints_workspace_bytes(N, B), dev)
    i32, f32 = torch.int32, torch.float32
    if k is None:
        order = torch.empty((N,), dtype=i32, device=dev)
        _lib.check(lib.d3f_select_keypoints(_lib.ptr(s), _lib.ptr(lens), B, N, 0, None, None, 0, _lib.ptr(order),
                                            None, None, None, None, None, _lib.ptr(ws), ws.numel(), _lib.stream(),
                                            _lib.ptr(rows)), "d3f_select_keypoints")
        return order
    k = int(k)
    if k < 1:
        raise ValueError("select_keypoints: k=%d must be >= 1" % k)
    index = torch.empty((B, k), dtype=i32, device=dev)
    count = torch.empty((B,), dtype=i32, device=dev)
    out_s = torch.empty((B, k), dtype=f32, device=dev)
    out_p = torch.empty((B, k, 3), dtype=f32, device=dev) if pts is not None else None
    out_d = torch.empty((B, k, D), dtype=f32, device=dev) if desc is not None else None
    _lib.check(lib.d3f_select_keypoints(_lib.ptr(s), _lib.ptr(lens), B, N, k, _lib.ptr(pts), _lib.ptr(desc), D, None,
                                        _lib.ptr(index), _lib.ptr(count), _lib.ptr(out_p), _lib.ptr(out_d),
                                        _lib.ptr(out_s), _lib.ptr(ws), ws.numel(), _lib.stream(), _lib.ptr(rows)),
               "d3f_select_keypoints")
    return KeypointSet(index, count, out_p, out_d, out_s)


INT32_MAX = 2 ** 31 - 1
MAX_BATCH = 1024         # kMaxBatch of the library


def sample_keypoints(lengths, k, seed=0, points=None, descriptors=None, scores=None, *, rows=None):
    """Uniform random keypoints, k per cloud, drawn with replacement -- the testers' `-rand` arm, np.random.choice(n_b,
    k) per cloud (utils/tester.py:238-279, geometric_registration/evaluate.py:45-54) -- in select_keypoints' layout.

    Slot j of cloud b holds row start_b + (((z >> 32) * n_b) >> 32), z = splitmix64(seed + ((b << 32) | j) *
    0x9E3779B97F4A7C15) (oracle/keypoints_np.py). Each slot is its own draw, so the first c slots of a k-slot sample are
    the c-slot sample with the same seed. count[b] = k when cloud b has a row, else 0 (index -1, zero rows). Rows of no
    cloud are never drawn; a row may be drawn more than once. Slots are in draw order, not score order.
    lengths [B] stack lengths; points [N,3], descriptors [N,D], scores [N] or [N,1] (CUDA float32, each optional) are
    gathered. The clouds are cut at N, the rows of the inputs given (unbounded when none is), and at `rows`, an
    optional device int32 scalar with the actual row count (the static pyramid's level-0 count). No host
    synchronisation: the call can be captured in a CUDA graph."""
    op = "sample_keypoints"
    k = int(k)
    seed = int(seed)
    if not 0 <= seed < 2 ** 64:
        raise ValueError("%s: seed=%d must be in [0, 2^64)" % (op, seed))
    B = int(lengths.shape[0]) if torch.is_tensor(lengths) else len(lengths)
    if not 1 <= B <= MAX_BATCH:
        raise ValueError("%s: B=%d clouds must be in [1, %d]" % (op, B, MAX_BATCH))
    if k < 1 or B * k > INT32_MAX:
        raise ValueError("%s: k=%d must be >= 1 with B*k = %d within int32" % (op, k, B * k))
    dev = None
    N = None
    given = []
    for name, x, shape in (("points", points, (None, 3)), ("descriptors", descriptors, (None, None)),
                           ("scores", scores, None)):
        x = _lib.tensor_arg(x, "%s: %s" % (op, name), torch.float32, shape, dev, optional=True)
        if x is not None:
            if name == "scores":
                if x.dim() not in (1, 2) or (x.dim() == 2 and int(x.shape[1]) != 1):
                    raise ValueError("%s: scores must be [N] or [N, 1], got %s" % (op, list(x.shape)))
                x = x.reshape(-1)
            dev = x.device
            if N is not None and int(x.shape[0]) != N:
                raise ValueError("%s: %s has %d rows, the other inputs %d" % (op, name, int(x.shape[0]), N))
            N = int(x.shape[0])
        given.append(x)
    pts, desc, s = given
    if dev is None:
        dev = lengths.device if torch.is_tensor(lengths) and lengths.is_cuda else torch.device("cuda")
        N = INT32_MAX
    lens = _lib.i32(lengths, dev)
    rows = _lib.row_count_arg(rows, op + ": rows", dev)
    D = int(desc.shape[1]) if desc is not None else 0
    lib = _lib.lib()
    ws = _lib.workspace(lib.d3f_sample_keypoints_workspace_bytes(B), dev)
    i32, f32 = torch.int32, torch.float32
    index = torch.empty((B, k), dtype=i32, device=dev)
    count = torch.empty((B,), dtype=i32, device=dev)
    out_p = torch.empty((B, k, 3), dtype=f32, device=dev) if pts is not None else None
    out_d = torch.empty((B, k, D), dtype=f32, device=dev) if desc is not None else None
    out_s = torch.empty((B, k), dtype=f32, device=dev) if s is not None else None
    _lib.check(lib.d3f_sample_keypoints(_lib.ptr(lens), B, N, k, seed, _lib.ptr(pts), _lib.ptr(desc), D, _lib.ptr(s),
                                        _lib.ptr(index), _lib.ptr(count), _lib.ptr(out_p), _lib.ptr(out_d),
                                        _lib.ptr(out_s), _lib.ptr(ws), ws.numel(), _lib.stream(), _lib.ptr(rows)),
               "d3f_sample_keypoints")
    return KeypointSet(index, count, out_p, out_d, out_s)
