"""CPU: the voxel down-sampling contract (Open3D 0.7's voxel_down_sample, include/d3feat_b200.h) in two independent
restatements -- the C port (oracle/voxel_oracle.c) and a plain-Python dict loop below -- that agree bit for bit, a
hand-computed case, the sensitivity of the boundary data to every plausible wrong index computation, and the argument
contract of voxel.voxel_down_sample and of the C ABI, refused before any launch."""
import ctypes
import math
from fractions import Fraction

import numpy as np
import pytest
import torch

import _voxel_cases as vc


def dict_voxel_down_sample(points, lengths, v):
    """The literal loop in Python floats (IEEE doubles, one rounding per operation): per cloud the minimum of the
    finite rows, the voxel of every finite row, fp64 sums in input order, then ascending (iz, iy, ix)."""
    pts = np.asarray(points, np.float32)
    out, out_len, start = [], [], 0
    for n in lengths:
        rows = [tuple(float(c) for c in pts[i]) for i in range(min(start, len(pts)), min(start + int(n), len(pts)))]
        start += int(n)
        rows = [r for r in rows if all(math.isfinite(c) for c in r)]
        acc = {}
        if rows:
            lo = [min(r[a] for r in rows) - v * 0.5 for a in range(3)]
            for r in rows:
                key = tuple(math.floor((r[a] - lo[a]) / v) for a in (2, 1, 0))
                s = acc.setdefault(key, [0.0, 0.0, 0.0, 0])
                for a in range(3):
                    s[a] += r[a]
                s[3] += 1
        for key in sorted(acc):
            s = acc[key]
            out.append([np.float32(s[a] / float(s[3])) for a in range(3)])
        out_len.append(len(acc))
    return np.array(out, np.float32).reshape(-1, 3), np.array(out_len, np.int32)


def port(points, lengths, v):
    from oracle.voxel_native import port_voxel_down_sample
    return port_voxel_down_sample(points, lengths, v)


def assert_same(a, b):
    assert np.array_equal(a[1], b[1]), (a[1], b[1])
    assert np.array_equal(a[0].view(np.uint32), b[0].view(np.uint32))


def cases():
    rng = np.random.default_rng(7)
    out = [("boundary-%g" % v, p, l, v) for p, l, v in vc.boundary_clouds()]
    for s in range(3):
        p, l, v = vc.random_clouds(s, v=(0.1, 0.3, 0.03)[s], scale=(1.0, 3.0, 0.2)[s])
        out.append(("random-%d" % s, p, l, v))
        out.append(("non-finite-%d" % s, vc.with_non_finite(p, rng), l, v))
    p, l, v = vc.random_clouds(9)
    out.append(("rows-of-no-cloud", p, l[:2], v))
    out.append(("lengths-past-N", p[:500], l, v))
    out.append(("offset-1e5", p + np.float32(1e5), l, 0.0625))
    return out


@pytest.mark.parametrize("name,points,lengths,v", cases(), ids=[c[0] for c in cases()])
def test_c_port_equals_the_dict_restatement(name, points, lengths, v):
    assert_same(port(points, lengths, v), dict_voxel_down_sample(points, lengths, v))


def test_hand_computed_case():
    # v = 1: cloud 0 has min (0, 0, 0), so the grid starts at -0.5 and x = 0.4 -> voxel 0, x = 1.6 -> voxel 2,
    # y = 0.9 -> voxel 1. Cloud 1 is empty; cloud 2 keeps its one finite row.
    pts = np.array([[0, 0, 0], [0.4, 0, 0], [1.6, 0, 0], [0.2, 0.9, 0],
                    [np.nan, 1, 1], [5, 6, 7]], np.float32)
    want = np.array([[0.2, 0, 0], [1.6, 0, 0], [0.2, 0.9, 0], [5, 6, 7]], np.float32)
    for got in (port(pts, [4, 0, 2], 1.0), dict_voxel_down_sample(pts, [4, 0, 2], 1.0)):
        assert_same(got, (want, np.array([3, 0, 1], np.int32)))


# ---- sensitivity: the boundary data tells the contract from its plausible mistakes ---------------------------------

def _fma(a, b, c):
    return float(Fraction(a) * Fraction(b) + Fraction(c))


def voxel_indices(points, v, mode):
    """[n,3] voxel index of every row of ONE finite cloud, computed the contract's way ("exact") or a wrong way."""
    p = np.asarray(points, np.float32)
    if mode == "fp32":
        v32 = np.float32(v)
        lo = p.min(0) - v32 * np.float32(0.5)
        return np.floor((p - lo) / v32).astype(np.int64)
    vv = float(np.float32(v)) if mode == "float_v" else v
    lo = p.min(0).astype(np.float64) - vv * 0.5
    d = p.astype(np.float64)
    if mode in ("exact", "float_v"):
        return np.floor((d - lo) / vv).astype(np.int64)
    inv = 1.0 / vv
    if mode == "reciprocal":
        return np.floor((d - lo) * inv).astype(np.int64)
    assert mode == "fma"       # (p - lo) * inv expanded and contracted: fma(p, inv, -(lo * inv))
    return np.array([[math.floor(_fma(float(d[i, a]), inv, -(float(lo[a]) * inv))) for a in range(3)]
                     for i in range(d.shape[0])], np.int64)


@pytest.mark.parametrize("mode", ["reciprocal", "fp32", "fma", "float_v"])
def test_boundary_data_catches_a_wrong_index(mode):
    moved = 0
    for pts, lens, v in vc.boundary_clouds():
        start = 0
        for n in lens:
            c = pts[start:start + n]
            start += n
            moved += int((voxel_indices(c, v, mode) != voxel_indices(c, v, "exact")).any(1).sum())
    assert moved > 0, "no boundary row changes voxel under %s" % mode


def test_fp32_sums_would_change_the_average():
    """The fp64 sums matter: summing the same rows in fp32 changes some voxel's average."""
    pts, lens, v = vc.random_clouds(0, n=3000, scale=0.05, v=0.3, dup=0.0)
    want, _ = port(pts, lens, v)
    c = pts[:lens[0]]
    idx = voxel_indices(c, v, "exact")
    keys = np.unique(idx[:, ::-1], axis=0)[:, ::-1]
    got = []
    for k in keys:
        s = np.zeros(3, np.float32)
        rows = c[(idx == k).all(1)]
        for r in rows:
            s = (s + r).astype(np.float32)
        got.append(s / np.float32(rows.shape[0]))
    got = np.array(got, np.float32)
    assert not np.array_equal(got.view(np.uint32), want[:len(got)].view(np.uint32))


def test_double_voxel_size_is_not_float_voxel_size():
    """0.03 is used as the double 0.03: the float32 0.03 voxelises the boundary data differently."""
    pts, lens, v = vc.boundary_clouds()[0]
    assert v == 0.03
    a = port(pts, lens, 0.03)
    b = port(pts, lens, float(np.float32(0.03)))
    assert not (np.array_equal(a[1], b[1]) and np.array_equal(a[0].view(np.uint32), b[0].view(np.uint32)))


# ---- argument contract ------------------------------------------------------------------------------------------------

class Stub:
    def __getattr__(self, symbol):
        raise AssertionError("reached the library with a bad argument: %s" % symbol)


@pytest.fixture
def stub_lib(monkeypatch):
    """The library replaced by a stub whose every symbol raises, and CPU tensors standing in for device tensors (the
    checks only read attributes): a missing check cannot reach a GPU, it fails here."""
    from d3feat_b200 import _lib
    monkeypatch.setattr(_lib, "DEVICE_TYPE", "cpu")
    monkeypatch.setattr(_lib, "lib", lambda: Stub())


def _legal():
    return dict(points=torch.zeros((6, 3), dtype=torch.float32), lengths=torch.tensor([4, 2], dtype=torch.int32),
                voxel_size=0.03)


BAD = [
    ("points", torch.zeros((6, 3), dtype=torch.float64), "points"),
    ("points", torch.zeros((6, 3), dtype=torch.float16), "points"),
    ("points", torch.zeros((6, 3), dtype=torch.int32), "points"),
    ("points", torch.zeros((6, 3), dtype=torch.float32, device="meta"), "points"),
    ("points", torch.zeros((6, 2), dtype=torch.float32), "points"),
    ("points", torch.zeros((18,), dtype=torch.float32), "points"),
    ("points", np.zeros((6, 3), np.float32), "points"),
    ("lengths", torch.tensor([4, 2], dtype=torch.int64), "lengths"),
    ("lengths", torch.tensor([4.0, 2.0], dtype=torch.float32), "lengths"),
    ("lengths", torch.tensor([[4, 2]], dtype=torch.int32), "lengths"),
    ("lengths", torch.zeros((2,), dtype=torch.int32, device="meta"), "lengths"),
    ("lengths", torch.zeros((0,), dtype=torch.int32), "lengths"),
    ("lengths", torch.ones((1025,), dtype=torch.int32), "lengths"),
    ("voxel_size", 0.0, "voxel_size"),
    ("voxel_size", -0.03, "voxel_size"),
    ("voxel_size", float("nan"), "voxel_size"),
    ("voxel_size", float("inf"), "voxel_size"),
    ("voxel_size", float("-inf"), "voxel_size"),
    ("voxel_size", None, "voxel_size"),
    ("voxel_size", "0.03", "voxel_size"),
    ("bbox", [0, 0, 0, 1, 1], "bbox"),
    ("bbox", [0, 0, 0, 1, float("nan"), 1], "bbox"),
]


@pytest.mark.parametrize("key,value,name", BAD, ids=["%s-%d" % (b[0], i) for i, b in enumerate(BAD)])
def test_bad_argument_is_refused(stub_lib, key, value, name):
    from d3feat_b200.voxel import voxel_down_sample
    a = _legal()
    a[key] = value
    with pytest.raises(ValueError) as e:
        voxel_down_sample(**a)
    assert name in str(e.value), e.value


@pytest.mark.parametrize("strided", [False, True])
def test_legal_arguments_reach_the_library(stub_lib, strided):
    from d3feat_b200.voxel import voxel_down_sample
    a = _legal()
    if strided:   # a strided view is copied, not refused
        a["points"] = torch.zeros((6, 4), dtype=torch.float32)[:, :3]
    with pytest.raises(AssertionError, match="reached the library"):
        voxel_down_sample(**a)


def test_pipeline_needs_a_raw_capacity_with_a_voxel_size():
    from d3feat_b200.encoder import GraphPipeline
    with pytest.raises(ValueError, match="raw_capacity"):
        GraphPipeline(None, [256], 1, np.zeros(6, np.float32), voxel_size=0.03)


@pytest.fixture(scope="module")
def abi():
    from d3feat_b200 import _lib, build
    build.build()
    return _lib.lib()


def _call(lib, B=2, N=100, v=0.03, bbox=(0, 0, 0, 1, 1, 1), ws_bytes=1 << 30, cap=-1):
    fake = ctypes.c_void_p(256)
    bb = None if bbox is None else (ctypes.c_float * 6)(*bbox)
    return lib.d3f_voxel_down_sample(fake, fake, B, N, None, v, bb, fake, fake, fake, cap, None, fake, ws_bytes, None)


@pytest.mark.parametrize("kw,code,msg", [
    (dict(v=0.0), -1, b"voxel_size"), (dict(v=-1.0), -1, b"voxel_size"), (dict(v=float("nan")), -1, b"voxel_size"),
    (dict(v=float("inf")), -1, b"voxel_size"), (dict(B=0), -1, b"B=0"), (dict(B=1025), -1, b"B=1025"),
    (dict(N=-1), -1, b"N=-1"), (dict(bbox=None), -1, b"host_bbox"),
    (dict(bbox=(0, 0, 0, 1, float("inf"), 1)), -1, b"host_bbox"), (dict(ws_bytes=16), -4, b"workspace"),
    (dict(bbox=(0, 0, 0, 1e5, 1e5, 1e5), v=1e-4), -2, b"sort key"),
], ids=lambda x: str(x) if not isinstance(x, dict) else ",".join("%s=%s" % i for i in x.items()))
def test_abi_refuses_before_any_cuda_call(abi, kw, code, msg):
    """Every argument error is returned before a CUDA call (the fake pointers are never dereferenced)."""
    assert _call(abi, **kw) == code
    assert msg in abi.d3f_last_error()
