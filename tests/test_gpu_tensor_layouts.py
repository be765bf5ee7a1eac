"""GPU: legal but awkward tensors give the same answer.

Every other GPU test feeds the ops fresh, 256-byte aligned, contiguous allocations. Here each pointer argument in turn
is a contiguous view that starts 4, 8 or 12 bytes past a 16-byte boundary (what a row slice P[n0:n1] of a stacked
[N, 3] batch is for three of every four n0), or a strided view (a column slice, every second row, a transpose, an
expanded row, scan[:, :3] of a KITTI [N, 4] scan). Where the argument cannot change which kernel or arm runs, the result
equals the plain-tensor result bit for bit; where a 16-byte alignment predicate flips, the table names the kernel that
must run instead (torch.profiler) and the result is checked element by element against float64. The C ABI takes a
caller-owned output, so the output halves of the predicates are reached by calling it with a shifted, sentinel-filled
buffer: nothing outside the rows and columns of the result is written.

The cases run in an interpreter of their own (one child pytest session for the whole file, started by the first case).
Most of them name kernels from torch.profiler's records, and in a long session the profiler can stop delivering any:
after tests/test_gpu_tensor_core.py or tests/test_gpu_real_configs.py has run in the same process every later capture
comes back empty, retries included. Which kernel ran is the point of this file, so it does not depend on what the
process did before.
"""
import functools
import os
import subprocess
import sys
import tempfile
import xml.etree.ElementTree as ET

import numpy as np
import pytest
import torch

from _oracle import TOL, assert_close, epilogue, gemm_mag, kpconv_ref
from oracle import kpconv_np as ok
from oracle import native as on
from test_gpu_gemm_epilogue import SENTINEL, unary_into
from test_gpu_kernel_variants import (ANYK, F32, FAST4, FAST8, GENERIC, GENERIC_D, SPLITK, STAGED8, assert_ran, kc,
                                      kp_inputs, launched, mma, t)

pytestmark = pytest.mark.gpu

TC = "tc_gemm_kernel<"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CHILD = "D3F_LAYOUTS_CHILD"          # set in the child session, where the cases really run
_child = None


def child_results():
    """{case name: None if it passed, else its failure text} of one child pytest session over this file."""
    global _child
    if _child is None:
        with tempfile.TemporaryDirectory() as d:
            report = os.path.join(d, "report.xml")
            cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + [
                "-m", "pytest", os.path.abspath(__file__), "-m", "gpu", "-q", "-s", "-p", "no:cacheprovider",
                "--junitxml", report]
            r = subprocess.run(cmd, env=dict(os.environ, **{CHILD: "1"}), cwd=ROOT, capture_output=True, text=True,
                               timeout=1700)
            print("\n".join(l for l in r.stdout.splitlines() if l.lstrip(".").startswith(("RATIO", "PREDICATE"))))
            assert os.path.exists(report), "the child session wrote no report:\n%s\n%s" % (r.stdout[-3000:],
                                                                                          r.stderr[-3000:])
            _child = {}
            for case in ET.parse(report).getroot().iter("testcase"):
                bad = [e for e in case if e.tag in ("failure", "error", "skipped")]
                text = "\n".join("%s: %s\n%s" % (e.tag, e.get("message"), e.text) for e in bad)
                _child[case.get("name")] = text or None
    return _child


def fresh_process(fn):
    """Run the case in the child session; in the parent, report what it did there."""
    @functools.wraps(fn)
    def wrapper(*args, **kw):
        if os.environ.get(CHILD):
            return fn(*args, **kw)
        name = os.environ["PYTEST_CURRENT_TEST"].split("::")[-1].rsplit(" ", 1)[0]
        results = child_results()
        assert name in results, "the child session did not run %s (it ran %s)" % (name, sorted(results))
        assert results[name] is None, results[name]
    return wrapper
FLIPPED = {}          # predicate -> kernel / arm that ran when it was false


def shifted(a, dev, off=1):
    """Contiguous device copy of `a` that starts `off` elements past a 16-byte boundary (8 bytes for float64)."""
    a = np.ascontiguousarray(a)
    src = torch.from_numpy(a)
    buf = torch.empty(a.size + 8, dtype=src.dtype, device=dev)
    assert buf.data_ptr() % 16 == 0
    view = buf[off:off + a.size].view(a.shape)
    view.copy_(src)
    assert view.is_contiguous() and view.data_ptr() % 16 == (off * a.itemsize) % 16 != 0
    return view


def strided(a, dev, how):
    """A non-contiguous device view holding `a`."""
    src = torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    n, c = a.shape
    if how == "cols0":                                   # wide[:, :C], e.g. scan[:, :3] of an [N, 4] scan
        v = torch.zeros((n, c + 1), dtype=src.dtype, device=dev)[:, :c]
    elif how == "cols1":                                 # wide[:, 1:C + 1]
        v = torch.zeros((n, c + 2), dtype=src.dtype, device=dev)[:, 1:c + 1]
    elif how == "rows2":                                 # tall[::2]
        v = torch.zeros((2 * n, c), dtype=src.dtype, device=dev)[::2]
    else:                                                # a transposed buffer
        v = torch.zeros((c, n), dtype=src.dtype, device=dev).t()
    v.copy_(src)
    assert not v.is_contiguous() or min(n, c) <= 1
    return v


HOWS = ("cols0", "cols1", "rows2", "t")


names_of = launched          # (result of fn(), names of the kernels it launched)


def ran(names, kernel):
    return any(kernel in n for n in names)


# ---------------------------------------------------------------------------------------------------------------------
#  unary convolution
# ---------------------------------------------------------------------------------------------------------------------

UNARY = [(3000, 64, 32), (3000, 64, 128), (3000, 256, 128), (645, 1024, 256), (195, 512, 2048), (9000, 64, 48)]


def unary_case(N, Cin, Cout):
    rng = np.random.default_rng(N + 7 * Cin + Cout)
    a = dict(features=rng.normal(size=(N, Cin)).astype(np.float32),
             K_values=(rng.normal(size=(Cin, Cout)) * np.sqrt(2.0 / Cout)).astype(np.float32),
             scale=rng.uniform(0.5, 1.5, Cout).astype(np.float32), shift=rng.normal(size=Cout).astype(np.float32),
             residual=rng.normal(size=(N, Cout)).astype(np.float32))
    ref, mag = epilogue(a["features"].astype(np.float64) @ a["K_values"].astype(np.float64),
                        gemm_mag(a["features"], a["K_values"]), a["scale"], a["shift"], residual=a["residual"],
                        alpha=0.2)
    return a, ref, mag


def run_unary(T):
    from d3feat_b200 import convolution_ops as co
    return names_of(lambda: co.unary_convolution(T["features"], T["K_values"], epilogue=(T["scale"], T["shift"], 0.2),
                                                 residual=T["residual"]))


@pytest.mark.parametrize("N,Cin,Cout", UNARY)
@fresh_process
def test_unary_convolution_layouts(cuda, N, Cin, Cout):
    a, ref, mag = unary_case(N, Cin, Cout)
    what = "layout unary %dx%d->%d" % (N, Cin, Cout)
    plain = {k: t(v, cuda) for k, v in a.items()}
    base, names = run_unary(plain)
    assert ran(names, TC) and not ran(names, F32)
    assert_close(base.cpu().numpy(), ref, mag, TOL, what)
    # the weights are repacked, the vectors go through shared memory, and a misaligned residual takes the float-by-
    # float arm of the same epilogue: same kernel, same bits
    for i, key in enumerate(("K_values", "scale", "shift", "residual")):
        out, names = run_unary(dict(plain, **{key: shifted(a[key], cuda, 1 + i % 3)}))
        assert ran(names, TC) and not ran(names, F32), key
        assert torch.equal(out, base), key
    if Cout % 4 == 0:
        FLIPPED["tc epilogue vec (residual)"] = "tc_gemm_kernel, scalar arm"
    # features off a 16-byte boundary cannot be fetched by TMA: the CUDA-core GEMM, scalar A loads
    fall = []
    for off in (1, 2, 3):
        out, names = run_unary(dict(plain, features=shifted(a["features"], cuda, off)))
        assert ran(names, F32) and not ran(names, TC), off
        assert_close(out.cpu().numpy(), ref, mag, TOL, what + " (features + %d B: gemm_f32)" % (4 * off))
        fall.append(out)
    FLIPPED["tc_gemm_supported (A)"] = FLIPPED["gemm_f32 a_vec"] = F32
    assert torch.equal(fall[0], fall[1]) and torch.equal(fall[0], fall[2])
    out, names = run_unary({k: shifted(v, cuda, 1 + i % 3) for i, (k, v) in enumerate(a.items())})
    assert ran(names, F32) and not ran(names, TC)
    assert torch.equal(out, fall[0])              # b_vec false as well: the same sums, element by element
    FLIPPED["gemm_f32 b_vec"] = F32
    for how in HOWS:                              # strided views are copied, and the copy is aligned
        out, names = run_unary({k: strided(v, cuda, how) if v.ndim == 2 else t(v, cuda) for k, v in a.items()})
        assert ran(names, TC) and torch.equal(out, base), how


@pytest.mark.parametrize("N,Cin,Cout", [(3000, 64, 32), (645, 1024, 256), (9000, 64, 48)])
@pytest.mark.parametrize("with_rows", [False, True])
@fresh_process
def test_unary_abi_shifted_output(cuda, N, Cin, Cout, with_rows):
    """d3f_unary_forward into a caller's misaligned buffer: the rows below the count equal the aligned result bit for
    bit, and no other float of the buffer is written."""
    a, ref, mag = unary_case(N, Cin, Cout)
    T = {k: t(v, cuda) for k, v in a.items()}
    m = N - 77 if with_rows else N
    rows = torch.tensor([m], dtype=torch.int32, device=cuda) if with_rows else None
    kw = dict(scale=T["scale"], shift=T["shift"], residual=T["residual"], alpha=0.2, rows=rows)
    want = torch.full((N * Cout,), SENTINEL, dtype=torch.float32, device=cuda)
    unary_into(want, T["features"], T["K_values"], N, **kw)
    for off in (1, 2, 3):
        buf = torch.full((N * Cout + 16,), SENTINEL, dtype=torch.float32, device=cuda)
        out = buf[4 + off:4 + off + N * Cout]
        assert out.data_ptr() % 16 == 4 * off
        _, names = names_of(lambda: unary_into(out, T["features"], T["K_values"], N, **kw))
        assert ran(names, TC)
        assert torch.equal(out, want)
        assert bool((out[m * Cout:] == SENTINEL).all()) and bool((buf[:4 + off] == SENTINEL).all())
        assert bool((buf[4 + off + N * Cout:] == SENTINEL).all())
    assert_close(want[:m * Cout].view(m, Cout).cpu().numpy(), ref[:m], mag[:m], TOL, "layout unary abi %d" % N)
    if Cout % 4 == 0:
        FLIPPED["tc epilogue vec (C)"] = "tc_gemm_kernel, scalar arm"


# ---------------------------------------------------------------------------------------------------------------------
#  the resnetb tail pair
# ---------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("N,C1,C2,Cout", [(5000, 32, 64, 128), (700, 512, 1024, 2048)])
@fresh_process
def test_unary_pair_layouts(cuda, N, C1, C2, Cout):
    from d3feat_b200 import convolution_ops as co
    rng = np.random.default_rng(N + C1)
    a = dict(x1=rng.normal(size=(N, C1)), w1=rng.normal(size=(C1, Cout)) * np.sqrt(2.0 / Cout),
             s1=rng.uniform(0.5, 1.5, Cout), t1=rng.normal(size=Cout), x2=rng.normal(size=(N, C2)),
             w2=rng.normal(size=(C2, Cout)) * np.sqrt(2.0 / Cout), s2=rng.uniform(0.5, 1.5, Cout),
             t2=rng.normal(size=Cout))
    a = {k: v.astype(np.float32) for k, v in a.items()}
    f = lambda v: v.astype(np.float64)
    y1, m1 = epilogue(f(a["x1"]) @ f(a["w1"]), gemm_mag(a["x1"], a["w1"]), a["s1"], a["t1"])
    y2, m2 = epilogue(f(a["x2"]) @ f(a["w2"]), gemm_mag(a["x2"], a["w2"]), a["s2"], a["t2"])
    ref, mag = epilogue(y1 + y2, m1 + m2, alpha=0.2)
    what = "layout pair %dx(%d|%d)->%d" % (N, C1, C2, Cout)

    def run(T):
        return names_of(lambda: co.unary_pair_convolution(T["x1"], T["w1"], (T["s1"], T["t1"]), T["x2"], T["w2"],
                                                          (T["s2"], T["t2"]), 0.2))
    plain = {k: t(v, cuda) for k, v in a.items()}
    base, names = run(plain)
    assert ran(names, TC) and not ran(names, F32)
    assert_close(base.cpu().numpy(), ref, mag, TOL, what)
    for i, key in enumerate(("s1", "t1", "s2", "t2")):      # folded into the packed image and the bias: same bits
        plain_w = dict(plain, w1=t(a["w1"], cuda), w2=t(a["w2"], cuda))      # fresh weights: the fold is cached per pair
        out, names = run(dict(plain_w, **{key: shifted(a[key], cuda, 1 + i % 3)}))
        assert not ran(names, F32) and torch.equal(out, base), key
    # one misaligned A operand: the one-GEMM kernel fetches both by TMA, so the two-call path must serve the call
    for key in ("x1", "x2"):
        for off in (1, 3):
            out, names = run(dict(plain, **{key: shifted(a[key], cuda, off)}))
            assert ran(names, F32) and ran(names, TC), (key, off)
            assert_close(out.cpu().numpy(), ref, mag, TOL, what + " (%s + %d B: two calls)" % (key, 4 * off))
    FLIPPED["pair: 16-byte aligned x1 / x2"] = "two unary_convolution calls"
    out, names = run({k: shifted(v, cuda, 2) for k, v in a.items()})
    assert ran(names, F32) and not ran(names, TC)
    assert_close(out.cpu().numpy(), ref, mag, TOL, what + " (all + 8 B)")
    out, names = run({k: strided(v, cuda, "cols1") if k in ("x1", "x2") else t(v, cuda) for k, v in a.items()})
    assert torch.equal(out, base) and not ran(names, F32)


# ---------------------------------------------------------------------------------------------------------------------
#  KPConv
# ---------------------------------------------------------------------------------------------------------------------

def lc(id, base, fallback, Cin, Cout, H, **kw):
    """A KPConv case: the stage-1 kernel of plain tensors, and of a misaligned feature tensor (None: the same)."""
    c = kc("layout_" + id, [base], Cin, Cout, 300, 450, H, **kw)
    c["fallback"] = fallback
    return c


KP_LAYOUT = [
    lc("fast4", FAST4, GENERIC, 32, 32, 40, epi=True),
    lc("fast8_h13", FAST8, GENERIC, 64, 64, 13, order=True),
    lc("fast8_wide", FAST8, GENERIC, 256, 32, 13),
    lc("mma4_gaussian", mma(4, False, False), GENERIC, 32, 32, 40, infl="gaussian"),
    lc("v2_2_2", "kpconv_stage1_v2_kernel<2,2,false>", GENERIC, 96, 32, 13, epi=True),
    lc("generic_cin5", GENERIC, None, 5, 32, 40),
    lc("anyk_k7", ANYK, None, 32, 32, 13, K=7),
    lc("cin1", "kpconv_cin1_kernel<true>", None, 1, 64, 40, epi=True),
    lc("staged8", STAGED8, GENERIC, 64, 32, 40, env={"D3F_S1_STAGED": "1"}),
    lc("splitk_cin64", SPLITK, GENERIC, 64, 64, 37, epi=True),
    dict(kc("layout_fused_cin32", ["kpconv_fused32_kernel"], 32, 32, 4000, 4000, 35, epi=True, extent=0.05,
            env={"D3F_FUSED_KPCONV": "1"}), fallback=GENERIC),
    lc("mma4_deform", mma(4, True, True), GENERIC_D, 32, 32, 40, kind="deform"),
    lc("mma16_modulated", mma(16, True, True), GENERIC_D, 128, 32, 13, kind="mod", epi=True),
    lc("v2_2_1_deform", "kpconv_stage1_v2_kernel<2,1,true>", GENERIC_D, 192, 32, 13, kind="deform"),
    lc("generic_deform", GENERIC_D, None, 5, 32, 40, kind="deform"),
    lc("anyk_k8_modulated", "kpconv_stage1_anyk_kernel<true>", None, 32, 32, 13, K=8, kind="mod"),
]


def kp_tensors(c):
    q, s, idx, f, Kp, W, off, mod, epi, order = kp_inputs(c)
    a = dict(query_points=q, support_points=s, neighbors_indices=idx, features=f, K_points=Kp, K_values=W)
    if off is not None:
        a["offsets"] = off
    if mod is not None:
        a["modulations"] = mod
    if epi is not None:
        a["scale"], a["shift"] = epi[0], epi[1]
    if order is not None:
        a["query_order"] = order
    ref = kpconv_ref(q, s, idx, f, Kp, W, c["extent"], c["infl"], c["mode"], off, mod, deform=c["kind"] != "rigid",
                     epi=epi)
    return a, ref


def run_kp(c, T):
    from d3feat_b200 import convolution_ops as co
    e = (T["scale"], T["shift"], 0.2) if "scale" in T else None
    head = [T[k] for k in ("query_points", "support_points", "neighbors_indices", "features", "K_points")]
    if c["kind"] == "rigid":
        fn = lambda: co.KPConv_ops(*head, T["K_values"], c["extent"], c["infl"], c["mode"], epilogue=e,
                                   query_order=T.get("query_order"))
    else:
        fn = lambda: co.KPConv_deform_ops(*head, T["offsets"], T.get("modulations"), T["K_values"], c["extent"],
                                          c["infl"], c["mode"], epilogue=e, query_order=T.get("query_order"))
    return names_of(fn)


@pytest.mark.parametrize("c", KP_LAYOUT, ids=[c["id"][7:] for c in KP_LAYOUT])
@fresh_process
def test_kpconv_layouts(cuda, monkeypatch, c):
    for k, v in c["env"].items():
        monkeypatch.setenv(k, v)
    a, (ref, mag, alt) = kp_tensors(c)
    plain = {k: t(v, cuda) for k, v in a.items()}
    base, names = run_kp(c, plain)
    assert_ran(names, c["expect"])
    assert_close(base.cpu().numpy(), ref, mag, TOL, c["id"], alt=alt)
    # no kernel makes a 16-byte access to any of these: same kernels, same bits
    for i, key in enumerate(k for k in a if k != "features"):
        out, names = run_kp(c, dict(plain, **{key: shifted(a[key], cuda, 1 + i % 3)}))
        assert_ran(names, c["expect"])
        assert torch.equal(out, base), key
    for off in (1, 2, 3):
        out, names = run_kp(c, dict(plain, features=shifted(a["features"], cuda, off)))
        if c["fallback"] is None:                 # scalar feature reads already
            assert_ran(names, c["expect"])
            assert torch.equal(out, base), off
        else:                                     # al16 / the fused kernel's eligibility / the vectorised packing flip
            assert_ran(names, [c["fallback"]])
            assert not ran(names, "prep_supports_vec_kernel") and not ran(names, "kpconv_fused32_kernel")
            assert_close(out.cpu().numpy(), ref, mag, TOL, c["id"] + " (features + %d B)" % (4 * off), alt=alt)
            fall = out if off == 1 else fall
            assert torch.equal(out, fall), off
    if c["fallback"] is not None:
        FLIPPED["kpconv al16 (feat)"] = FLIPPED["prep_supports vec"] = c["fallback"] + ", prep_supports_kernel"
        if c["env"].get("D3F_FUSED_KPCONV"):
            FLIPPED["fused eligibility (feat)"] = c["fallback"]
        out, names = run_kp(c, {k: shifted(v, cuda, 1 + i % 3) for i, (k, v) in enumerate(a.items())})
        assert_ran(names, [c["fallback"]])
        assert torch.equal(out, fall)
    T = dict(plain)
    for how, key in zip(HOWS, ("query_points", "support_points", "neighbors_indices", "features")):
        if a[key].shape[1] > 1:
            T[key] = strided(a[key], cuda, how)
    out, names = run_kp(c, T)
    assert_ran(names, c["expect"])
    assert torch.equal(out, base)


@fresh_process
def test_kpconv_abi_shifted_output(cuda):
    """d3f_kpconv_forward into a caller's misaligned buffer, with a device row count and a query order: the rows below
    the count equal the aligned result bit for bit, nothing else is written."""
    from d3feat_b200 import _lib
    from d3feat_b200 import convolution_ops as co
    c = lc("abi", FAST4, GENERIC, 32, 32, 40, epi=True, order=True)
    a, (ref, mag, alt) = kp_tensors(c)
    T = {k: t(v, cuda) for k, v in a.items()}
    Nq, Ns, H, K, Cin, Cout = c["Nq"], c["Ns"], c["H"], 15, 32, 32
    m = Nq - 77
    order = np.concatenate([np.random.default_rng(3).permutation(m), np.arange(m, Nq)]).astype(np.int32)
    T["query_order"] = t(order, cuda)             # the first m visits are the rows below the count
    rows_q = torch.tensor([m], dtype=torch.int32, device=cuda)
    L = _lib.lib()
    ws = _lib.workspace(L.d3f_kpconv_workspace_bytes(Nq, Ns, H, K, Cin, Cout), cuda)

    def into(out):
        _lib.check(L.d3f_kpconv_forward(
            *[_lib.ptr(T[k]) for k in ("query_points", "support_points", "neighbors_indices", "features", "K_points",
                                       "K_values")], _lib.ptr(co.packed_weight(T["K_values"])),
            _lib.ptr(T["query_order"]), Nq, Ns, H, K, Cin, Cout, c["extent"], 1, 0, 1, _lib.ptr(T["scale"]),
            _lib.ptr(T["shift"]), None, 0.2, _lib.ptr(out), _lib.ptr(ws), ws.numel(), _lib.stream(), _lib.ptr(rows_q),
            None), "d3f_kpconv_forward")
    want = torch.full((Nq * Cout,), SENTINEL, dtype=torch.float32, device=cuda)
    into(want)
    got = want.view(Nq, Cout).cpu().numpy()
    assert_close(got[:m], ref[:m], mag[:m], TOL, "layout kpconv abi", alt=alt[:m])
    assert np.all(got[m:] == SENTINEL)
    for off in (1, 2, 3):
        buf = torch.full((Nq * Cout + 16,), SENTINEL, dtype=torch.float32, device=cuda)
        out = buf[4 + off:4 + off + Nq * Cout]
        _, names = names_of(lambda: into(out))
        assert ran(names, FAST4) and ran(names, TC)
        assert torch.equal(out, want)
        assert bool((buf[:4 + off] == SENTINEL).all()) and bool((buf[4 + off + Nq * Cout:] == SENTINEL).all())


# ---------------------------------------------------------------------------------------------------------------------
#  pools and the point-wise kernels
# ---------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("C", [64, 128, 45])
@fresh_process
def test_pool_layouts(cuda, C):
    from d3feat_b200 import _lib
    from d3feat_b200 import network_blocks as nb
    rng = np.random.default_rng(C)
    N1, N2, H = 900, 301, 17
    x = rng.normal(size=(N1, C)).astype(np.float32)
    inds = rng.integers(0, N1 + 1, (N2, H)).astype(np.int32)
    inds[5] = N1                                                     # an all-shadow row -> column minima
    want_max, want_closest = ok.ind_max_pool(x, inds), ok.closest_pool(x, inds)
    v4 = "ind_max_pool_kernel<4>" if C % 4 == 0 else "ind_max_pool_kernel<1>"
    base, names = names_of(lambda: nb.ind_max_pool(t(x, cuda), t(inds, cuda)))
    assert ran(names, v4) and np.array_equal(base.cpu().numpy(), want_max)
    for off in (1, 2, 3):
        out, names = names_of(lambda: nb.ind_max_pool(shifted(x, cuda, off), t(inds, cuda)))
        assert ran(names, "ind_max_pool_kernel<1>") and torch.equal(out, base)
        out, names = names_of(lambda: nb.ind_max_pool(t(x, cuda), shifted(inds, cuda, off)))
        assert ran(names, v4) and torch.equal(out, base)
        out = nb.closest_pool(shifted(x, cuda, off), shifted(inds, cuda, 4 - off))
        assert np.array_equal(out.cpu().numpy(), want_closest)
    if C % 4 == 0:
        FLIPPED["pool v4 (x)"] = "ind_max_pool_kernel<1>"
    for how in HOWS:
        assert torch.equal(nb.ind_max_pool(strided(x, cuda, how), strided(inds, cuda, how)), base)
        assert np.array_equal(nb.closest_pool(strided(x, cuda, how), strided(inds, cuda, how)).cpu().numpy(),
                              want_closest)
    # the ABI with a caller's misaligned output and device row counts
    L = _lib.lib()
    tx, ti = t(x, cuda), t(inds, cuda)
    m = N2 - 40
    rows_out = torch.tensor([m], dtype=torch.int32, device=cuda)
    ws = _lib.workspace(L.d3f_ind_max_pool_workspace_bytes(C), cuda)
    for off in (1, 3):
        for pool in ("max", "closest"):
            buf = torch.full((N2 * C + 16,), SENTINEL, dtype=torch.float32, device=cuda)
            out = buf[4 + off:4 + off + N2 * C]
            if pool == "max":
                fn = lambda: _lib.check(L.d3f_ind_max_pool(_lib.ptr(tx), _lib.ptr(ti), N1, N2, H, C, _lib.ptr(out),
                                                           _lib.ptr(ws), ws.numel(), _lib.stream(), None,
                                                           _lib.ptr(rows_out)), "d3f_ind_max_pool")
            else:
                fn = lambda: _lib.check(L.d3f_closest_pool(_lib.ptr(tx), _lib.ptr(ti), N1, N2, H, C, _lib.ptr(out),
                                                           _lib.stream(), None, _lib.ptr(rows_out)), "d3f_closest_pool")
            _, names = names_of(fn)
            if pool == "max":
                assert ran(names, "ind_max_pool_kernel<1>")
            got = out.view(N2, C).cpu().numpy()
            assert np.array_equal(got[:m], (want_max if pool == "max" else want_closest)[:m])
            assert np.all(got[m:] == SENTINEL)
            assert bool((buf[:4 + off] == SENTINEL).all()) and bool((buf[4 + off + N2 * C:] == SENTINEL).all())
    if C % 4 == 0:
        FLIPPED["pool v4 (out)"] = "ind_max_pool_kernel<1>"


@pytest.mark.parametrize("C", [32, 33])
@fresh_process
def test_pointwise_layouts(cuda, C):
    from d3feat_b200 import network_blocks as nb
    rng = np.random.default_rng(C)
    lengths = np.array([700, 1, 500], np.int32)
    N, H = int(lengths.sum()), 20
    x = rng.normal(size=(N, C)).astype(np.float32)
    scale, shift = rng.uniform(0.5, 1.5, C).astype(np.float32), rng.normal(size=C).astype(np.float32)
    res = rng.normal(size=(N, C)).astype(np.float32)
    start = np.concatenate([[0], np.cumsum(lengths)])
    nbr = np.full((N, H), N, np.int32)
    for b in range(3):
        nbr[start[b]:start[b + 1], :H - 3] = rng.integers(start[b], start[b + 1], (lengths[b], H - 3))
    a = dict(x=x, scale=scale, shift=shift, res=res)
    affine = lambda T: nb._affine_leaky(T["x"], T["scale"], T["shift"], T["res"], 0.2)
    plain = {k: t(v, cuda) for k, v in a.items()}
    base = affine(plain)
    y, mag = epilogue(x, np.abs(x), scale, shift, residual=res, alpha=0.2)
    assert_close(base.cpu().numpy(), y, mag, TOL, "layout affine_leaky C=%d" % C)
    for i, key in enumerate(a):
        assert torch.equal(affine(dict(plain, **{key: shifted(a[key], cuda, 1 + i % 3)})), base), key
    assert torch.equal(affine({k: strided(v, cuda, "cols1") if v.ndim == 2 else t(v, cuda) for k, v in a.items()}), base)
    l2 = nb.l2_normalize(plain["x"])
    x64 = x.astype(np.float64)
    want = x64 / np.sqrt(np.maximum((x64 * x64).sum(1, keepdims=True), 1e-10))
    assert np.abs(l2.cpu().numpy() - want).max() < 1e-6
    for off in (1, 2, 3):
        assert torch.equal(nb.l2_normalize(shifted(x, cuda, off)), l2)
    assert torch.equal(nb.l2_normalize(strided(x, cuda, "rows2")), l2)
    s = dict(x=x, nbr=nbr, lengths=lengths)
    scores = lambda T: nb.detection_scores(T["x"], T["nbr"], T["lengths"])
    plain = {k: t(v, cuda) for k, v in s.items()}
    base = scores(plain)
    ref, mag, alt = ok.detection_scores(x64, nbr, lengths, magnitude=True)
    assert_close(base.cpu().numpy(), ref, mag, TOL, "layout detection_scores C=%d" % C, alt=alt)
    for i, key in enumerate(s):
        assert torch.equal(scores(dict(plain, **{key: shifted(s[key], cuda, 1 + i % 3)})), base), key
    assert torch.equal(scores(dict(plain, x=strided(x, cuda, "t"), nbr=strided(nbr, cuda, "cols0"))), base)


# ---------------------------------------------------------------------------------------------------------------------
#  the native ops: hash grid, radius neighbours, grid subsampling
# ---------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("B", [1, 3, 33])
@pytest.mark.parametrize("n0", [1, 2, 3])
@fresh_process
def test_native_ops_on_row_slices(cuda, B, n0):
    """The clouds are rows [n0, n1) of a longer stacked batch and the lengths a slice of a longer vector: contiguous,
    12 n0 bytes and 4 n0 bytes past a 16-byte boundary."""
    from d3feat_b200 import tf_custom_ops as ops
    rng = np.random.default_rng(10 * B + n0)
    lens = rng.integers(40, 400, B).astype(np.int32)
    if B > 1:
        lens[1] = 1
    N = int(lens.sum())
    P = rng.uniform(0, 1, (N, 3)).astype(np.float32)
    r, dl = 0.11, 0.08
    whole = torch.zeros((N + 8, 3), dtype=torch.float32, device=cuda)
    whole[n0:n0 + N].copy_(torch.from_numpy(P))
    pts = whole[n0:n0 + N]
    lv = torch.zeros((B + 8,), dtype=torch.int32, device=cuda)
    lv[n0:n0 + B].copy_(torch.from_numpy(lens))
    tl = lv[n0:n0 + B]
    assert pts.is_contiguous() and pts.data_ptr() % 16 == (12 * n0) % 16 and tl.data_ptr() % 16 == 4 * n0
    scan = torch.zeros((N, 4), dtype=torch.float32, device=cuda)
    scan[:, :3].copy_(torch.from_numpy(P))
    want_nb = on.port_batch_neighbors(P, P, lens, lens, r)
    want_p, want_b = on.port_batch_subsampling(P, lens, dl)
    for points in (pts, scan[:, :3]):
        got = ops.batch_ordered_neighbors(points, points, tl, tl, r)
        assert np.array_equal(got.cpu().numpy(), want_nb)
        sp, sb = ops.batch_grid_subsampling(points, tl, dl)
        assert np.array_equal(sb.cpu().numpy(), want_b)
        assert np.array_equal(sp.cpu().numpy().view(np.uint32), want_p.view(np.uint32))
        grid = ops.NeighborGrid(points, tl, r)
        # (the order inside a cell is whatever the scatter's atomics made it: a permutation is all that is promised)
        assert np.array_equal(np.sort(grid.order().cpu().numpy()), np.arange(N))
        counts, mx = grid.count(points, tl)
        assert np.array_equal(counts.cpu().numpy(), (want_nb < N).sum(1))
        assert int(mx.item()) == want_nb.shape[1]
        assert np.array_equal(grid.fill(points, tl, want_nb.shape[1], N).cpu().numpy(), want_nb)
    feats = rng.normal(size=(N, 5)).astype(np.float32)
    classes = rng.integers(0, 4, (N, 1)).astype(np.int32)
    plain = ops._subsample(t(P, cuda), t(lens, cuda), dl, t(feats, cuda), t(classes, cuda))
    moved = ops._subsample(pts, tl, dl, shifted(feats, cuda, n0), shifted(classes, cuda, 4 - n0))
    for u, v in zip(plain, moved):
        assert torch.equal(u, v)


# ---------------------------------------------------------------------------------------------------------------------
#  keypoints, registration
# ---------------------------------------------------------------------------------------------------------------------

@fresh_process
def test_select_keypoints_layouts(cuda):
    from d3feat_b200.keypoints import select_keypoints
    rng = np.random.default_rng(5)
    lens = np.array([300, 1, 40, 0, 500], np.int32)
    N, k, D = int(lens.sum()), 64, 32
    a = dict(scores=rng.normal(size=N).astype(np.float32), lengths=lens,
             points=rng.normal(size=(N, 3)).astype(np.float32), descriptors=rng.normal(size=(N, D)).astype(np.float32))
    a["scores"][::7] = a["scores"][3]                     # ties
    start = np.concatenate([[0], np.cumsum(lens)])
    want = np.concatenate([np.argsort(a["scores"][start[b]:start[b + 1]], kind="stable") + start[b] for b in range(5)])
    run = lambda T: select_keypoints(T["scores"], T["lengths"], k, points=T["points"], descriptors=T["descriptors"])
    plain = {key: t(v, cuda) for key, v in a.items()}
    assert np.array_equal(select_keypoints(plain["scores"], plain["lengths"]).cpu().numpy(), want)
    base = run(plain)
    for b in range(5):
        n = min(k, int(lens[b]))
        assert np.array_equal(base.index[b, :n].cpu().numpy(), want[start[b]:start[b + 1]][-n:] if n else want[:0])
    variants = [dict(plain, **{key: shifted(a[key], cuda, 1 + i % 3)}) for i, key in enumerate(a)]
    variants.append({key: shifted(v, cuda, 3 - i % 3) for i, (key, v) in enumerate(a.items())})
    variants.append(dict(plain, points=strided(a["points"], cuda, "cols0"),
                         descriptors=strided(a["descriptors"], cuda, "t"), scores=plain["scores"][:, None]))
    for T in variants:
        assert np.array_equal(select_keypoints(T["scores"], T["lengths"]).cpu().numpy(), want)
        for u, v in zip(run(T), base):
            assert torch.equal(u, v)


@fresh_process
def test_register_pairs_abi_on_shifted_arguments(cuda):
    """d3f_register_pairs with every pointer argument in turn 4, 8 or 12 bytes past a 16-byte boundary -- the
    correspondences of one pair are a slice of a longer match buffer -- bit for bit against oracle/register_np.py."""
    from d3feat_b200 import _lib
    from oracle import register_np
    from test_gpu_registration import FIELDS, mismatches, rows, scene
    rng = np.random.default_rng(11)
    B, k, L, P = 3, 60, 200, 3
    points, _ = scene(rng, B, k)
    a = dict(points=points, count=np.array([k, k - 7, k], np.int32),
             corr=np.stack([rows(rng, L, k - 7, k - 7, out) for out in (0.2, 0.6, 0.9)]),
             n_corr=np.array([L, L - 3, 150], np.int32), pairs=np.array([(0, 1), (1, 2), (2, 0)], np.int32))
    o = dict(distance=0.05, ransac_n=3, edge_ratio=0.9, max_iterations=2000, max_validation=200, seed=5)
    want = register_np.register(a["points"], a["count"], a["corr"], a["n_corr"], a["pairs"], **o)
    lib = _lib.lib()
    ws = _lib.workspace(lib.d3f_register_pairs_workspace_bytes(L, P, 2000, 200), cuda)
    plain = {key: t(v, cuda) for key, v in a.items()}
    variants = [plain] + [dict(plain, **{key: shifted(a[key], cuda, off)}) for key in a for off in (1, 2, 3)]
    variants.append({key: shifted(v, cuda, 1 + i % 3) for i, (key, v) in enumerate(a.items())})
    for T in variants:
        pose = torch.full((P, 4, 4), 7.0, dtype=torch.float64, device=cuda)
        ints = [torch.full((P,), 7, dtype=torch.int32, device=cuda) for _ in range(3)]
        _lib.check(lib.d3f_register_pairs(_lib.ptr(T["points"]), _lib.ptr(T["count"]), B, k, _lib.ptr(T["corr"]),
                                          _lib.ptr(T["n_corr"]), L, _lib.ptr(T["pairs"]), P, 3, 2000, 200, 0.05, 0.9, 5,
                                          _lib.ptr(pose), *[_lib.ptr(x) for x in ints], _lib.ptr(ws), ws.numel(),
                                          _lib.stream()), "d3f_register_pairs")
        got = dict(zip(FIELDS, [pose.cpu().numpy()] + [x.cpu().numpy() for x in ints]))
        assert mismatches(got, want) == []
    assert (want["n_inliers"] > 3).any()


# ---------------------------------------------------------------------------------------------------------------------
#  the whole network
# ---------------------------------------------------------------------------------------------------------------------

@fresh_process
def test_network_on_a_scan_column_slice(cuda):
    """KPFCNN on scan[:, :3] of an [N, 4] device tensor with the lengths taken at an odd offset of a longer vector:
    every returned tensor equals the same call on plain copies."""
    from d3feat_b200 import synth
    from d3feat_b200.encoder import KPFCNN
    cfg = synth.Config()
    clouds = [synth.room_fragment(50, 4000), synth.room_fragment(51, 3000)]
    P = np.concatenate(clouds, 0)
    L = np.array([4000, 3000], np.int32)
    enc = KPFCNN(cfg, synth.make_params(cfg, 0), [35, 33, 34, 36, 30], device=cuda)
    base = enc(t(P, cuda), t(L, cuda), decoder=True)
    scan = torch.zeros((P.shape[0], 4), dtype=torch.float32, device=cuda)
    scan[:, :3].copy_(torch.from_numpy(P))
    lv = torch.zeros((9,), dtype=torch.int32, device=cuda)
    lv[3:5].copy_(torch.from_numpy(L))
    out = enc(scan[:, :3], lv[3:5], features=torch.ones(1, 1, device=cuda).expand(P.shape[0], 1), decoder=True)
    assert torch.equal(out["descriptors"], base["descriptors"]) and torch.equal(out["scores"], base["scores"])
    for u, v in zip(out["F"], base["F"]):
        assert torch.equal(u, v)
    for key, vals in base["inputs"].items():
        if key == "orders":                       # a scheduling hint; its order inside a cell is not deterministic
            continue
        for u, v in zip(out["inputs"][key], vals) if isinstance(vals, list) else [(out["inputs"][key], vals)]:
            assert torch.equal(u, v), key


# ---------------------------------------------------------------------------------------------------------------------

PREDICATES = ["tc_gemm_supported (A)", "tc epilogue vec (residual)", "tc epilogue vec (C)", "gemm_f32 a_vec",
              "gemm_f32 b_vec", "pair: 16-byte aligned x1 / x2", "kpconv al16 (feat)", "prep_supports vec",
              "fused eligibility (feat)", "pool v4 (x)", "pool v4 (out)"]


@fresh_process
def test_every_alignment_predicate_was_false_once(cuda, monkeypatch):
    """Every 16-byte alignment predicate of the library was false in some case above, and the case named the kernel or
    arm that ran instead (cases that did not run in this session, e.g. under -k, are run here)."""
    if "tc_gemm_supported (A)" not in FLIPPED or "tc epilogue vec (residual)" not in FLIPPED:
        test_unary_convolution_layouts(cuda, *UNARY[0])
    if "tc epilogue vec (C)" not in FLIPPED:
        test_unary_abi_shifted_output(cuda, 3000, 64, 32, True)
    if "pair: 16-byte aligned x1 / x2" not in FLIPPED:
        test_unary_pair_layouts(cuda, 5000, 32, 64, 128)
    if "kpconv al16 (feat)" not in FLIPPED:
        with monkeypatch.context() as m:
            test_kpconv_layouts(cuda, m, KP_LAYOUT[0])
    if "fused eligibility (feat)" not in FLIPPED:
        with monkeypatch.context() as m:
            test_kpconv_layouts(cuda, m, next(c for c in KP_LAYOUT if c["env"].get("D3F_FUSED_KPCONV")))
    if "pool v4 (x)" not in FLIPPED or "pool v4 (out)" not in FLIPPED:
        test_pool_layouts(cuda, 64)
    missing = [p for p in PREDICATES if p not in FLIPPED]
    assert not missing, "alignment predicates never false: %s" % missing
    for p in PREDICATES:
        print("PREDICATE %-34s false -> %s" % (p, FLIPPED[p]))
