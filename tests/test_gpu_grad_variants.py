"""GPU: every kernel the KPConv and unary gradients can reach, pinned by name, each case element by element against the
float64 restatement (tests/_kpconv_grad_oracle.py) at TOL = 1e-5 * mag.

The gradients reuse the forward's dispatch with arguments the forward never passes (kpconv_grad.cu):
  * dL/dW recomputes wf through launch_stage1 without a neighbour count, so the layer's Cin picks its stage 1;
  * dL/df is a forward KPConv over the transposed neighbourhood (Ns queries, Nq supports, width Hr, kernel points -Kp,
    weights W^T, features G = dout / nn, no normalisation), so the layer's Cout picks the stage 1 of its feature
    gradient (kpconv_cin1_kernel for Cout = 1, kpconv_fused32_kernel under D3F_FUSED_KPCONV=1) and its Cin picks the
    contraction (tc_gemm_kernel<32|64|128>, split-K, or gemm_f32 when K * Cout % 4 != 0 or without tensor cores).
Each table case runs the two gradients separately under torch.profiler, so every kernel name is asserted for the
gradient that launched it, then checks that the combined call gives the same bits. The index edges (padding, a hub
support, duplicates, unreached supports, shadow rows, a single point) run on the fast, mma, generic, anyk and cin1
families. The unary backward is pinned the same way: dx through the forward GEMMs, dW through wgrad_partial_kernel at the
edges of its 2048-row blocks.

Switches read once per process run in child processes: D3F_KPCONV_CHUNK (both gradients over >= 3 chunks, with device
row counts inside a chunk and on a chunk boundary) and D3F_S1_PARED=0 (kpconv_stage1_mma_kernel<NT, false, true>,
forward and backward).

All cases run in one child pytest session of this file: in a long session torch.profiler can stop delivering kernel
records (see tests/test_gpu_tensor_layouts.py), and which kernel ran is the point here.
"""
import functools
import json
import os
import subprocess
import sys
import tempfile
import xml.etree.ElementTree as ET
import zlib

import numpy as np
import pytest
import torch

import _kpconv_grad_oracle as og
from _oracle import TOL, assert_close, kpconv_ref
from test_gpu_kernel_variants import ANYK, F32, FAST4, FAST8, GENERIC, SPLITK, STAGED4, STAGED8, launched, mma, t
from test_gpu_kpconv_grad import check, make_case

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CHILD = "D3F_GRAD_VARIANTS_CHILD"    # set in the child session, where the cases really run
_child = None
SEEN = set()                         # kernel names launched by the cases of this module (in the child session)


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
                               timeout=2400)
            print("\n".join(l for l in r.stdout.splitlines() if l.lstrip(".").startswith(("RATIO", "CHUNKS", "PARED"))))
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


def names_of(fn):
    out, names = launched(fn)
    SEEN.update(names)
    return out, names


def assert_ran(names, expect, what):
    for e in expect:
        assert any(e in n for n in names), "%s: expected kernel %s; launched: %s" % (what, e, sorted(names))


def assert_absent(names, kernels, what):
    for e in kernels:
        assert not any(e in n for n in names), "%s: kernel %s must not run; launched: %s" % (what, e, sorted(names))


TC = "tc_gemm_kernel<%d>"
WG = "wgrad_partial_kernel<%d>"
V2_21, V2_22 = "kpconv_stage1_v2_kernel<2,1,false>", "kpconv_stage1_v2_kernel<2,2,false>"
CIN1_T, CIN1_F, CIN1 = "kpconv_cin1_kernel<true>", "kpconv_cin1_kernel<false>", "kpconv_cin1_kernel"
FUSED = "kpconv_fused32_kernel"
GEMMS = ("tc_gemm_kernel", "gemm_f32_kernel")
STAGED = {"D3F_S1_STAGED": "1"}


def wgrad(Cout):
    return WG % (32 if Cout <= 32 else 64)


# ---------------------------------------------------------------------------------------------------------------------
#  KPConv backward table
# ---------------------------------------------------------------------------------------------------------------------

def gv(id, Cin, Cout, dw, df, Nq=600, H=32, K=15, infl="linear", mode="sum", tc=True, env=None, misalign=0,
       absent=(), extent=None):
    """One case: dw = the stage 1 of the weight gradient's recompute, df = the stage 1 (or whole-operator kernel) and
    contraction of the transposed forward, absent = kernels the feature gradient must not launch. Nq = Ns."""
    return dict(id=id, Cin=Cin, Cout=Cout, dw=list(dw) + [wgrad(Cout)], df=list(df), Nq=Nq, H=H, K=K, infl=infl,
                mode=mode, tc=tc, env=env or {}, misalign=misalign, absent=list(absent),
                extent=extent or round(0.9 * Nq ** (-1 / 3), 4))   # ~ H neighbours within 2.5 extent


M4, M8, M16 = mma(4, False, False), mma(8, False, False), mma(16, False, False)
CASES = [
    gv("fast4_32x32", 32, 32, [FAST4], [FAST4, TC % 32]),
    gv("fast8_64x64", 64, 64, [FAST8], [FAST8, TC % 64]),
    gv("fast8_128x128", 128, 128, [FAST8], [FAST8, TC % 128], Nq=400),
    gv("fast8_512x64", 512, 64, [FAST8], [FAST8, TC % 128], Nq=250, H=24),
    gv("mma4_32x48_gaussian", 32, 48, [M4], [GENERIC, TC % 32], infl="gaussian"),
    gv("mma4_32x32_closest", 32, 32, [M4], [M4, TC % 32], mode="closest"),
    gv("mma8_64x64_constant", 64, 64, [M8], [M8, TC % 64], infl="constant"),
    gv("mma16_128x64_closest", 128, 64, [M16], [M8, TC % 128], mode="closest", Nq=400),
    gv("mma8_64x128_gaussian", 64, 128, [M8], [M16, TC % 64], infl="gaussian", Nq=400),
    gv("v2_192x96", 192, 96, [V2_21], [V2_22, TC % 128], Nq=300),
    gv("v2_96x192", 96, 192, [V2_22], [V2_21, TC % 128], Nq=300),
    gv("generic_5x48", 5, 48, [GENERIC], [GENERIC, TC % 32]),
    gv("generic_48x40", 48, 40, [GENERIC], [GENERIC, TC % 64]),
    gv("misaligned4_32x32", 32, 32, [GENERIC], [FAST4, TC % 32], misalign=1),
    gv("misaligned8_32x32", 32, 32, [GENERIC], [FAST4, TC % 32], misalign=2),
    gv("misaligned12_32x32", 32, 32, [GENERIC], [FAST4, TC % 32], misalign=3),
    gv("anyk_k1_32x32", 32, 32, [ANYK], [ANYK, TC % 32], K=1),
    gv("anyk_k7_1x20", 1, 20, [ANYK], [ANYK, TC % 32], K=7),
    gv("anyk_k7_20x1", 20, 1, [ANYK], [ANYK, F32], K=7),
    gv("anyk_k33_12x21_closest", 12, 21, [ANYK], [ANYK, F32], K=33, mode="closest"),
    gv("anyk_k64_32x32_gaussian", 32, 32, [ANYK], [ANYK, TC % 32], K=64, infl="gaussian", Nq=400),
    gv("cin1_64x1", 64, 1, [FAST8], [CIN1_T], absent=GEMMS),
    gv("cin1_64x1_gaussian_closest", 64, 1, [M8], [CIN1_F], infl="gaussian", mode="closest", absent=GEMMS),
    gv("cin1_816x1", 816, 1, [GENERIC], [CIN1_T], Nq=300, H=24, absent=GEMMS),
    gv("cin1_816x1_gaussian_closest", 816, 1, [GENERIC], [CIN1_F], Nq=300, H=24, infl="gaussian", mode="closest",
       absent=GEMMS),
    gv("wide_817x1", 817, 1, [GENERIC], [GENERIC, F32], Nq=300, H=24, absent=[CIN1]),
    gv("wide_817x1_gaussian_closest", 817, 1, [GENERIC], [GENERIC, F32], Nq=300, H=24, infl="gaussian",
       mode="closest", absent=[CIN1]),
    gv("wide_1024x1", 1024, 1, [FAST8], [GENERIC, F32], Nq=300, H=24, absent=[CIN1]),
    gv("first_layer_1x64", 1, 64, [GENERIC], [FAST8, TC % 32]),
    gv("splitk_64x64_ns300", 64, 64, [FAST8], [FAST8, TC % 64, SPLITK], Nq=300),
    gv("fused32_4000", 32, 32, [FAST4], [FUSED], Nq=4000, H=35, env={"D3F_FUSED_KPCONV": "1"}, absent=GEMMS),
    gv("staged4_32x32", 32, 32, [STAGED4], [STAGED4, TC % 32], env=STAGED),
    gv("staged8_64x64", 64, 64, [STAGED8], [STAGED8, TC % 64], env=STAGED),
    gv("staged_256x32", 256, 32, [STAGED8], [STAGED4, TC % 128], Nq=300, env=STAGED),
    gv("f32_32x32", 32, 32, [FAST4], [FAST4, F32], tc=False, absent=["tc_gemm_kernel"]),
    gv("f32_64x64", 64, 64, [FAST8], [FAST8, F32], tc=False, absent=["tc_gemm_kernel"]),
    gv("f32_128x128", 128, 128, [FAST8], [FAST8, F32], Nq=400, tc=False, absent=["tc_gemm_kernel"]),
    gv("f32_512x64", 512, 64, [FAST8], [FAST8, F32], Nq=250, H=24, tc=False, absent=["tc_gemm_kernel"]),
    gv("f32_5x48", 5, 48, [GENERIC], [GENERIC, F32], tc=False, absent=["tc_gemm_kernel"]),
    gv("f32_1x64", 1, 64, [GENERIC], [FAST8, F32], tc=False, absent=["tc_gemm_kernel"]),
]


def case_inputs(c):
    rng = np.random.default_rng(zlib.crc32(c["id"].encode()))
    q, s, idx, f, Kp, W, dout = make_case(rng, c["Nq"], c["Nq"], c["H"], c["Cin"], c["Cout"], K=c["K"],
                                          extent=c["extent"], unreached=3)
    f[::5] = -np.abs(f[::5])              # supports that do not count towards nn
    return q, s, idx, f, Kp, W, dout


def feature_tensor(f, dev, off):
    """f on the device, `off` floats past a 16-byte boundary."""
    if not off:
        return t(f, dev)
    buf = torch.empty(f.size + 4, dtype=torch.float32, device=dev)
    view = buf[off:off + f.size].view(f.shape)
    view.copy_(torch.from_numpy(f))
    assert view.data_ptr() % 16 == 4 * off
    return view


def run_case(c, dev, monkeypatch):
    """(df, dW, names of the df-only call, names of the dW-only call, inputs)."""
    from d3feat_b200 import convolution_ops as co
    for k, v in c["env"].items():
        monkeypatch.setenv(k, v)
    monkeypatch.setattr(co, "USE_TENSOR_CORES", c["tc"])
    q, s, idx, f, Kp, W, dout = inputs = case_inputs(c)
    args = [t(q, dev), t(s, dev), t(idx, dev), feature_tensor(f, dev, c["misalign"]), t(Kp, dev), t(W, dev),
            c["extent"], c["infl"], c["mode"], t(dout, dev)]
    (df, none), n_df = names_of(lambda: co.kpconv_backward(*args, weights_grad=False))
    assert none is None
    (none, dW), n_dw = names_of(lambda: co.kpconv_backward(*args, features_grad=False))
    assert none is None
    both = co.kpconv_backward(*args)
    assert torch.equal(both[0], df) and torch.equal(both[1], dW), "the combined call differs from the separate ones"
    return df.cpu().numpy(), dW.cpu().numpy(), n_df, n_dw, inputs


@pytest.mark.parametrize("c", CASES, ids=[c["id"] for c in CASES])
@fresh_process
def test_kpconv_backward_variant(cuda, monkeypatch, c):
    df, dW, n_df, n_dw, (q, s, idx, f, Kp, W, dout) = run_case(c, cuda, monkeypatch)
    assert_ran(n_dw, c["dw"], c["id"] + " dW")
    assert_ran(n_df, c["df"], c["id"] + " df")
    assert_absent(n_df, c["absent"], c["id"] + " df")
    assert np.all(df[-3:] == 0), "supports no query reaches must get an exact zero"
    check("grad variant %s" % c["id"], q, s, idx, f, Kp, W, dout, c["extent"], c["infl"], c["mode"], df, dW)


# ---- index edges, on each family ------------------------------------------------------------------------------------

FAMILIES = {
    "fast": dict(Cin=32, Cout=32, kernels=[FAST4]),
    "mma": dict(Cin=32, Cout=32, infl="gaussian", kernels=[M4]),
    "generic": dict(Cin=5, Cout=40, kernels=[GENERIC]),
    "anyk": dict(Cin=12, Cout=20, K=7, kernels=[ANYK]),
    "cin1": dict(Cin=64, Cout=1, kernels=[FAST8, CIN1_T]),
}
EDGES = ["padding", "hub", "duplicates", "unreached", "shadow_rows", "all_shadow", "tiny"]


def edge_case(fam, edge):
    """(q, s, idx, f, Kp, W, dout, extent, rows of df that must be exactly 0)."""
    F = FAMILIES[fam]
    K = F.get("K", 15)
    rng = np.random.default_rng(zlib.crc32((fam + edge).encode()))
    N, H, extent, unreached = 500, 24, 0.11, 0
    if edge == "hub":
        N, extent = 1000, 0.6            # 2 * extent spans the cube: every query has a linear weight on the hub
    if edge == "unreached":
        unreached = 40
    if edge == "tiny":
        N, H = 1, 1
    q, s, idx, f, Kp, W, dout = make_case(rng, N, N, H, F["Cin"], F["Cout"], K=K, extent=extent, unreached=unreached)
    f[::5] = -np.abs(f[::5])
    zero = np.zeros(N, bool)
    zero[N - unreached:] = True
    if edge == "padding":
        idx[::3, -2] = -1                                  # -1 padding of the non-batch op
        idx[1::4, -3] = N + 1 + np.arange(len(idx[1::4])) % 5   # above the shadow index: treated as the shadow
        idx[2::5, 1] = -1
    elif edge == "hub":
        s[0] = q[0] = 0.5
        idx[:, 0] = 0                                      # support 0 named by every query: Hr ~ Nq
    elif edge == "duplicates":
        idx[:, -1] = idx[:, 0]                             # every row names its first support twice,
        idx[::2, -2] = idx[::2, 0]                         # every second row three times
    elif edge == "shadow_rows":
        idx[::3] = N                                       # rows whose every neighbour is the shadow,
        idx[1::6] = -1                                     # or -1
    elif edge == "all_shadow":
        idx[:] = N                                         # Hr = 0
        zero[:] = True
    elif edge == "tiny":
        idx[:] = 0
    reached = np.zeros(N + 1, bool)
    reached[np.where((idx < 0) | (idx > N), N, idx)] = True
    zero |= ~reached[:N]
    return q, s, idx, f, Kp, W, dout, extent, zero


@pytest.mark.parametrize("edge", EDGES)
@pytest.mark.parametrize("fam", sorted(FAMILIES))
@fresh_process
def test_kpconv_backward_index_edges(cuda, fam, edge):
    from d3feat_b200 import convolution_ops as co
    F = FAMILIES[fam]
    infl = F.get("infl", "linear")
    q, s, idx, f, Kp, W, dout, extent, zero = edge_case(fam, edge)
    args = [t(a, cuda) for a in (q, s, idx, f, Kp, W)] + [extent, infl, "sum", t(dout, cuda)]
    (df, dW), names = names_of(lambda: co.kpconv_backward(*args))
    df, dW = df.cpu().numpy(), dW.cpu().numpy()
    assert_ran(names, F["kernels"] if edge != "all_shadow" else F["kernels"][:1], "%s %s" % (fam, edge))
    assert np.all(df[zero] == 0), "supports no query reaches must get an exact zero"
    if edge == "all_shadow":
        assert np.all(df == 0) and np.all(dW == 0)
    check("grad edge %s %s" % (fam, edge), q, s, idx, f, Kp, W, dout, extent, infl, "sum", df, dW)


# ---------------------------------------------------------------------------------------------------------------------
#  unary backward
# ---------------------------------------------------------------------------------------------------------------------

def unary_inputs(N, Cin, Cout):
    rng = np.random.default_rng(N * 7 + Cin * 3 + Cout)
    return (rng.normal(size=(N, Cin)).astype(np.float32), rng.normal(size=(Cin, Cout)).astype(np.float32),
            rng.normal(size=(N, Cout)).astype(np.float32))


def unary_check(what, x, w, g, dx, dw):
    ref, mag, alt = og.unary_features_grad(x, w, g)
    assert_close(dx, ref, mag, what=what + " dx", alt=alt)
    ref, mag, alt = og.unary_weights_grad(x, w, g)
    assert_close(dw, ref, mag, what=what + " dW", alt=alt)


def unary_named(dev, x, w, g, rows=None):
    """(dx, dW, names of the dx-only call, names of the dW-only call) for device tensors x, w, g."""
    from d3feat_b200 import convolution_ops as co
    (dx, _), n_dx = names_of(lambda: co.unary_backward(x, w, g, rows=rows, weights_grad=False))
    (_, dw), n_dw = names_of(lambda: co.unary_backward(x, w, g, rows=rows, features_grad=False))
    return dx.cpu().numpy(), dw.cpu().numpy(), n_dx, n_dw


UNARY_DX = [(3000, 32, 64, TC % 32), (3000, 64, 32, TC % 64), (3000, 256, 64, TC % 128)]


@pytest.mark.parametrize("N,Cin,Cout,kernel", UNARY_DX)
@fresh_process
def test_unary_dx_tensor_cores(cuda, N, Cin, Cout, kernel):
    x, w, g = unary_inputs(N, Cin, Cout)
    dx, dw, n_dx, n_dw = unary_named(cuda, t(x, cuda), t(w, cuda), t(g, cuda))
    assert_ran(n_dx, [kernel], "unary dx")
    assert_absent(n_dx, ["gemm_f32_kernel"], "unary dx")
    assert_ran(n_dw, [wgrad(Cout)], "unary dW")
    unary_check("unary %dx%d->%d" % (N, Cin, Cout), x, w, g, dx, dw)


@pytest.mark.parametrize("why", ["cout33", "grad_out_misaligned", "tensor_cores_off"])
@fresh_process
def test_unary_dx_cuda_cores(cuda, monkeypatch, why):
    from d3feat_b200 import convolution_ops as co
    N, Cin, Cout = 3000, 64, 33 if why == "cout33" else 32
    x, w, g = unary_inputs(N, Cin, Cout)
    gt = feature_tensor(g, cuda, 1) if why == "grad_out_misaligned" else t(g, cuda)
    monkeypatch.setattr(co, "USE_TENSOR_CORES", why != "tensor_cores_off")
    dx, dw, n_dx, n_dw = unary_named(cuda, t(x, cuda), t(w, cuda), gt)
    assert_ran(n_dx, [F32], "unary dx " + why)
    assert_absent(n_dx, ["tc_gemm_kernel"], "unary dx " + why)
    unary_check("unary %s" % why, x, w, g, dx, dw)


@pytest.mark.parametrize("Cout", [32, 64])
@pytest.mark.parametrize("N", [2047, 2048, 2049, 4097])
@fresh_process
def test_unary_dw_row_blocks(cuda, N, Cout):
    x, w, g = unary_inputs(N, 48, Cout)
    dx, dw, n_dx, n_dw = unary_named(cuda, t(x, cuda), t(w, cuda), t(g, cuda))
    assert_ran(n_dw, [wgrad(Cout), "wgrad_reduce_kernel"], "unary dW")
    unary_check("unary blocks N=%d Cout=%d" % (N, Cout), x, w, g, dx, dw)


@pytest.mark.parametrize("n", [2048, 2049])
@fresh_process
def test_unary_dw_device_row_count(cuda, n):
    """A capacity of 5000 rows with the count at the edge of the first block: NaN past it is never read."""
    x, w, g = unary_inputs(5000, 48, 64)
    x[n:], g[n:] = np.nan, np.nan
    rows = torch.tensor([n], dtype=torch.int32, device=cuda)
    dx, dw, n_dx, n_dw = unary_named(cuda, t(x, cuda), t(w, cuda), t(g, cuda), rows=rows)
    assert_ran(n_dw, [WG % 64], "unary dW rows")
    assert np.all(dx[n:] == 0) and np.isfinite(dw).all()
    unary_check("unary rows=%d" % n, x[:n], w, g[:n], dx[:n], dw)


@fresh_process
def test_unary_layouts_give_the_same_bits(cuda):
    """No predicate depends on where features start, or on how grad_out is laid out (it is made contiguous): a
    misaligned x, a strided grad_out and the expanded grad_out of out.sum().backward() give the plain call's bits."""
    from d3feat_b200 import convolution_ops as co
    x, w, g = unary_inputs(3000, 64, 32)
    xt, wt, gt = t(x, cuda), t(w, cuda), t(g, cuda)
    base = co.unary_backward(xt, wt, gt)
    for off in (1, 2, 3):
        other = co.unary_backward(feature_tensor(x, cuda, off), wt, gt)
        assert all(torch.equal(a, b) for a, b in zip(base, other)), "features %d B off" % (4 * off)
    wide = torch.zeros((3000, 64), device=cuda)
    wide[:, ::2] = gt
    for gs in (wide[:, ::2], gt.t().contiguous().t()):
        assert not gs.is_contiguous()
        other = co.unary_backward(xt, wt, gs)
        assert all(torch.equal(a, b) for a, b in zip(base, other)), "strided grad_out"
    xr, wr = xt.clone().requires_grad_(True), wt.clone().requires_grad_(True)
    co.unary_convolution(xr, wr).sum().backward()
    ones = co.unary_backward(xt, wt, torch.ones((3000, 32), device=cuda))
    assert torch.equal(xr.grad, ones[0]) and torch.equal(wr.grad, ones[1])
    unary_check("unary sum().backward()", x, w, np.ones((3000, 32), np.float32), xr.grad.cpu().numpy(),
                wr.grad.cpu().numpy())


# ---------------------------------------------------------------------------------------------------------------------
#  switches read once per process (child processes)
# ---------------------------------------------------------------------------------------------------------------------

DRIVER_COMMON = r"""
import json, sys
import numpy as np, torch
sys.path.insert(0, sys.argv[1])
from torch.profiler import ProfilerActivity, profile
from d3feat_b200 import convolution_ops as co
d = sys.argv[2]
cases = json.load(open(d + "/cases.json"))
dev = torch.device("cuda", 0)
def t(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)
def counted(fn):
    # (fn(), {kernel name: launches}); an empty CUPTI buffer is retried, the ops are deterministic
    for attempt in range(5):
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            out = fn()
            torch.cuda.synchronize()
        n = {}
        for e in prof.events():
            if e.device_type == torch.autograd.DeviceType.CUDA and not e.name.startswith(("Memcpy", "Memset")):
                k = e.name.replace(" ", "")
                n[k] = n.get(k, 0) + 1
        if n:
            return out, n
    raise AssertionError("the profiler recorded no CUDA kernel at all")
report = {}
"""

CHUNK_DRIVER = DRIVER_COMMON + r"""
for c in cases:
    z = np.load(d + "/in_%s.npz" % c["id"])
    co.USE_TENSOR_CORES = c["tc"]
    rows = {k: None if c[k] is None else torch.tensor([c[k]], dtype=torch.int32, device=dev) for k in ("rows_q", "rows_s")}
    args = [t(z[k]) for k in ("q", "s", "idx", "f", "Kp", "W")] + [c["extent"], "linear", "sum", t(z["dout"])]
    (df, _), n_df = counted(lambda: co.kpconv_backward(*args, weights_grad=False, **rows))
    (_, dW), n_dw = counted(lambda: co.kpconv_backward(*args, features_grad=False, **rows))
    both = co.kpconv_backward(*args, **rows)
    assert torch.equal(both[0], df) and torch.equal(both[1], dW), c["id"]
    np.save(d + "/df_%s.npy" % c["id"], df.cpu().numpy())
    np.save(d + "/dW_%s.npy" % c["id"], dW.cpu().numpy())
    report[c["id"]] = dict(df=n_df, dw=n_dw)
json.dump(report, open(d + "/report.json", "w"))
"""

CHUNK_CASES = [
    dict(id="fast_32x32", Cin=32, Cout=32, s1=FAST4, gemm=TC % 32, tc=True, rows=None),
    dict(id="fast_64x64", Cin=64, Cout=64, s1=FAST8, gemm=TC % 64, tc=True, rows=None),
    dict(id="generic_5x48", Cin=5, Cout=48, s1=GENERIC, gemm=TC % 32, tc=True, rows=None),
    dict(id="f32_32x32", Cin=32, Cout=32, s1=FAST4, gemm=F32, tc=False, rows=None),
    dict(id="rows_mid_64x64", Cin=64, Cout=64, s1=FAST8, gemm=TC % 64, tc=True, rows="mid"),
    dict(id="rows_boundary_64x64", Cin=64, Cout=64, s1=FAST8, gemm=TC % 64, tc=True, rows="boundary"),
]


def launches(counts, kernel):
    return sum(v for k, v in counts.items() if kernel in k)


@pytest.mark.parametrize("chunk", [128, 1024])
@fresh_process
def test_kpconv_backward_multi_chunk(cuda, chunk):
    """D3F_KPCONV_CHUNK = 128 / 1024 queries: Nq = Ns span 3 chunks and a ragged fourth, so the weight gradient walks
    its chunk loop (the per-chunk offset into the partials, the device row count taken from the chunk's first row) and
    the feature gradient's transposed forward runs its chunk pipeline on the auxiliary stream, followed by the weight
    gradient in the same workspace region. Device row counts end inside a middle chunk, or exactly on a chunk boundary:
    rows below them are compared with float64, rows of dL/df past rows_s are exactly 0."""
    n = 3 * chunk + chunk // 2 - 3
    rng = np.random.default_rng(chunk + 5)
    extent = round(0.9 * n ** (-1 / 3), 4)
    with tempfile.TemporaryDirectory() as d:
        cases, data = [], {}
        for c in CHUNK_CASES:
            c = dict(c, extent=extent, rows_q=None, rows_s=None)
            nq = ns = n
            if c["rows"] == "mid":
                nq, ns = chunk + 37, 2 * chunk + 11
            elif c["rows"] == "boundary":
                nq = ns = 2 * chunk
            q, s, idx, f, Kp, W, dout = make_case(rng, nq, ns, 36, c["Cin"], c["Cout"], extent=extent, unreached=3)
            f[::5] = -np.abs(f[::5])
            ref_in = (q, s, idx, f, Kp, W, dout)
            if c["rows"] is not None:
                # capacity-sized buffers: NaN past the counts, indices past rows_q anywhere in [0, n]; inside, ns is the
                # shadow and indices above it are treated as the shadow too
                c["rows_q"], c["rows_s"] = nq, ns
                cap = lambda a, m: np.concatenate([a, np.full((n - m,) + a.shape[1:], np.nan, np.float32)])
                q, dout, s, f = cap(q, nq), cap(dout, nq), cap(s, ns), cap(f, ns)
                idx = np.concatenate([idx, rng.integers(0, n + 1, (n - nq, idx.shape[1])).astype(np.int32)])
                idx[:nq:5, 3] = ns + 7
                ref_in = (ref_in[0], ref_in[1], np.where(idx[:nq] > ns, ns, idx[:nq])) + ref_in[3:]
            np.savez(os.path.join(d, "in_%s.npz" % c["id"]), q=q, s=s, idx=idx, f=f, Kp=Kp, W=W, dout=dout)
            cases.append(c)
            data[c["id"]] = ref_in
        with open(os.path.join(d, "cases.json"), "w") as fh:
            json.dump(cases, fh)
        env = dict(os.environ, D3F_KPCONV_CHUNK=str(chunk))
        r = subprocess.run([sys.executable, "-c", CHUNK_DRIVER, ROOT, d], env=env, capture_output=True, text=True,
                           timeout=900)
        assert r.returncode == 0, r.stderr[-4000:]
        report = json.load(open(os.path.join(d, "report.json")))
        chunks = -(-n // chunk)
        assert chunks >= 4 and n % chunk != 0
        for c in cases:
            rep, what = report[c["id"]], "chunk %d %s" % (chunk, c["id"])
            # every case's Cin and Cout pick the same stage 1, so s1 names both gradients' kernel
            counts = dict(dw_stage1=launches(rep["dw"], c["s1"]), wgrad=launches(rep["dw"], "wgrad_partial_kernel<"),
                          df_stage1=launches(rep["df"], c["s1"]), df_gemm=launches(rep["df"], c["gemm"]))
            print("CHUNKS %-40s %s" % (what, counts))
            assert all(v == chunks for v in counts.values()), (what, counts, chunks)
            q, s, idx, f, Kp, W, dout = data[c["id"]]
            df = np.load(os.path.join(d, "df_%s.npy" % c["id"]))
            dW = np.load(os.path.join(d, "dW_%s.npy" % c["id"]))
            ns = len(s)
            assert np.all(df[ns:] == 0) and np.all(df[ns - 3:ns] == 0)
            check(what, q, s, idx, f, Kp, W, dout, extent, "linear", "sum", df[:ns], dW)


PARED_DRIVER = DRIVER_COMMON + r"""
for c in cases:
    z = np.load(d + "/in_%s.npz" % c["id"])
    a = [t(z[k]) for k in ("q", "s", "idx", "f", "Kp", "W")]
    co.packed_weight(a[5])
    out, n_fw = counted(lambda: co.KPConv_ops(*a, c["extent"], "linear", "sum"))
    (df, _), n_df = counted(lambda: co.kpconv_backward(*a, c["extent"], "linear", "sum", t(z["dout"]), weights_grad=False))
    (_, dW), n_dw = counted(lambda: co.kpconv_backward(*a, c["extent"], "linear", "sum", t(z["dout"]), features_grad=False))
    for k, v in (("out", out), ("df", df), ("dW", dW)):
        np.save(d + "/%s_%s.npy" % (k, c["id"]), v.cpu().numpy())
    report[c["id"]] = dict(fw=sorted(n_fw), df=sorted(n_df), dw=sorted(n_dw))
json.dump(report, open(d + "/report.json", "w"))
"""


@fresh_process
def test_unpared_mma_stage1_forward_and_backward(cuda):
    """D3F_S1_PARED=0 switches the rigid linear-sum layers from the 64-channel-pass kernels to the general mma.sync
    kernel's FAST instance, kpconv_stage1_mma_kernel<NT, false, true>: the forward, the weight gradient's recompute
    and the transposed forward of the feature gradient, for NT = 4, 8 and 16."""
    rng = np.random.default_rng(31)
    cases, data = [], {}
    with tempfile.TemporaryDirectory() as d:
        for C, N in ((32, 600), (64, 600), (128, 400)):
            c = dict(id="pared0_%dx%d" % (C, C), C=C, extent=round(0.9 * N ** (-1 / 3), 4),
                     kernel=mma(C // 8, False, True))
            z = dict(zip(("q", "s", "idx", "f", "Kp", "W", "dout"),
                         make_case(rng, N, N, 32, C, C, extent=c["extent"], unreached=3)))
            z["f"][::5] = -np.abs(z["f"][::5])
            np.savez(os.path.join(d, "in_%s.npz" % c["id"]), **z)
            cases.append(c)
            data[c["id"]] = z
        with open(os.path.join(d, "cases.json"), "w") as fh:
            json.dump(cases, fh)
        r = subprocess.run([sys.executable, "-c", PARED_DRIVER, ROOT, d], env=dict(os.environ, D3F_S1_PARED="0"),
                           capture_output=True, text=True, timeout=900)
        assert r.returncode == 0, r.stderr[-4000:]
        report = json.load(open(os.path.join(d, "report.json")))
        for c in cases:
            z, rep = data[c["id"]], report[c["id"]]
            print("PARED %-20s forward %s" % (c["id"], [n for n in rep["fw"] if "stage1" in n]))
            for part in ("fw", "df", "dw"):
                SEEN.update(rep[part])
                assert_ran(rep[part], [c["kernel"]], "%s %s" % (c["id"], part))
                assert_absent(rep[part], ["kpconv_stage1_fast_kernel"], "%s %s" % (c["id"], part))
            out, df, dW = (np.load(os.path.join(d, "%s_%s.npy" % (k, c["id"]))) for k in ("out", "df", "dW"))
            args = [z[k] for k in ("q", "s", "idx", "f", "Kp", "W")]
            ref, mag, alt = kpconv_ref(*args, c["extent"])
            assert_close(out, ref, mag, TOL, "grad pared0 %s forward" % c["id"], alt=alt)
            check("grad pared0 %s" % c["id"], *args, z["dout"], c["extent"], "linear", "sum", df, dW)


# ---------------------------------------------------------------------------------------------------------------------

@fresh_process
def test_every_backward_instance_was_launched(cuda, monkeypatch):
    """The union of kernel names the cases above launched covers every instance the table names (cases that did not
    run in this session are run here for their kernel names), and the FAST mma instances of the D3F_S1_PARED=0 child."""
    for c in CASES:
        if not all(any(e in n for n in SEEN) for e in c["dw"] + c["df"]):
            with monkeypatch.context() as m:
                run_case(c, cuda, m)
    expect = {e for c in CASES for e in c["dw"] + c["df"]} | {mma(nt, False, True) for nt in (4, 8, 16)}
    missing = sorted(e for e in expect if not any(e in n for n in SEEN))
    assert not missing, "backward instances never launched: %s (seen: %s)" % (missing, sorted(SEEN))
