"""Every KPConv stage-1 instance and every GEMM shape class, each run under torch.profiler to prove WHICH kernel
instance ran, and each checked element by element against float64 (tests/_oracle.py).

launch_stage1 (kpconv.cu) and tc_gemm / gemm_f32 pick among many template instances by channel count, alignment,
influence, mode, K and the number of rows. The table below names the instance each case must reach, so a dispatch
change that moves a case off its kernel fails here instead of silently dropping that kernel from the suite.

Not in the table: kpconv_stage1_mma_kernel<NT, false, true> (rigid linear-sum with the 64-channel-pass kernels
switched off by D3F_S1_PARED=0, which is read once per process: tests/test_gpu_grad_variants.py runs it forward and
backward in a child process), and split-K with a residual (not reachable: only the KPConv contraction splits K, and it
has no residual).

The multi-chunk KPConv pipeline (chunks of D3F_KPCONV_CHUNK queries; the variable is read once per process) runs in a
child process at two chunk sizes.
"""
import json
import os
import subprocess
import sys
import tempfile
import time
import zlib

import numpy as np
import pytest
import torch

from _oracle import TOL, assert_close, epilogue, gemm_mag, kpconv_ref
from test_gpu_kpconv import make_case, rel_err

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RTOL = 1e-4
SEEN = set()          # kernel names launched by the cases of this module


def t(a, dev):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def norm_name(n):
    return n.replace(" ", "")


def launched(fn):
    """(result of fn(), set of kernel names it launched), from torch.profiler's CUDA activity."""
    from torch.profiler import ProfilerActivity, profile
    names = set()
    # CUPTI occasionally delivers an empty activity buffer, at times for two sessions in a row; the ops are
    # deterministic, so the capture is simply repeated after a short pause
    for attempt in range(5):
        if attempt:
            time.sleep(0.1)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            out = fn()
            torch.cuda.synchronize()
        for e in prof.events():
            if e.device_type == torch.autograd.DeviceType.CUDA and not e.name.startswith(("Memcpy", "Memset")):
                names.add(norm_name(e.name))
        if names:
            break
    assert names, "the profiler recorded no CUDA kernel at all"
    SEEN.update(names)
    return out, names


def assert_ran(names, expect):
    for e in expect:
        assert any(e in n for n in names), "expected kernel %s; launched: %s" % (e, sorted(names))


# ---------------------------------------------------------------------------------------------------------------------
#  KPConv
# ---------------------------------------------------------------------------------------------------------------------

def kc(id, expect, Cin, Cout, Nq, Ns, H, **kw):
    d = dict(id=id, expect=expect, Cin=Cin, Cout=Cout, Nq=Nq, Ns=Ns, H=H, K=15, infl="linear", mode="sum",
             kind="rigid", misalign=False, env={}, epi=False, order=False, extent=0.1)
    d.update(kw)
    return d


FAST4, FAST8 = "kpconv_stage1_fast_kernel<4>", "kpconv_stage1_fast_kernel<8>"
STAGED4, STAGED8 = "kpconv_stage1_staged_kernel<4>", "kpconv_stage1_staged_kernel<8>"
GENERIC, GENERIC_D = "kpconv_stage1_kernel<15,1,false>", "kpconv_stage1_kernel<15,1,true>"
ANYK, ANYK_D = "kpconv_stage1_anyk_kernel<false>", "kpconv_stage1_anyk_kernel<true>"
SPLITK, F32 = "splitk_reduce_kernel", "gemm_f32_kernel<"


def mma(nt, deform, fast):
    return "kpconv_stage1_mma_kernel<%d,%s,%s>" % (nt, "true" if deform else "false", "true" if fast else "false")


KP_CASES = [
    kc("fast4_cin32", [FAST4, "prep_supports_vec_kernel<8>", "tc_gemm_kernel<32>"], 32, 32, 700, 700, 40, epi=True),
    kc("fast8_cin64", [FAST8, "prep_supports_vec_kernel<16>", "tc_gemm_kernel<64>"], 64, 64, 600, 900, 37),
    kc("fast8_cin128", [FAST8, "prep_supports_vec_kernel<32>", "tc_gemm_kernel<128>"], 128, 128, 400, 400, 40),
    kc("fast8_cin256", [FAST8], 256, 64, 300, 300, 30),
    kc("fast8_cin512", [FAST8, SPLITK], 512, 64, 200, 200, 21, epi=True),
    kc("fast8_cin1024", [FAST8], 1024, 32, 130, 130, 21),
    kc("staged4_cin32", [STAGED4], 32, 32, 700, 700, 40, env={"D3F_S1_STAGED": "1"}),
    kc("staged8_cin64", [STAGED8], 64, 64, 600, 900, 37, env={"D3F_S1_STAGED": "1"}),
    kc("staged8_cin256", [STAGED8], 256, 32, 300, 300, 29, env={"D3F_S1_STAGED": "1"}),
    kc("mma4_rigid_gaussian", [mma(4, False, False)], 32, 48, 600, 600, 32, infl="gaussian"),
    kc("mma4_rigid_closest", [mma(4, False, False)], 32, 32, 600, 600, 32, mode="closest"),
    kc("mma8_rigid_constant", [mma(8, False, False)], 64, 64, 500, 500, 30, infl="constant"),
    kc("mma8_rigid_gaussian_closest", [mma(8, False, False)], 64, 40, 500, 500, 30, infl="gaussian", mode="closest"),
    kc("mma16_rigid_closest", [mma(16, False, False)], 128, 64, 300, 300, 27, mode="closest"),
    kc("mma16_rigid_constant", [mma(16, False, False)], 256, 32, 200, 200, 24, infl="constant"),
    kc("mma4_deform", [mma(4, True, True)], 32, 32, 600, 600, 40, kind="deform"),
    kc("mma4_modulated", [mma(4, True, True)], 32, 32, 600, 600, 40, kind="mod", epi=True),
    kc("mma8_deform", [mma(8, True, True)], 64, 64, 500, 500, 33, kind="deform"),
    kc("mma8_modulated", [mma(8, True, True)], 64, 64, 500, 500, 33, kind="mod"),
    kc("mma16_deform", [mma(16, True, True)], 128, 64, 300, 300, 27, kind="deform"),
    kc("mma16_modulated", [mma(16, True, True)], 128, 64, 300, 300, 27, kind="mod"),
    kc("mma4_deform_gaussian", [mma(4, True, False)], 32, 32, 600, 600, 40, kind="deform", infl="gaussian"),
    kc("mma4_modulated_closest", [mma(4, True, False)], 32, 32, 600, 600, 40, kind="mod", mode="closest"),
    kc("mma8_deform_constant", [mma(8, True, False)], 64, 64, 500, 500, 33, kind="deform", infl="constant"),
    kc("mma8_modulated_gaussian", [mma(8, True, False)], 64, 48, 500, 500, 33, kind="mod", infl="gaussian"),
    kc("mma16_deform_closest", [mma(16, True, False)], 128, 64, 300, 300, 27, kind="deform", mode="closest"),
    kc("mma16_modulated_constant", [mma(16, True, False)], 128, 32, 300, 300, 27, kind="mod", infl="constant"),
    kc("v2_2_1_cin192", ["kpconv_stage1_v2_kernel<2,1,false>"], 192, 64, 300, 300, 30),
    kc("v2_2_2_cin96", ["kpconv_stage1_v2_kernel<2,2,false>"], 96, 64, 401, 401, 30, epi=True),
    kc("v2_2_1_cin192_deform", ["kpconv_stage1_v2_kernel<2,1,true>"], 192, 32, 300, 300, 30, kind="deform"),
    kc("v2_2_2_cin96_modulated", ["kpconv_stage1_v2_kernel<2,2,true>"], 96, 32, 401, 401, 30, kind="mod"),
    kc("generic_cin3", [GENERIC, F32], 3, 32, 500, 500, 30),
    kc("generic_cin5", [GENERIC, F32, "prep_supports_kernel"], 5, 64, 500, 500, 30, infl="gaussian"),
    kc("generic_cin48", [GENERIC, "tc_gemm_kernel<64>"], 48, 40, 500, 500, 40),
    kc("generic_cin5_deform", [GENERIC_D], 5, 32, 500, 500, 30, kind="deform"),
    kc("unaligned_cin32", [GENERIC, "prep_supports_kernel"], 32, 32, 600, 600, 40, misalign=True),
    kc("unaligned_cin64_closest", [GENERIC], 64, 32, 500, 500, 33, misalign=True, mode="closest"),
    kc("anyk_k1", [ANYK], 32, 32, 400, 400, 24, K=1),
    kc("anyk_k2", [ANYK], 32, 32, 400, 400, 24, K=2, mode="closest"),
    kc("anyk_k8", [ANYK], 32, 48, 400, 400, 24, K=8, infl="gaussian"),
    kc("anyk_k16", [ANYK], 16, 32, 400, 400, 24, K=16),
    kc("anyk_k31", [ANYK], 32, 32, 300, 300, 24, K=31),
    kc("anyk_k32", [ANYK], 32, 32, 300, 300, 24, K=32, infl="constant"),
    kc("anyk_k33", [ANYK], 32, 32, 300, 300, 24, K=33),
    kc("anyk_k64", [ANYK], 32, 32, 300, 300, 24, K=64, mode="closest"),
    kc("anyk_cin1_k33", [ANYK, F32], 1, 64, 400, 400, 30, K=33),
    kc("anyk_cin3_k7", [ANYK, F32], 3, 32, 400, 400, 30, K=7),
    kc("anyk_k13_deform", [ANYK_D], 32, 48, 400, 400, 30, K=13, kind="deform"),
    kc("anyk_k8_modulated", [ANYK_D], 32, 32, 400, 400, 30, K=8, kind="mod", infl="gaussian"),
    kc("cin1_fast", ["kpconv_cin1_kernel<true>"], 1, 64, 3000, 3000, 40, epi=True),
    kc("cin1_gaussian", ["kpconv_cin1_kernel<false>"], 1, 64, 1000, 1000, 40, infl="gaussian"),
    kc("cin1_closest", ["kpconv_cin1_kernel<false>"], 1, 32, 1000, 1000, 40, mode="closest"),
    kc("cin1_cout816", ["kpconv_cin1_kernel<true>"], 1, 816, 300, 300, 30),
    kc("fused_cin32", ["kpconv_fused32_kernel"], 32, 32, 4000, 4000, 35, epi=True, extent=0.05,
       env={"D3F_FUSED_KPCONV": "1"}),
    kc("splitk_cin64", [FAST8, SPLITK], 64, 64, 300, 300, 37, epi=True),
    kc("splitk_cin64_query_order", [FAST8, SPLITK], 64, 64, 300, 300, 37, order=True),
]


def kp_inputs(c):
    rng = np.random.default_rng(zlib.crc32(c["id"].encode()))
    q, s, idx, f, Kp, W = make_case(rng, c["Nq"], c["Ns"], c["H"], c["Cin"], c["Cout"], K=c["K"], extent=c["extent"])
    if c["Cin"] > 1:
        f[::5] = -np.abs(f[::5])          # some supports do not count towards nn
    off = mod = None
    if c["kind"] != "rigid":
        off = (rng.normal(size=(c["Nq"], c["K"], 3)) * 0.3 * c["extent"]).astype(np.float32)
    if c["kind"] == "mod":
        mod = rng.uniform(0.5, 1.5, (c["Nq"], c["K"])).astype(np.float32)
    epi = None
    if c["epi"]:
        epi = (rng.uniform(0.5, 1.5, c["Cout"]).astype(np.float32), rng.normal(size=c["Cout"]).astype(np.float32), 0.2)
    order = rng.permutation(c["Nq"]).astype(np.int32) if c["order"] else None
    return q, s, idx, f, Kp, W, off, mod, epi, order


def feature_tensor(f, dev, misalign):
    if not misalign:
        return t(f, dev)
    buf = torch.empty(f.size + 1, dtype=torch.float32, device=dev)
    view = buf[1:].view(f.shape)                  # contiguous, 4 bytes past a 16-byte boundary
    view.copy_(torch.from_numpy(f))
    assert view.data_ptr() % 16 != 0
    return view


def run_kp(c, dev, monkeypatch):
    from d3feat_b200 import convolution_ops as co
    for k, v in c["env"].items():
        monkeypatch.setenv(k, v)
    q, s, idx, f, Kp, W, off, mod, epi, order = kp_inputs(c)
    args = [t(q, dev), t(s, dev), t(idx, dev), feature_tensor(f, dev, c["misalign"]), t(Kp, dev)]
    e = None if epi is None else (t(epi[0], dev), t(epi[1], dev), epi[2])
    o = None if order is None else t(order, dev)
    Wt = t(W, dev)
    co.packed_weight(Wt)
    if c["kind"] == "rigid":
        fn = lambda: co.KPConv_ops(*args, Wt, c["extent"], c["infl"], c["mode"], epilogue=e, query_order=o)
    else:
        fn = lambda: co.KPConv_deform_ops(*args, t(off, dev), None if mod is None else t(mod, dev), Wt, c["extent"],
                                          c["infl"], c["mode"], epilogue=e, query_order=o)
    out, names = launched(fn)
    return out.cpu().numpy(), names, (q, s, idx, f, Kp, W, off, mod, epi)


@pytest.mark.parametrize("c", KP_CASES, ids=[c["id"] for c in KP_CASES])
def test_kpconv_variant(cuda, monkeypatch, c):
    out, names, (q, s, idx, f, Kp, W, off, mod, epi) = run_kp(c, cuda, monkeypatch)
    assert_ran(names, c["expect"])
    ref, mag, alt = kpconv_ref(q, s, idx, f, Kp, W, c["extent"], c["infl"], c["mode"], off, mod,
                               deform=c["kind"] != "rigid", epi=epi)
    assert rel_err(out, ref) < RTOL
    assert_close(out, ref, mag, TOL, "kpconv " + c["id"], alt=alt)


def test_kpconv_cin1_cout817_runs_two_stage(cuda):
    """Cin = 1 with W[15, 817] past the first-layer kernel's 48 KB: the generic stage 1 and the CUDA-core contraction
    (K * Cin = 15) run instead, with the same normalisation."""
    from d3feat_b200 import convolution_ops as co
    q, s, idx, f, Kp, W = make_case(np.random.default_rng(1), 200, 200, 20, 1, 817)
    f[::3] = -np.abs(f[::3])              # supports that do not count towards nn
    out, names = launched(lambda: co.KPConv_ops(t(q, cuda), t(s, cuda), t(idx, cuda), t(f, cuda), t(Kp, cuda),
                                                t(W, cuda), 0.06, "linear", "sum"))
    assert_ran(names, [GENERIC, F32])
    assert not any("kpconv_cin1_kernel" in n for n in names)
    ref, mag, alt = kpconv_ref(q, s, idx, f, Kp, W, 0.06)
    assert_close(out.cpu().numpy(), ref, mag, TOL, "kpconv cin1 cout817", alt=alt)


# ---- edges, on each stage-1 family ----------------------------------------------------------------------------------

FAMILIES = {
    "fast4": dict(Cin=32, Cout=32), "fast8": dict(Cin=64, Cout=64), "fast8_wide": dict(Cin=256, Cout=32),
    "mma4": dict(Cin=32, Cout=32, infl="gaussian"), "mma16_deform": dict(Cin=128, Cout=32, kind="mod"),
    "v2_2_2": dict(Cin=96, Cout=32), "generic": dict(Cin=5, Cout=32), "anyk": dict(Cin=32, Cout=32, K=7),
    "cin1": dict(Cin=1, Cout=64), "staged8": dict(Cin=64, Cout=32, env={"D3F_S1_STAGED": "1"}),
}
EDGES = ["nq1", "nq3", "nq5", "nq0", "h1", "h13", "shadow_zero_cancelling_rows", "ns0", "query_order"]


@pytest.mark.parametrize("edge", EDGES)
@pytest.mark.parametrize("fam", sorted(FAMILIES))
def test_kpconv_edges(cuda, monkeypatch, fam, edge):
    from d3feat_b200 import convolution_ops as co
    c = kc(fam + "_" + edge, [], Nq=200, Ns=200, H=24, **FAMILIES[fam])
    if edge.startswith("nq"):
        c["Nq"] = int(edge[2:])
    if edge == "h1":
        c["H"] = 1
    if edge == "h13":
        c["H"] = 13
    c["order"] = edge == "query_order"
    for k, v in c["env"].items():
        monkeypatch.setenv(k, v)
    rng = np.random.default_rng(len(fam) * 31 + EDGES.index(edge))
    Nq, Ns, H, K, Cin, Cout = c["Nq"], c["Ns"], c["H"], c["K"], c["Cin"], c["Cout"]
    s = rng.uniform(0, 1, (Ns, 3)).astype(np.float32)
    q = s[:Nq].copy()
    idx = np.full((Nq, H), Ns, np.int32)
    if Nq:
        from oracle import native as on
        nbr = on.port_batch_neighbors(q, s, [Nq], [Ns], 0.25, max_cols=H)
        idx[:, :nbr.shape[1]] = nbr[:, :H]
    f = rng.normal(size=(Ns, Cin)).astype(np.float32)
    if edge == "shadow_zero_cancelling_rows":
        idx[::4] = Ns                                   # rows whose every neighbour is the shadow point
        f[::3] = 0                                      # zero feature rows
        if Cin % 2 == 0:
            f[1::3, 1::2] = -f[1::3, 0::2]              # exactly cancelling rows [a, -a, b, -b, ...]
    if edge == "ns0":
        Ns = 0
        s, f = s[:0], f[:0]
        idx[:] = 0                                      # every index is the shadow point
    Kp = np.concatenate([np.zeros((1, 3)), rng.normal(size=(K - 1, 3))], 0)
    Kp[1:] *= 0.15 / np.linalg.norm(Kp[1:], axis=1, keepdims=True)
    Kp = Kp.astype(np.float32)
    W = (rng.normal(size=(K, Cin, Cout)) * np.sqrt(2.0 / Cout)).astype(np.float32)
    off = mod = None
    if c["kind"] != "rigid":
        off = (rng.normal(size=(Nq, K, 3)) * 0.03).astype(np.float32)
        mod = rng.uniform(0.5, 1.5, (Nq, K)).astype(np.float32)
    order = t(rng.permutation(Nq).astype(np.int32), cuda) if c["order"] else None
    args = [t(q, cuda), t(s, cuda), t(idx, cuda), t(f, cuda), t(Kp, cuda), t(W, cuda)]
    if c["kind"] == "rigid":
        out = co.KPConv_ops(*args, 0.1, c["infl"], "sum", query_order=order)
    else:
        out = co.KPConv_deform_ops(*args[:5], t(off, cuda), t(mod, cuda), args[5], 0.1, c["infl"], "sum",
                                   query_order=order)
    out = out.cpu().numpy()
    assert out.shape == (Nq, Cout)
    ref, mag, alt = kpconv_ref(q, s, idx, f, Kp, W, 0.1, c["infl"], "sum", off, mod, deform=c["kind"] != "rigid")
    assert_close(out, ref, mag, TOL, "kpconv edge %s %s" % (fam, edge), alt=alt)
    if edge == "ns0":
        assert np.all(out == 0)
    if edge == "shadow_zero_cancelling_rows":
        assert np.all(out[::4] == 0)                    # all-shadow rows: nothing to accumulate, exactly zero


# ---------------------------------------------------------------------------------------------------------------------
#  GEMM (unary convolution, the resnetb tail pair)
# ---------------------------------------------------------------------------------------------------------------------

def gc(id, expect, N, Cin, Cout, env=None, epi=True):
    return dict(id=id, expect=expect, N=N, Cin=Cin, Cout=Cout, env=env or {}, epi=epi)


TC = "tc_gemm_kernel<%d>"
GEMM_CASES = [
    gc("bn32", [TC % 32], 3000, 64, 32),
    gc("bn64", [TC % 64], 3000, 64, 48),
    gc("bn128", [TC % 128], 3000, 256, 128),
    gc("bn64_skinny_k_override", [TC % 64], 9000, 64, 128),
    gc("one_tile_k512", [TC % 128], 3000, 512, 128),
    gc("persistent_stream_k512", [TC % 128], 3000, 512, 128, env={"D3F_TC_STREAM": "1"}),
    gc("persistent_nk4", [TC % 64], 20000, 128, 64),
    gc("n1", [TC % 32], 1000, 64, 1),
    gc("n8", [TC % 32], 1000, 64, 8),
    gc("n33", [TC % 64], 1000, 64, 33),
    gc("n45", [TC % 64], 1000, 64, 45),
    gc("k4", [TC % 64], 1000, 4, 64),
    gc("k8", [TC % 64], 1000, 8, 64),
    gc("k36", [TC % 64], 1000, 36, 64),
    gc("f32_small", [F32], 1000, 5, 64),
    gc("f32_narrow", [F32], 1000, 7, 33),
    gc("f32_wide", ["gemm_f32_kernel<128,128,8,8,8>"], 34000, 6, 128, epi=False),
]


@pytest.mark.parametrize("c", GEMM_CASES, ids=[c["id"] for c in GEMM_CASES])
def test_gemm_variant(cuda, monkeypatch, c):
    from d3feat_b200 import convolution_ops as co
    for k, v in c["env"].items():
        monkeypatch.setenv(k, v)
    rng = np.random.default_rng(c["N"] + c["Cin"] * 7 + c["Cout"])
    N, Cin, Cout = c["N"], c["Cin"], c["Cout"]
    x = rng.normal(size=(N, Cin)).astype(np.float32)
    w = (rng.normal(size=(Cin, Cout)) * np.sqrt(2.0 / Cout)).astype(np.float32)
    wt = t(w, cuda)
    co.packed_weight(wt)
    ref, mag = x.astype(np.float64) @ w.astype(np.float64), gemm_mag(x, w)
    if c["epi"]:
        scale = rng.uniform(0.5, 1.5, Cout).astype(np.float32)
        shift = rng.normal(size=Cout).astype(np.float32)
        res = rng.normal(size=(N, Cout)).astype(np.float32)
        fn = lambda: co.unary_convolution(t(x, cuda), wt, epilogue=(t(scale, cuda), t(shift, cuda), 0.2),
                                          residual=t(res, cuda))
        ref, mag = epilogue(ref, mag, scale, shift, residual=res, alpha=0.2)
    else:
        fn = lambda: co.unary_convolution(t(x, cuda), wt)
    out, names = launched(fn)
    assert_ran(names, c["expect"])
    out = out.cpu().numpy()
    assert rel_err(out, ref) < RTOL
    assert_close(out, ref, mag, TOL, "gemm " + c["id"])


PAIR_CASES = [(32, 36), (64, 4), (32, 2048)]


@pytest.mark.parametrize("C1,C2", PAIR_CASES)
def test_unary_pair_variant(cuda, C1, C2):
    from d3feat_b200 import convolution_ops as co
    rng = np.random.default_rng(C1 + C2)
    N, Cout = 1500, 64
    x1 = rng.normal(size=(N, C1)).astype(np.float32)
    x2 = rng.normal(size=(N, C2)).astype(np.float32)
    w1 = (rng.normal(size=(C1, Cout)) * np.sqrt(2.0 / Cout)).astype(np.float32)
    w2 = (rng.normal(size=(C2, Cout)) * np.sqrt(2.0 / Cout)).astype(np.float32)
    s1, s2 = (rng.uniform(0.5, 1.5, Cout).astype(np.float32) for _ in range(2))
    t1, t2 = (rng.normal(size=Cout).astype(np.float32) for _ in range(2))
    T = [t(a, cuda) for a in (x1, w1, s1, t1, x2, w2, s2, t2)]
    out, names = launched(lambda: co.unary_pair_convolution(T[0], T[1], (T[2], T[3]), T[4], T[5], (T[6], T[7]), 0.2))
    assert_ran(names, ["tc_gemm_kernel<"])
    assert not any("gemm_f32" in n for n in names)
    y, m = epilogue(x1.astype(np.float64) @ w1.astype(np.float64), gemm_mag(x1, w1), s1, t1)
    y2, m2 = epilogue(x2.astype(np.float64) @ w2.astype(np.float64), gemm_mag(x2, w2), s2, t2)
    ref, mag = epilogue(y + y2, m + m2, alpha=0.2)
    out = out.cpu().numpy()
    assert rel_err(out, ref) < RTOL
    assert_close(out, ref, mag, TOL, "unary_pair %d+%d" % (C1, C2))


# ---------------------------------------------------------------------------------------------------------------------
#  multi-chunk KPConv (child process: the chunk size is read once per process)
# ---------------------------------------------------------------------------------------------------------------------

CHUNK_DRIVER = r"""
import json, sys
import numpy as np, torch
sys.path.insert(0, sys.argv[1])
from d3feat_b200 import convolution_ops as co
d = sys.argv[2]
cases = json.load(open(d + "/cases.json"))
dev = torch.device("cuda", 0)
def t(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)
for c in cases:
    z = np.load(d + "/in_%s.npz" % c["id"])
    args = [t(z[k]) for k in ("q", "s", "idx", "f", "Kp")]
    order = t(z["order"]) if "order" in z else None
    rows_q = torch.tensor([c["rows_q"]], dtype=torch.int32, device=dev) if c["rows_q"] is not None else None
    if c["deform"]:
        out = co.KPConv_deform_ops(*args, t(z["off"]), None, t(z["W"]), c["extent"], "linear", "sum",
                                   query_order=order, rows_q=rows_q)
    else:
        out = co.KPConv_ops(*args, t(z["W"]), c["extent"], "linear", "sum", query_order=order, rows_q=rows_q)
    np.save(d + "/out_%s.npy" % c["id"], out.cpu().numpy())
torch.cuda.synchronize()
"""

CHUNK_CASES = [
    dict(id="rigid_cin32", Cin=32, Cout=32, Nq=700, deform=False, order=False, rows_q=None),
    dict(id="rigid_cin64", Cin=64, Cout=64, Nq=700, deform=False, order=False, rows_q=None),
    dict(id="rigid_cin512_splitk", Cin=512, Cout=64, Nq=450, deform=False, order=False, rows_q=None),
    dict(id="deform_cin64", Cin=64, Cout=32, Nq=700, deform=True, order=False, rows_q=None),
    dict(id="query_order_cin32", Cin=32, Cout=32, Nq=700, deform=False, order=True, rows_q=None),
    dict(id="rows_q_mid_cin64", Cin=64, Cout=64, Nq=700, deform=False, order=False, rows_q=300),
]


@pytest.mark.parametrize("chunk", [128, 1024])
def test_kpconv_multi_chunk_pipeline(cuda, chunk):
    """D3F_KPCONV_CHUNK = 128 / 1024 queries: every case spans >= 3 chunks with a ragged last one (auxiliary stream,
    event joins, double-buffered wf / inv_nn, buffer-reuse waits, per-chunk row-map offset, split-K inside a chunk).
    One device row count ends inside a middle chunk, so the later chunks have no rows (the m_off clamp); the rows
    below the count are compared (tests/test_gpu_row_counts.py covers what happens past it)."""
    scale = chunk // 128
    rng = np.random.default_rng(chunk)
    with tempfile.TemporaryDirectory() as d:
        cases, data = [], {}
        for c in CHUNK_CASES:
            c = dict(c, Nq=c["Nq"] * scale, extent=0.06)
            n = c["Nq"]
            assert -(-n // chunk) >= 3 and n % chunk != 0
            H = 24 if c["Cin"] >= 512 else 36
            q, s, idx, f, Kp, W = make_case(rng, n, n, H, c["Cin"], c["Cout"], extent=c["extent"])
            f[::5] = -np.abs(f[::5])
            z = dict(q=q, s=s, idx=idx, f=f, Kp=Kp, W=W)
            if c["deform"]:
                z["off"] = (rng.normal(size=(n, 15, 3)) * 0.02).astype(np.float32)
            if c["order"]:
                z["order"] = rng.permutation(n).astype(np.int32)
            if c["rows_q"] is not None:
                c["rows_q"] = c["rows_q"] * scale + 17
                assert chunk <= c["rows_q"] < n - chunk
            np.savez(os.path.join(d, "in_%s.npz" % c["id"]), **z)
            cases.append(c)
            data[c["id"]] = z
        with open(os.path.join(d, "cases.json"), "w") as fh:
            json.dump(cases, fh)
        env = dict(os.environ, D3F_KPCONV_CHUNK=str(chunk))
        r = subprocess.run([sys.executable, "-c", CHUNK_DRIVER, ROOT, d], env=env, capture_output=True, text=True,
                           timeout=600)
        assert r.returncode == 0, r.stderr[-4000:]
        for c in cases:
            z = data[c["id"]]
            out = np.load(os.path.join(d, "out_%s.npy" % c["id"]))
            n = c["rows_q"] if c["rows_q"] is not None else c["Nq"]
            ref, mag, alt = kpconv_ref(z["q"][:n], z["s"], z["idx"][:n], z["f"], z["Kp"], z["W"], c["extent"],
                                       offsets=None if not c["deform"] else z["off"][:n], deform=c["deform"])
            assert_close(out[:n], ref, mag, TOL, "chunk %d %s" % (chunk, c["id"]), alt=alt)


# ---------------------------------------------------------------------------------------------------------------------

def test_every_table_instance_was_launched(cuda, monkeypatch):
    """The union of kernel names the cases above launched covers every instance the tables name (cases that did not
    run in this session, e.g. under -k, are run here for their kernel names)."""
    missing = []
    for c in KP_CASES:
        if not all(any(e in n for n in SEEN) for e in c["expect"]):
            with monkeypatch.context() as m:
                run_kp(c, cuda, m)
    for e in sorted({e for c in KP_CASES + GEMM_CASES for e in c["expect"]}):
        if not any(e in n for n in SEEN):
            missing.append(e)
    assert not missing, "table instances never launched: %s (seen: %s)" % (missing, sorted(SEEN))
