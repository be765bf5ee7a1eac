"""Workspace layouts: every `d3f_*_workspace_bytes` query measures the same layout its entry point carves.

CPU: the 23 queries on a fixed table of argument sets (empty inputs, B = 1024, 3DMatch level-0 shapes) give the
values the library gave before each layout was written once, as one function that both sizes and carves, minus
only what that change removed:
  * the unexplained slack: +1024 in kpconv, kpconv_backward, unary_backward, batch_norm_train,
    ind_max_pool_backward, gather_rows_backward, detection_scores_backward and pyramid; +256 in grid_subsample,
    voxel_down_sample, radius_neighbors and momentum_clip; +512 around the pyramid's subsampling region (the
    pyramid's level counts and status are now two explicit buffers of their own);
  * the 256-byte padding that the hand-written formulas put after the last buffer of a layout;
  * four of batch norm's six C-vectors: the old formula reserved six, the forward uses two and the backward the same
    two (e.g. (60000, 64): 33280 -> 31232 bytes = 1024 of slack + 4 x 256);
  * +256 after the fused KPConv weight image, which is read at the 256-byte alignment it is carved at;
  * the pyramid's pool grid over the last level, which the build never makes.
Argument sets that were refused (0) are still refused.

GPU (-m gpu): every entry point that takes a workspace, on real inputs and on each branch that changes its layout,
is called with `need - 1` bytes (it must return D3F_ERR_WORKSPACE and leave the buffer untouched) and with `need`
bytes inside a sentinel-filled allocation of `need + 4096` (the guard must survive and the outputs must equal those of
a call with a fresh 2 * need workspace, bit for bit). Ops called through their Python wrappers get their workspaces
that way by replacing the allocator the wrapper uses. d3f_kpconv_reverse_width only reads the table-build phase of the
backward layout, so it accepts less than its query: it is checked at the exact size only.
"""
import ctypes as C
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from d3feat_b200 import _lib, pyramid, synth  # noqa: E402

def _bbox(lo, hi):
    return (C.c_float * 6)(*lo, *hi)


ROOM = _bbox((-1.5, -1.5, -1.5), (1.5, 1.5, 1.5))
FAR = _bbox((-400.0, -400.0, -400.0), (400.0, 400.0, 400.0))


def _spec(kind):
    if kind == "3dmatch":
        spec, _ = pyramid.make_spec(synth.Config(), [40, 30, 34, 35, 35])
    else:   # every level subsampled, the last one included
        spec = pyramid.PyramidSpec()
        spec.n_levels = 3
        for l in range(3):
            spec.conv_radius[l] = 0.075 * 2 ** l
            spec.sub_dl[l] = 0.06 * 2 ** l
            spec.pool_radius[l] = 0.09 * 2 ** l
            spec.up_radius[l] = 0.15 * 2 ** l
            spec.limit[l] = 30
        if kind == "bad_levels":
            spec.n_levels = 9
    return spec


def _caps(*c):
    return (C.c_int * 8)(*(list(c) + [0] * (8 - len(c))))


# (query, args): the table the expected values below were taken on
CASES = [
    ("d3f_grid_subsample_workspace_bytes", (0, 1)),
    ("d3f_grid_subsample_workspace_bytes", (60000, 2)),
    ("d3f_grid_subsample_workspace_bytes", (1000000, 1024)),
    ("d3f_voxel_down_sample_workspace_bytes", (0, 1)),
    ("d3f_voxel_down_sample_workspace_bytes", (250000, 2)),
    ("d3f_voxel_down_sample_workspace_bytes", (1000000, 1024)),
    ("d3f_voxel_down_sample_workspace_bytes", (-1, 1)),
    ("d3f_voxel_down_sample_workspace_bytes", (10, 0)),
    ("d3f_voxel_down_sample_workspace_bytes", (10, 1025)),
    ("d3f_radius_neighbors_workspace_bytes", (0, 1, 0.075, ROOM)),
    ("d3f_radius_neighbors_workspace_bytes", (60000, 2, 0.075, ROOM)),
    ("d3f_radius_neighbors_workspace_bytes", (1000000, 1024, 0.6, ROOM)),
    ("d3f_radius_neighbors_workspace_bytes", (100, 1, 0.0, ROOM)),
    ("d3f_radius_neighbors_workspace_bytes", (100, 0, 0.075, ROOM)),
    ("d3f_radius_neighbors_workspace_bytes", (100, 1, 0.075, None)),
    ("d3f_radius_neighbors_workspace_bytes", (100, 1, 0.001, FAR)),
    ("d3f_pyramid_workspace_bytes", (2, "3dmatch", (60000, 16000, 4000, 1000, 300), ROOM)),
    ("d3f_pyramid_workspace_bytes", (1, "3dmatch", (0, 0, 0, 0, 0), ROOM)),
    ("d3f_pyramid_workspace_bytes", (1024, "3dmatch", (1000000, 300000, 80000, 20000, 5000), ROOM)),
    ("d3f_pyramid_workspace_bytes", (2, "all_sub", (5000, 2000, 800), ROOM)),
    ("d3f_pyramid_workspace_bytes", (2, "bad_levels", (5000, 2000, 800), ROOM)),
    ("d3f_pyramid_workspace_bytes", (2, "3dmatch", (60000, 16000, 4000, 1000, 300), None)),
    ("d3f_pyramid_workspace_bytes", (2, "3dmatch", (60000, 16000, 4000, 1000, 300), FAR)),
    ("d3f_kpconv_workspace_bytes", (0, 0, 40, 15, 1, 64)),
    ("d3f_kpconv_workspace_bytes", (60000, 60000, 40, 15, 1, 64)),
    ("d3f_kpconv_workspace_bytes", (60000, 60000, 40, 15, 32, 32)),
    ("d3f_kpconv_workspace_bytes", (16000, 60000, 30, 15, 64, 128)),
    ("d3f_kpconv_workspace_bytes", (300, 1000, 35, 15, 512, 1024)),
    ("d3f_kpconv_workspace_bytes", (1000000, 1000000, 40, 15, 32, 32)),
    ("d3f_kpconv_backward_workspace_bytes", (0, 0, 40, 15, 32, 32, 0)),
    ("d3f_kpconv_backward_workspace_bytes", (60000, 60000, 40, 15, 32, 32, 0)),
    ("d3f_kpconv_backward_workspace_bytes", (60000, 60000, 40, 15, 32, 32, 55)),
    ("d3f_kpconv_backward_workspace_bytes", (16000, 60000, 30, 15, 64, 128, 12)),
    ("d3f_kpconv_backward_workspace_bytes", (300, 1000, 35, 15, 512, 1024, 20)),
    ("d3f_kpconv_backward_workspace_bytes", (-1, 10, 4, 15, 1, 1, 0)),
    ("d3f_kpconv_backward_workspace_bytes", (10, 10, 4, 0, 1, 1, 0)),
    ("d3f_kpconv_backward_workspace_bytes", (10, 10, 4, 15, 1, 1, -1)),
    ("d3f_unary_backward_workspace_bytes", (0, 1, 1)),
    ("d3f_unary_backward_workspace_bytes", (60000, 64, 32)),
    ("d3f_unary_backward_workspace_bytes", (1000000, 1024, 2048)),
    ("d3f_unary_backward_workspace_bytes", (-1, 1, 1)),
    ("d3f_unary_backward_workspace_bytes", (10, 0, 1)),
    ("d3f_ind_max_pool_workspace_bytes", (0,)),
    ("d3f_ind_max_pool_workspace_bytes", (1,)),
    ("d3f_ind_max_pool_workspace_bytes", (64,)),
    ("d3f_ind_max_pool_workspace_bytes", (1024,)),
    ("d3f_detection_scores_workspace_bytes", (0, 1)),
    ("d3f_detection_scores_workspace_bytes", (60000, 2)),
    ("d3f_detection_scores_workspace_bytes", (1000000, 1024)),
    ("d3f_batch_norm_train_workspace_bytes", (0, 1)),
    ("d3f_batch_norm_train_workspace_bytes", (60000, 64)),
    ("d3f_batch_norm_train_workspace_bytes", (1000000, 1024)),
    ("d3f_batch_norm_train_workspace_bytes", (-1, 1)),
    ("d3f_batch_norm_train_workspace_bytes", (10, 0)),
    ("d3f_ind_max_pool_backward_workspace_bytes", (1, 0, 0, 1)),
    ("d3f_ind_max_pool_backward_workspace_bytes", (60000, 16000, 34, 64)),
    ("d3f_ind_max_pool_backward_workspace_bytes", (1000000, 300000, 40, 1024)),
    ("d3f_ind_max_pool_backward_workspace_bytes", (0, 10, 1, 1)),
    ("d3f_ind_max_pool_backward_workspace_bytes", (10, 1 << 20, 1 << 11, 1)),
    ("d3f_gather_rows_backward_workspace_bytes", (0, 0)),
    ("d3f_gather_rows_backward_workspace_bytes", (60000, 16000)),
    ("d3f_gather_rows_backward_workspace_bytes", (1000000, 1000000)),
    ("d3f_gather_rows_backward_workspace_bytes", (-1, 0)),
    ("d3f_detection_scores_backward_workspace_bytes", (0, 0, 1, 1)),
    ("d3f_detection_scores_backward_workspace_bytes", (60000, 40, 2, 32)),
    ("d3f_detection_scores_backward_workspace_bytes", (1000000, 40, 1024, 32)),
    ("d3f_detection_scores_backward_workspace_bytes", (10, 4, 0, 32)),
    ("d3f_detection_scores_backward_workspace_bytes", (1 << 20, 1 << 11, 1, 32)),
    ("d3f_select_keypoints_workspace_bytes", (0, 1)),
    ("d3f_select_keypoints_workspace_bytes", (60000, 2)),
    ("d3f_select_keypoints_workspace_bytes", (1000000, 1024)),
    ("d3f_select_keypoints_workspace_bytes", (-1, 1)),
    ("d3f_select_keypoints_workspace_bytes", (10, 0)),
    ("d3f_sample_keypoints_workspace_bytes", (1,)),
    ("d3f_sample_keypoints_workspace_bytes", (1024,)),
    ("d3f_sample_keypoints_workspace_bytes", (0,)),
    ("d3f_match_descriptors_workspace_bytes", (1, 1)),
    ("d3f_match_descriptors_workspace_bytes", (5000, 1)),
    ("d3f_match_descriptors_workspace_bytes", (250, 1024)),
    ("d3f_match_descriptors_workspace_bytes", (0, 1)),
    ("d3f_match_descriptors_workspace_bytes", (65536, 65536)),
    ("d3f_register_pairs_workspace_bytes", (1, 1, 1, 1)),
    ("d3f_register_pairs_workspace_bytes", (5000, 1, 50000, 1000)),
    ("d3f_register_pairs_workspace_bytes", (250, 1024, 50000, 1000)),
    ("d3f_register_pairs_workspace_bytes", (0, 6, 50000, 1000)),
    ("d3f_register_pairs_workspace_bytes", (250, 6, 50000, 50001)),
    ("d3f_icp_pairs_workspace_bytes", (0, 2, 1, 0.05, ROOM)),
    ("d3f_icp_pairs_workspace_bytes", (60000, 2, 1, 0.05, ROOM)),
    ("d3f_icp_pairs_workspace_bytes", (1000000, 1024, 512, 0.1, ROOM)),
    ("d3f_icp_pairs_workspace_bytes", (100, 2, 0, 0.05, ROOM)),
    ("d3f_icp_pairs_workspace_bytes", (100, 2, 1, 0.05, None)),
    ("d3f_evaluate_pairs_workspace_bytes", (1, 0)),
    ("d3f_evaluate_pairs_workspace_bytes", (1024, 2)),
    ("d3f_evaluate_pairs_workspace_bytes", (0, 1)),
    ("d3f_evaluate_pairs_workspace_bytes", (10, 3)),
    ("d3f_pair_correspondences_workspace_bytes", (0, 2, 1, 0.0375, ROOM)),
    ("d3f_pair_correspondences_workspace_bytes", (60000, 2, 1, 0.0375, ROOM)),
    ("d3f_pair_correspondences_workspace_bytes", (1000000, 1024, 512, 0.0375, ROOM)),
    ("d3f_pair_correspondences_workspace_bytes", (100, 2, 0, 0.0375, ROOM)),
    ("d3f_pair_correspondences_workspace_bytes", (100, 2, 1, -1.0, ROOM)),
    ("d3f_sample_correspondences_workspace_bytes", (0, 1)),
    ("d3f_sample_correspondences_workspace_bytes", (3000000, 2)),
    ("d3f_sample_correspondences_workspace_bytes", (20000000, 512)),
    ("d3f_sample_correspondences_workspace_bytes", (10, 0)),
    ("d3f_augment_pairs_workspace_bytes", (1, 1)),
    ("d3f_augment_pairs_workspace_bytes", (1024, 512)),
    ("d3f_augment_pairs_workspace_bytes", (0, 1)),
    ("d3f_momentum_clip_workspace_bytes", (0, 0)),
    ("d3f_momentum_clip_workspace_bytes", (60, 9000000)),
    ("d3f_momentum_clip_workspace_bytes", (1024, 1 << 34)),
    ("d3f_momentum_clip_workspace_bytes", (-1, 10)),
    ("d3f_momentum_clip_workspace_bytes", (1, -1)),
]


def query(lib, name, args):
    if name == "d3f_pyramid_workspace_bytes":
        B, kind, caps, bb = args
        spec = _spec(kind)
        return getattr(lib, name)(B, C.byref(spec), _caps(*caps), bb)
    return getattr(lib, name)(*args)


# value of each CASES entry before and after the layouts were unified (0 = refused)
EXPECTED = [
    (4356, 4100),
    (2432772, 2432516),
    (40532228, 40531972),
    (4100, 3844),
    (8128772, 8128516),
    (32520196, 32519940),
    (0, 0),
    (0, 0),
    (0, 0),
    (552844, 552588),
    (2304020, 2303764),
    (21779380, 21779124),
    (0, 0),
    (0, 0),
    (0, 0),
    (0, 0),
    (5344768, 5341960),
    (653568, 650760),
    (722539520, 722536836),
    (2596864, 2560524),
    (0, 0),
    (0, 0),
    (0, 0),
    (125440, 124160),
    (8764928, 8763648),
    (231964672, 231963392),
    (173899776, 173898496),
    (31157760, 31156480),
    (1091840512, 1091839232),
    (314880, 312576),
    (241030656, 241028352),
    (253990656, 253988352),
    (960872448, 960870144),
    (235492608, 235490304),
    (0, 0),
    (0, 0),
    (0, 0),
    (9728, 8452),
    (271360, 270336),
    (4127196160, 4127195136),
    (0, 0),
    (0, 0),
    (8, 8),
    (8, 8),
    (260, 260),
    (4100, 4100),
    (768, 513),
    (60672, 60513),
    (1008640, 1008449),
    (3072, 772),
    (33280, 31232),
    (8037376, 8019968),
    (0, 0),
    (0, 0),
    (3592, 2568),
    (18042880, 18041856),
    (1578821632, 1578820608),
    (0, 0),
    (0, 0),
    (2568, 1544),
    (873596, 872572),
    (32504232, 32503208),
    (0, 0),
    (3841, 2817),
    (90302817, 90301793),
    (1505020993, 1505019969),
    (0, 0),
    (0, 0),
    (1280, 1280),
    (1471232, 1471232),
    (24505088, 24505088),
    (0, 0),
    (0, 0),
    (256, 8),
    (4352, 4100),
    (0, 0),
    (512, 264),
    (80384, 80192),
    (4096000, 4096000),
    (0, 0),
    (0, 0),
    (1536, 1288),
    (23296, 23104),
    (22794240, 22794240),
    (0, 0),
    (0, 0),
    (3635068, 3634812),
    (5108604, 5108348),
    (2592638148, 2592637892),
    (0, 0),
    (0, 0),
    (256, 4),
    (8192, 8192),
    (0, 0),
    (0, 0),
    (8507424, 8507168),
    (9709088, 9708832),
    (0, 0),
    (0, 0),
    (0, 0),
    (2048, 2048),
    (73500160, 73500160),
    (490000384, 490000384),
    (0, 0),
    (272, 272),
    (12544, 12544),
    (0, 0),
    (256, 8),
    (36096, 35640),
    (67117312, 67117056),
    (0, 0),
    (0, 0),
]


def test_every_query_is_in_the_table():
    names = {s[0] for s in _lib.SYMBOLS if s[0].endswith("_workspace_bytes")}
    assert len(names) == 23
    assert {n for n, _ in CASES} == names


def test_query_values():
    lib = _lib.lib()
    for (name, args), (before, after) in zip(CASES, EXPECTED):
        got = query(lib, name, args)
        assert got == after, (name, args, got, after)
        assert (after == 0) == (before == 0), (name, args)
        assert after <= before, (name, args)


# ---- GPU: every entry point on exactly its workspace ----------------------------------------------------------------
SENTINEL = 0xA5
GUARD = 4096


def _ptr(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def _stream():
    import torch
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def check_exact_workspace(need, run):
    """run(ws_ptr, nbytes) -> (rc, [outputs]) with fresh outputs per call."""
    import torch
    assert need > 0
    buf = torch.full((need + GUARD,), SENTINEL, dtype=torch.uint8, device="cuda")
    rc, _ = run(buf.data_ptr(), need - 1)
    torch.cuda.synchronize()
    assert rc == -4, rc
    assert bool((buf == SENTINEL).all()), "a refused call wrote to its workspace"
    rc, outs = run(buf.data_ptr(), need)
    torch.cuda.synchronize()
    assert rc == 0, (rc, _lib.lib().d3f_last_error())
    assert bool((buf[need:] == SENTINEL).all()), "the op wrote past the bytes its query asked for"
    fresh = torch.zeros((2 * need,), dtype=torch.uint8, device="cuda")
    rc, ref = run(fresh.data_ptr(), 2 * need)
    torch.cuda.synchronize()
    assert rc == 0
    for a, b in zip(outs, ref):
        assert torch.equal(a.view(torch.uint8), b.view(torch.uint8))


def _cloud(n, seed, scale=1.2):
    import torch
    g = torch.Generator().manual_seed(seed)
    return ((torch.rand((n, 3), generator=g) * 2 - 1) * scale).cuda()


def _lens(*l):
    import torch
    return torch.tensor(l, dtype=torch.int32, device="cuda")


@pytest.mark.gpu
def test_grid_subsample_voxel_and_neighbors_on_exact_workspaces(cuda):
    import torch
    L = _lib.lib()
    pts, lens = _cloud(5000, 0), _lens(3000, 2000)
    N, B = 5000, 2

    def subsample(ws, nb):
        o = [torch.zeros((N, 3), device="cuda"), torch.zeros((B,), dtype=torch.int32, device="cuda"),
             torch.zeros((1,), dtype=torch.int32, device="cuda")]
        rc = L.d3f_grid_subsample(_ptr(pts), _ptr(lens), B, N, 0.06, None, 0, None, 0, ROOM, _ptr(o[0]), None, None,
                                  _ptr(o[1]), _ptr(o[2]), ws, nb, _stream())
        return rc, o
    check_exact_workspace(L.d3f_grid_subsample_workspace_bytes(N, B), subsample)

    def voxel(ws, nb):
        o = [torch.zeros((N, 3), device="cuda"), torch.zeros((B,), dtype=torch.int32, device="cuda"),
             torch.zeros((1,), dtype=torch.int32, device="cuda"), torch.zeros((1,), dtype=torch.int32, device="cuda")]
        rc = L.d3f_voxel_down_sample(_ptr(pts), _ptr(lens), B, N, None, 0.05, ROOM, _ptr(o[0]), _ptr(o[1]), _ptr(o[2]),
                                     N, _ptr(o[3]), ws, nb, _stream())
        return rc, o
    check_exact_workspace(L.d3f_voxel_down_sample_workspace_bytes(N, B), voxel)

    def neighbors(ws, nb):
        o = [torch.zeros((N,), dtype=torch.int32, device="cuda"), torch.zeros((1,), dtype=torch.int32, device="cuda"),
             torch.zeros((N, 40), dtype=torch.int32, device="cuda")]
        rc = L.d3f_radius_neighbors_build(_ptr(pts), _ptr(lens), B, N, 0.075, ROOM, ws, nb, _stream())
        if rc == 0:
            rc = L.d3f_radius_neighbors_count(_ptr(pts), _ptr(lens), N, _ptr(pts), _ptr(lens), B, N, 0.075, ROOM, ws,
                                              _ptr(o[0]), _ptr(o[1]), _stream())
        if rc == 0:
            rc = L.d3f_radius_neighbors_fill(_ptr(pts), _ptr(lens), N, _ptr(pts), _ptr(lens), B, N, 0.075, ROOM, ws,
                                             40, N, _ptr(o[2]), _stream())
        return rc, o
    check_exact_workspace(L.d3f_radius_neighbors_workspace_bytes(N, B, 0.075, ROOM), neighbors)


def _kpconv_inputs(Nq, Ns, H, K, Cin, Cout, seed=0):
    import torch
    g = torch.Generator().manual_seed(seed)
    q = ((torch.rand((Nq, 3), generator=g) * 2 - 1) * 0.3).cuda()
    s = ((torch.rand((Ns, 3), generator=g) * 2 - 1) * 0.3).cuda()
    idx = torch.randint(0, Ns + 1, (Nq, H), generator=g, dtype=torch.int32).cuda()
    feat = torch.randn((Ns, Cin), generator=g).cuda()
    Kp = (torch.randn((K, 3), generator=g) * 0.03).cuda()
    W = torch.randn((K, Cin, Cout), generator=g).cuda()
    return q, s, idx, feat, Kp, W


KPCONV_SHAPES = [(3000, 3000, 20, 15, 1, 64), (2000, 3000, 20, 15, 32, 64), (1500, 3000, 16, 15, 64, 128)]


def run_kpconv_checks(shapes=KPCONV_SHAPES):
    import torch
    L = _lib.lib()
    for (Nq, Ns, H, K, Cin, Cout) in shapes:
        q, s, idx, feat, Kp, W = _kpconv_inputs(Nq, Ns, H, K, Cin, Cout)
        need = L.d3f_kpconv_workspace_bytes(Nq, Ns, H, K, Cin, Cout)
        # packed weights: the tensor-core contraction and its split-K buffer, the layout's last buffers but one
        Wp = torch.empty((L.d3f_packed_weight_floats(K * Cin, Cout),), dtype=torch.float32, device="cuda")
        assert L.d3f_pack_weight(_ptr(W), K * Cin, Cout, _ptr(Wp), _stream()) == 0
        for deform, packed in [(False, False), (True, False)] + ([(False, True)] if Cin > 1 else []):
            offsets = (torch.randn((Nq, K, 3)) * 0.1).cuda() if deform else None

            def fwd(ws, nb):
                out = torch.zeros((Nq, Cout), device="cuda")
                if deform:
                    rc = L.d3f_kpconv_deform_forward(_ptr(q), _ptr(s), _ptr(idx), _ptr(feat), _ptr(Kp), _ptr(offsets),
                                                     None, _ptr(W), None, None, Nq, Ns, H, K, Cin, Cout, 0.06, 0, 0,
                                                     None, None, None, -1.0, _ptr(out), ws, nb, _stream(), None, None)
                else:
                    rc = L.d3f_kpconv_forward(_ptr(q), _ptr(s), _ptr(idx), _ptr(feat), _ptr(Kp), _ptr(W),
                                              _ptr(Wp) if packed else None, None,
                                              Nq, Ns, H, K, Cin, Cout, 0.06, 0, 0, 1, None, None, None, -1.0,
                                              _ptr(out), ws, nb, _stream(), None, None)
                return rc, [out]
            check_exact_workspace(need, fwd)
        if Cin == 1:
            continue
        dout = torch.randn((Nq, Cout)).cuda()
        width = C.c_int(0)
        wsr = torch.empty((L.d3f_kpconv_backward_workspace_bytes(Nq, Ns, H, K, Cin, Cout, 0),), dtype=torch.uint8,
                          device="cuda")
        assert L.d3f_kpconv_reverse_width(_ptr(idx), Nq, Ns, H, C.byref(width), _ptr(wsr), wsr.numel(), _stream(),
                                          None, None) == 0
        for with_dfeat in (True, False):
            Hr = width.value if with_dfeat else 0

            def bwd(ws, nb):
                dfeat = torch.zeros((Ns, Cin), device="cuda") if with_dfeat else None
                dW = torch.zeros((K, Cin, Cout), device="cuda")
                rc = L.d3f_kpconv_backward(_ptr(q), _ptr(s), _ptr(idx), _ptr(feat), _ptr(Kp), _ptr(W), _ptr(dout), Nq,
                                           Ns, H, Hr, K, Cin, Cout, 0.06, 0, 0, 1, 1, _ptr(dfeat), _ptr(dW), ws, nb,
                                           _stream(), None, None)
                return rc, [t for t in (dfeat, dW) if t is not None]
            check_exact_workspace(L.d3f_kpconv_backward_workspace_bytes(Nq, Ns, H, K, Cin, Cout, Hr), bwd)


@pytest.mark.gpu
def test_kpconv_forward_and_backward_on_exact_workspaces(cuda):
    run_kpconv_checks()


@pytest.mark.gpu
def test_kpconv_fused_image_on_an_exact_workspace(cuda, monkeypatch):
    """The opt-in fused kernel (read per call) packs its weight image into the last buffer of the forward layout."""
    monkeypatch.setenv("D3F_FUSED_KPCONV", "1")
    run_kpconv_checks([(12000, 12000, 20, 15, 32, 32)])


@pytest.mark.gpu
def test_kpconv_multi_chunk_on_exact_workspaces(cuda):
    """The chunk pipeline (D3F_KPCONV_CHUNK is read once per process) in a child process."""
    code = "import sys; sys.path.insert(0, %r); import test_workspace_layouts as t; t.run_kpconv_checks()" % (
        os.path.join(ROOT, "tests"))
    env = dict(os.environ, D3F_KPCONV_CHUNK="512")
    r = subprocess.run([sys.executable, "-c", code], env=env, cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]


@pytest.mark.gpu
def test_training_ops_on_exact_workspaces(cuda):
    import torch
    L = _lib.lib()
    N, C_, Cout = 4000, 64, 32
    g = torch.Generator().manual_seed(3)
    x = torch.randn((N, C_), generator=g).cuda()
    W = torch.randn((C_, Cout), generator=g).cuda()
    dout = torch.randn((N, Cout), generator=g).cuda()

    def unary(ws, nb):
        dx, dW = torch.zeros((N, C_), device="cuda"), torch.zeros((C_, Cout), device="cuda")
        return L.d3f_unary_backward(_ptr(x), _ptr(W), _ptr(dout), N, C_, Cout, 1, _ptr(dx), _ptr(dW), ws, nb,
                                    _stream(), None), [dx, dW]
    check_exact_workspace(L.d3f_unary_backward_workspace_bytes(N, C_, Cout), unary)

    gamma, beta = torch.rand((C_,), generator=g).cuda() + 0.5, torch.randn((C_,), generator=g).cuda()
    for with_gamma in (True, False):
        def bn_fwd(ws, nb):
            o = [torch.zeros((N, C_), device="cuda"), torch.zeros((C_,), device="cuda"),
                 torch.ones((C_,), device="cuda"), torch.zeros((C_,), device="cuda"), torch.zeros((C_,), device="cuda")]
            rc = L.d3f_batch_norm_train_forward(_ptr(x), N, C_, _ptr(gamma) if with_gamma else None, _ptr(beta),
                                                _ptr(o[1]), _ptr(o[2]), 0.98, 1e-5, None, 0.1, _ptr(o[0]), _ptr(o[3]),
                                                _ptr(o[4]), ws, nb, _stream())
            return rc, o
        check_exact_workspace(L.d3f_batch_norm_train_workspace_bytes(N, C_), bn_fwd)
    mean, invstd = x.mean(0).contiguous(), (1 / x.std(0)).contiguous()
    out = torch.randn((N, C_), generator=g).cuda()
    dbn = torch.randn((N, C_), generator=g).cuda()

    def bn_bwd(ws, nb):
        o = [torch.zeros((N, C_), device="cuda"), torch.zeros((C_,), device="cuda"), torch.zeros((C_,), device="cuda")]
        rc = L.d3f_batch_norm_train_backward(_ptr(x), _ptr(out), _ptr(dbn), N, C_, _ptr(gamma), _ptr(mean),
                                             _ptr(invstd), 0.1, _ptr(o[0]), None, _ptr(o[1]), _ptr(o[2]), ws, nb,
                                             _stream())
        return rc, o
    check_exact_workspace(L.d3f_batch_norm_train_workspace_bytes(N, C_), bn_bwd)

    N2, H = 1000, 12
    inds = torch.randint(0, N + 1, (N2, H), generator=g, dtype=torch.int32).cuda()
    pooled = torch.randn((N2, C_), generator=g).cuda()
    dp = torch.randn((N2, C_), generator=g).cuda()

    def maxpool_bwd(ws, nb):
        dx = torch.zeros((N, C_), device="cuda")
        return L.d3f_ind_max_pool_backward(_ptr(x), _ptr(inds), _ptr(pooled), _ptr(dp), N, N2, H, C_, _ptr(dx), ws,
                                           nb, _stream()), [dx]
    check_exact_workspace(L.d3f_ind_max_pool_backward_workspace_bytes(N, N2, H, C_), maxpool_bwd)

    rows = inds[:, 0].contiguous()

    def gather_bwd(ws, nb):
        dx = torch.zeros((N, C_), device="cuda")
        return L.d3f_gather_rows_backward(_ptr(rows), _ptr(dp), N, N2, C_, _ptr(dx), ws, nb, _stream()), [dx]
    check_exact_workspace(L.d3f_gather_rows_backward_workspace_bytes(N, N2), gather_bwd)

    grads = [torch.randn((n,), generator=g).cuda() for n in (1000, 70000, 3)]
    total = sum(t.numel() for t in grads)

    def momentum(ws, nb):
        vs = [torch.ones_like(t) for t in grads]
        acc = [torch.zeros_like(t) for t in grads]
        # the table of tensors lives in device memory: int64 (var, accum, grad, numel) rows
        table = torch.tensor([[v.data_ptr(), a.data_ptr(), t.data_ptr(), t.numel()] for v, a, t in zip(vs, acc, grads)],
                             dtype=torch.int64, device="cuda")
        return L.d3f_momentum_clip_update(_ptr(table), 3, total, 0.01, 0.98, 1.0, ws, nb, _stream()), vs + acc
    check_exact_workspace(L.d3f_momentum_clip_workspace_bytes(3, total), momentum)


@pytest.mark.gpu
def test_keypoints_and_matching_on_exact_workspaces(cuda):
    import torch
    L = _lib.lib()
    N, B, D, k = 5000, 2, 32, 250
    g = torch.Generator().manual_seed(5)
    scores = torch.rand((N,), generator=g).cuda()
    pts = torch.randn((N, 3), generator=g).cuda()
    desc = torch.nn.functional.normalize(torch.randn((N, D), generator=g), dim=1).cuda()
    lens = _lens(3000, 2000)
    for with_k in (True, False):
        def select(ws, nb):
            order = torch.zeros((N,), dtype=torch.int32, device="cuda")
            o = [order]
            if with_k:
                o += [torch.zeros((B, k), dtype=torch.int32, device="cuda"),
                      torch.zeros((B,), dtype=torch.int32, device="cuda"), torch.zeros((B, k, 3), device="cuda"),
                      torch.zeros((B, k, D), device="cuda"), torch.zeros((B, k), device="cuda")]
            p = [_ptr(t) for t in o[1:]] if with_k else [None] * 5
            rc = L.d3f_select_keypoints(_ptr(scores), _ptr(lens), B, N, k if with_k else 0, _ptr(pts), _ptr(desc), D,
                                        _ptr(order), *p, ws, nb, _stream(), None)
            return rc, o
        check_exact_workspace(L.d3f_select_keypoints_workspace_bytes(N, B), select)

    def sample(ws, nb):
        o = [torch.zeros((B, k), dtype=torch.int32, device="cuda"), torch.zeros((B,), dtype=torch.int32, device="cuda")]
        rc = L.d3f_sample_keypoints(_ptr(lens), B, N, k, 7, None, None, 0, None, _ptr(o[0]), _ptr(o[1]), None, None,
                                    None, ws, nb, _stream(), None)
        return rc, o
    check_exact_workspace(L.d3f_sample_keypoints_workspace_bytes(B), sample)

    kd = desc[:B * k].reshape(B, k, D).contiguous()
    count = torch.tensor([k, k - 17], dtype=torch.int32, device="cuda")
    pairs = torch.tensor([[0, 1]], dtype=torch.int32, device="cuda")

    def match(ws, nb):
        o = [torch.zeros((1, k), dtype=torch.int32, device="cuda"), torch.zeros((1, k), device="cuda"),
             torch.zeros((1, k), dtype=torch.int32, device="cuda"), torch.zeros((1, k), device="cuda"),
             torch.zeros((1, k, 2), dtype=torch.int32, device="cuda"), torch.zeros((1,), dtype=torch.int32, device="cuda")]
        rc = L.d3f_match_descriptors(_ptr(kd), _ptr(count), B, k, D, _ptr(pairs), 1, *[_ptr(t) for t in o], ws, nb,
                                     _stream())
        return rc, o
    check_exact_workspace(L.d3f_match_descriptors_workspace_bytes(k, 1), match)


# ---- GPU: the ops whose Python wrappers allocate the workspace ------------------------------------------------------
def _flat(x):
    """Every tensor / array / number of a wrapper's output, in order, on the host."""
    import numpy as np
    import torch
    if torch.is_tensor(x):
        return [x.detach().contiguous().cpu().view(torch.uint8).numpy().tobytes()]
    if isinstance(x, np.ndarray):
        return [x.tobytes()]
    if isinstance(x, dict):
        return [b for k in sorted(x) for b in _flat(x[k])]
    if isinstance(x, (list, tuple)):
        return [b for v in x for b in _flat(v)]
    return [x]


def check_wrapper_workspace(monkeypatch, fn, target=None, flat=_flat):
    """fn() runs an op whose wrapper takes its workspace from `target` (default _lib.workspace(nbytes, device)); every
    workspace it asks for is handed out one byte short, exactly, and twice as large, as in check_exact_workspace."""
    import torch
    owner, name = target or (_lib, "workspace")
    handed = []

    def alloc(mode):
        def ws(*args):
            n = int(args[-2] if owner is _lib else args[-1])
            assert n > 0
            if mode == "double":
                return torch.zeros((2 * n,), dtype=torch.uint8, device="cuda")
            buf = torch.full((n + GUARD,), SENTINEL, dtype=torch.uint8, device="cuda")
            handed.append((buf, n))
            return buf[:n - 1 if mode == "short" else n]
        return ws

    monkeypatch.setattr(owner, name, alloc("short"))
    with pytest.raises(_lib.D3FError, match=r"\(-4\)"):
        fn()
    torch.cuda.synchronize()
    assert handed and all(bool((b == SENTINEL).all()) for b, _ in handed), "a refused call wrote to its workspace"
    handed.clear()
    monkeypatch.setattr(owner, name, alloc("exact"))
    got = flat(fn())
    torch.cuda.synchronize()
    assert handed and all(bool((b[n:] == SENTINEL).all()) for b, n in handed), "an op wrote past its workspace"
    monkeypatch.setattr(owner, name, alloc("double"))
    want = flat(fn())
    assert len(got) == len(want) and all(a == b for a, b in zip(got, want))


@pytest.mark.gpu
def test_pyramid_on_exact_workspaces(cuda, monkeypatch):
    """The 3DMatch spec: every pool radius equals its level's conv radius and every upsample radius the next level's,
    so the build reuses grids; exact (host-synchronising) and static (capacity-sized) forms."""
    import numpy as np
    import torch
    from d3feat_b200 import pyramid as pm
    cfg = synth.Config()
    limits = [40, 30, 34, 35, 35]
    pts = np.concatenate([synth.room_fragment(0, 12000), synth.room_fragment(1, 9000)], 0)
    lens = np.array([12000, 9000], np.int32)
    bbox = np.array([-2, -2, -2, 2, 2, 2], np.float32)
    tp, tl = torch.from_numpy(pts).cuda(), torch.from_numpy(lens).cuda()
    check_wrapper_workspace(monkeypatch, lambda: pm.descriptor_input(cfg, tp, tl, limits, bbox=bbox))

    def static():
        buf = pm.PyramidBuffers(cfg, limits, [24000, 12000, 4000, 1500, 600], 2, "cuda", bbox=bbox)
        buf.points0[:len(pts)].copy_(tp)
        buf.lengths0.copy_(tl)
        buf.n0.fill_(len(pts))
        return pm.descriptor_input(cfg, buf.points0, buf.lengths0, limits, buffers=buf, static=True)

    def static_flat(out):
        n = out["counts"].cpu().tolist()
        assert int(out["status"].item()) == 0
        rows = [out["points"][l][:n[l]] for l in range(cfg.num_layers)]
        rows += [out["neighbors"][l][:n[l]] for l in range(cfg.num_layers)]
        rows += [out["pools"][l][:n[l + 1]] for l in range(cfg.num_layers - 1)]
        rows += [out["upsamples"][l][:n[l]] for l in range(cfg.num_layers - 1)]
        return _flat([n, out["lengths"], rows])
    check_wrapper_workspace(monkeypatch, static, target=(pm.PyramidBuffers, "workspace"), flat=static_flat)


@pytest.mark.gpu
def test_pool_and_detection_ops_on_exact_workspaces(cuda, monkeypatch):
    import torch
    from d3feat_b200 import network_blocks as nb
    from d3feat_b200 import training as tr
    g = torch.Generator().manual_seed(11)
    N, N2, H, C_ = 5000, 1200, 16, 64
    x = torch.randn((N, C_), generator=g).cuda()
    inds = torch.randint(0, N + 1, (N2, H), generator=g, dtype=torch.int32).cuda()
    check_wrapper_workspace(monkeypatch, lambda: nb.ind_max_pool(x, inds))
    feats = torch.relu(torch.randn((N, 32), generator=g)).cuda()
    neighbors = torch.randint(0, N + 1, (N, H), generator=g, dtype=torch.int32).cuda()
    lengths = torch.tensor([3000, 2000], dtype=torch.int32).cuda()
    check_wrapper_workspace(monkeypatch, lambda: nb.detection_scores(feats, neighbors, lengths))
    ds = torch.randn((N, 1), generator=g).cuda()
    check_wrapper_workspace(monkeypatch, lambda: tr.detection_scores_backward(feats, neighbors, lengths, ds))
    # the reverse width reads the table-build phase of the backward layout: exact size of its query, guard intact
    q, s, idx, feat, Kp, W = _kpconv_inputs(2000, 3000, 20, 15, 32, 64)
    L = _lib.lib()

    def width(ws, nb_):
        w = C.c_int(-1)
        rc = L.d3f_kpconv_reverse_width(_ptr(idx), 2000, 3000, 20, C.byref(w), ws, nb_, _stream(), None, None)
        return rc, [torch.tensor([w.value])]
    need = L.d3f_kpconv_backward_workspace_bytes(2000, 3000, 20, 15, 32, 64, 0)
    buf = torch.full((need + GUARD,), SENTINEL, dtype=torch.uint8, device="cuda")
    rc, got = width(buf.data_ptr(), need)
    torch.cuda.synchronize()
    assert rc == 0 and bool((buf[need:] == SENTINEL).all())
    fresh = torch.zeros((2 * need,), dtype=torch.uint8, device="cuda")
    assert width(fresh.data_ptr(), 2 * need)[1][0].item() == got[0].item() > 0


@pytest.mark.gpu
def test_correspondence_ops_on_exact_workspaces(cuda, monkeypatch):
    import numpy as np
    import torch
    import test_gpu_training_data as ttd
    from d3feat_b200 import training_data as td
    from oracle import pairs_np as op
    rng = np.random.default_rng(21)
    pts, lens = ttd._random_case(rng, (900, 700, 1))
    pairs = [[0, 1], [1, 0], [0, 2], [1, 1]]
    trans = [ttd._pose(rng) for _ in pairs]
    args = ttd._dev(cuda, pts, lens, pairs, trans)
    for mode in op.MODES:
        check_wrapper_workspace(monkeypatch, lambda: td.correspondences(*args, 0.0375, mode))
    corr, _, _, anchor = ttd._table(cuda, rng)
    anchor = torch.as_tensor(anchor).to(cuda)
    for replace in (True, False):
        check_wrapper_workspace(monkeypatch, lambda: td.sample_correspondences(corr, 64, replace, 20, 5, anchor))
    pts, lens, pairs, T = ttd._aug_case(rng)
    a = ttd._dev(cuda, pts, lens, pairs, T)
    for kw in ({}, dict(scale=(0.8, 1.2), shift_range=2.0)):
        check_wrapper_workspace(monkeypatch, lambda: td.augment(*a, seed=99, noise=0.01, num_axis=3, **kw))


@pytest.mark.gpu
def test_registration_icp_and_evaluation_on_exact_workspaces(cuda, monkeypatch):
    import numpy as np
    import test_gpu_evaluation as tev
    import test_gpu_icp as tic
    import test_gpu_registration as treg
    rng = np.random.default_rng(31)
    B, k = 4, 300
    pts, _ = treg.scene(rng, B, k)
    pairs = [(0, 1), (1, 2), (2, 3)]
    corr = np.stack([treg.rows(rng, 250, k, k, 0.5) for _ in pairs])
    check_wrapper_workspace(monkeypatch, lambda: treg.register_raw(cuda, pts, [k] * B, corr, [250, 200, 100], pairs,
                                                                   max_iterations=3000, max_validation=300))
    ipts, ilens, ipairs, init = tic.mixed_batch(41)
    check_wrapper_workspace(monkeypatch, lambda: tic.icp_raw(cuda, ipts, ilens, ipairs, init, tic.bbox_of(ipts),
                                                             distance=0.05))
    counts = [0, 1, 249, 250]
    epairs = [(a, b) for a in range(4) for b in range(4)]
    e = tev.make_case(rng, 250, counts, epairs)
    epts, cnt, matches, n_m, G, poses = e
    flags = rng.choice([0, 1, 3, 3], len(epairs))
    for poses_, levels in ((poses, (4, 64, 250)), ([], ())):
        check_wrapper_workspace(monkeypatch, lambda: tev.raw(cuda, epts, cnt, matches, n_m, epairs, G,
                                                             tev.info_matrices(len(epairs)), flags, poses_, levels))
