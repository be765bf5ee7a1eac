"""Mirror of kernels/convolution_ops.py: same function names, argument order and error behaviour, backed by
the fused sm_90a KPConv kernels through the C ABI (include/d3feat_b200.h).

  unary_convolution(features, K_values)                                   convolution_ops.py:90-99
  KPConv(query_points, support_points, neighbors_indices, features, K_values, fixed='center',
         KP_extent=1.0, KP_influence='linear', aggregation_mode='sum')    :102-158
  KPConv_ops(q, s, idx, features, K_points, K_values, KP_extent, KP_influence, aggregation_mode)   :161-255
  KPConv_deformable(..., modulated=False)                                 :258-376
  KPConv_deform_ops(q, s, idx, features, K_points, offsets, modulations, K_values, KP_extent,
                    KP_influence, mode)                                   :379-499

Extensions (keyword-only, default off, so reference call sites work unchanged):
  epilogue=(bn_scale, bn_shift, leaky_alpha)  -- fuse inference batch-norm + LeakyReLU into the kernel
  residual=tensor                             -- (unary only) fused shortcut add before the LeakyReLU

Tensors: contiguous CUDA float32 / int32. The kernel points of a KPConv are a restored, non-trainable
variable in the reference (:145-148); here they come from the active ParamStore under
'<scope>/kernel_points' or, without a store, from the seeded generator in synth.kernel_points.
"""
import os
import weakref

import numpy as np
import torch

from . import _lib
from . import variables as V

# Tensor-core path: static weights are packed once per weight tensor into the K-major TF32 hi/lo images the
# wgmma kernels consume (d3f_pack_weight). D3F_TENSOR_CORES=0 selects the CUDA-core fp32 kernels instead.
USE_TENSOR_CORES = os.environ.get("D3F_TENSOR_CORES", "1") != "0"
_packed_cache = {}     # id(tensor) -> (weakref, version, packed image); entries die with their tensor


def packed_weight(w2d_view_of):
    """Packed image of a weight tensor viewed as [K, N] (unary: [Cin, Cout]; KPConv: [K*Cin, Cout])."""
    if not USE_TENSOR_CORES:
        return None
    w = w2d_view_of
    # keyed by the tensor OBJECT (weak): the entry dies with the tensor, so a recycled device address can never
    # alias a stale image; _version catches in-place updates
    hit = _packed_cache.get(id(w))           # (a hit was checked when it was packed)
    if hit is not None and hit[0]() is w and hit[1] == w._version:
        return hit[2]
    w = _lib.tensor_arg(w, "packed_weight: weights", _F32)
    if w.dim() < 2:
        raise ValueError("packed_weight: weights must be [..., K, N], got %s" % (tuple(w.shape),))
    K = int(np.prod(w.shape[:-1]))
    N = int(w.shape[-1])
    L = _lib.lib()
    packed = torch.empty((L.d3f_packed_weight_floats(K, N),), dtype=torch.float32, device=w.device)
    _lib.check(L.d3f_pack_weight(_lib.ptr(w), K, N, _lib.ptr(packed), _lib.stream()), "d3f_pack_weight")
    if not _lib.publish_ready(w.device):
        return packed
    if hit is None or hit[0]() is not w:
        weakref.finalize(w, _packed_cache.pop, id(w), None)
    _packed_cache[id(w)] = (weakref.ref(w), w._version, packed)
    return packed


_F32, _I32 = torch.float32, torch.int32

_INFLUENCE = {"constant": 0, "linear": 1, "gaussian": 2}
_MODE = {"sum": 0, "closest": 1}


def _epilogue_args(epilogue, op, Cout, device):
    if epilogue is None:
        return None, None, -1.0
    scale, shift, alpha = epilogue
    scale = _lib.tensor_arg(scale, op + ": epilogue scale", _F32, (Cout,), device)
    shift = _lib.tensor_arg(shift, op + ": epilogue shift", _F32, (Cout,), device)
    return scale, shift, (-1.0 if alpha is None else float(alpha))


def unary_convolution(features, K_values, *, epilogue=None, residual=None, rows=None):
    """features[N,Cin] @ K_values[Cin,Cout] (tf.matmul, :90-99).
    rows (extension): int32 device scalar holding the actual row count when `features` is a capacity-sized buffer."""
    op = "unary_convolution"
    x = _lib.tensor_arg(features, op + ": features", _F32, (None, None))
    dev = x.device
    N, Cin = x.shape
    w = _lib.tensor_arg(K_values, op + ": K_values", _F32, (Cin, None), dev)
    Cout = w.shape[1]
    scale, shift, alpha = _epilogue_args(epilogue, op, Cout, dev)
    res = _lib.tensor_arg(residual, op + ": residual", _F32, (N, Cout), dev, optional=True)
    rows = _lib.row_count_arg(rows, op + ": rows", dev)
    out = torch.empty((N, Cout), dtype=torch.float32, device=dev)
    _lib.check(_lib.lib().d3f_unary_forward(_lib.ptr(x), _lib.ptr(w), _lib.ptr(packed_weight(w)), N, Cin, Cout, _lib.ptr(scale), _lib.ptr(shift),
                                            None, _lib.ptr(res), alpha, _lib.ptr(out), _lib.stream(), _lib.ptr(rows)),
               "d3f_unary_forward")
    return out


def _aligned16(t):
    return t.data_ptr() % 16 == 0


# (id(w1), id(w2)) -> (refs and versions of w1, w2, s1, s2, t1, t2, packed image of the folded [w1*s1 ; w2*s2],
# shift1 + shift2)
_pair_cache = {}


def unary_pair_convolution(x1, w1, affine1, x2, w2, affine2, alpha, *, rows=None):
    """leaky((x1 @ w1) * s1 + t1 + (x2 @ w2) * s2 + t2) as ONE GEMM over the concatenated K -- the conv3 + shortcut
    + add + LeakyReLU tail of a resnetb block (models/network_blocks.py:343-368). affine = (scale, shift) of the
    unary's inference batch norm. The scales are folded into the weights once per weight pair (float64), so neither
    the shortcut tensor nor [x1 | x2] exists in memory. Falls back to two unary_convolution calls without the
    tensor-core path, when the channel counts do not tile, or when x1 or x2 does not start on a 16-byte boundary (the
    one-GEMM kernel fetches both by TMA; a lone unary_convolution then runs its CUDA-core GEMM on that operand)."""
    op = "unary_pair_convolution"
    x1 = _lib.tensor_arg(x1, op + ": x1", _F32, (None, None))
    dev = x1.device
    N, C1 = x1.shape
    x2 = _lib.tensor_arg(x2, op + ": x2", _F32, (N, None), dev)
    C2 = int(x2.shape[1])
    w1 = _lib.tensor_arg(w1, op + ": w1", _F32, (C1, None), dev)
    Cout = int(w1.shape[1])
    w2 = _lib.tensor_arg(w2, op + ": w2", _F32, (C2, Cout), dev)
    (s1, t1), (s2, t2) = affine1, affine2
    s1, t1, s2, t2 = (_lib.tensor_arg(v, "%s: affine%s" % (op, n), _F32, (Cout,), dev)
                      for v, n in ((s1, "1 scale"), (t1, "1 shift"), (s2, "2 scale"), (t2, "2 shift")))
    rows = _lib.row_count_arg(rows, op + ": rows", dev)
    if not USE_TENSOR_CORES or C1 % 32 != 0 or C2 % 4 != 0 or not (_aligned16(x1) and _aligned16(x2)):
        shortcut = unary_convolution(x2, w2, epilogue=(s2, t2, None), rows=rows)
        return unary_convolution(x1, w1, epilogue=(s1, t1, alpha), residual=shortcut, rows=rows)
    key = (id(w1), id(w2))
    hit = _pair_cache.get(key)
    args = (w1, w2, s1, s2, t1, t2)
    vers = tuple(a._version for a in args)
    # the fold reads all six tensors: a new affine of other values at version 0 must not reuse an old fold
    if hit is None or any(r() is not a for r, a in zip(hit[0], args)) or hit[1] != vers:
        folded = torch.cat([w1.double() * s1.double()[None, :], w2.double() * s2.double()[None, :]], 0).float()
        shift = (t1.double() + t2.double()).float().contiguous()
        L = _lib.lib()
        packed = torch.empty((L.d3f_packed_weight_floats(C1 + C2, Cout),), dtype=torch.float32, device=w1.device)
        _lib.check(L.d3f_pack_weight(_lib.ptr(folded.contiguous()), C1 + C2, Cout, _lib.ptr(packed), _lib.stream()),
                   "d3f_pack_weight")
        fresh = hit is None
        hit = (tuple(weakref.ref(a) for a in args), vers, packed, shift)
        if _lib.publish_ready(dev):
            if fresh:
                weakref.finalize(w1, _pair_cache.pop, key, None)
            _pair_cache[key] = hit
    out = torch.empty((N, Cout), dtype=torch.float32, device=x1.device)
    _lib.check(_lib.lib().d3f_unary_pair_forward(_lib.ptr(x1), C1, _lib.ptr(x2), C2, _lib.ptr(hit[2]), N, Cout,
                                                 _lib.ptr(hit[3]), -1.0 if alpha is None else float(alpha),
                                                 _lib.ptr(out), _lib.stream(), _lib.ptr(rows)), "d3f_unary_pair_forward")
    return out


def _check_enums(KP_influence, aggregation_mode):
    if KP_influence not in _INFLUENCE:
        raise ValueError("Unknown influence function type (config.KP_influence)")          # :224, :469
    if aggregation_mode not in _MODE:
        raise ValueError("Unknown convolution mode. Should be 'closest' or 'sum'")         # :232, :477


def _kpconv_args(op, query_points, support_points, neighbors_indices, features, K_points, K_values, query_order,
                 rows_q, rows_s):
    """The tensor arguments both KPConv ops share, checked against each other (ValueError) and contiguous."""
    q = _lib.tensor_arg(query_points, op + ": query_points", _F32, (None, 3))
    dev = q.device
    Nq = q.shape[0]
    s = _lib.tensor_arg(support_points, op + ": support_points", _F32, (None, 3), dev)
    Ns = s.shape[0]
    idx = _lib.tensor_arg(neighbors_indices, op + ": neighbors_indices", _I32, (Nq, None), dev)
    f = _lib.tensor_arg(features, op + ": features", _F32, (Ns, None), dev)
    W = _lib.tensor_arg(K_values, op + ": K_values", _F32, (None, f.shape[1], None), dev)
    Kp = _lib.tensor_arg(K_points, op + ": K_points", _F32, (W.shape[0], 3), dev)
    order = _lib.tensor_arg(query_order, op + ": query_order", _I32, (Nq,), dev, optional=True)
    return (q, s, idx, f, Kp, W, order, _lib.row_count_arg(rows_q, op + ": rows_q", dev),
            _lib.row_count_arg(rows_s, op + ": rows_s", dev))


def KPConv_ops(query_points, support_points, neighbors_indices, features, K_points, K_values, KP_extent,
               KP_influence, aggregation_mode, *, epilogue=None, bias=None, query_order=None, rows_q=None,
               rows_s=None):
    """Rigid KPConv (:161-255): one fused launch sequence, no [N,H,K,*] intermediates.
    query_order (extension): int32[Nq] visiting order of the queries (hash-grid cell order from the pyramid);
    a pure scheduling hint -- every query still writes its own output row.
    rows_q / rows_s (extension): int32 device scalars with the actual query / support counts when the tensors are
    capacity-sized buffers (the shadow index is then the actual support count)."""
    _check_enums(KP_influence, aggregation_mode)
    op = "KPConv_ops"
    q, s, idx, f, Kp, W, query_order, rows_q, rows_s = _kpconv_args(
        op, query_points, support_points, neighbors_indices, features, K_points, K_values, query_order, rows_q, rows_s)
    Nq, Ns, H = q.shape[0], s.shape[0], idx.shape[1]
    K, Cin, Cout = W.shape
    scale, shift, alpha = _epilogue_args(epilogue, op, Cout, q.device)
    bias = _lib.tensor_arg(bias, op + ": bias", _F32, (Cout,), q.device, optional=True)
    L = _lib.lib()
    ws = _lib.workspace(L.d3f_kpconv_workspace_bytes(Nq, Ns, H, K, Cin, Cout), q.device)
    out = torch.empty((Nq, Cout), dtype=torch.float32, device=q.device)
    _lib.check(L.d3f_kpconv_forward(_lib.ptr(q), _lib.ptr(s), _lib.ptr(idx), _lib.ptr(f), _lib.ptr(Kp), _lib.ptr(W),
                                    _lib.ptr(packed_weight(W)), _lib.ptr(query_order), Nq, Ns, H, K, Cin, Cout, float(KP_extent), _INFLUENCE[KP_influence],
                                    _MODE[aggregation_mode], 1, _lib.ptr(scale), _lib.ptr(shift), _lib.ptr(bias),
                                    alpha, _lib.ptr(out), _lib.ptr(ws), ws.numel(), _lib.stream(), _lib.ptr(rows_q),
                                    _lib.ptr(rows_s)),
               "d3f_kpconv_forward")
    return out


def KPConv_deform_ops(query_points, support_points, neighbors_indices, features, K_points, offsets, modulations,
                      K_values, KP_extent, KP_influence, mode, *, epilogue=None, query_order=None, rows_q=None,
                      rows_s=None):
    """Deformable second stage (:379-499)."""
    _check_enums(KP_influence, mode)
    op = "KPConv_deform_ops"
    q, s, idx, f, Kp, W, query_order, rows_q, rows_s = _kpconv_args(
        op, query_points, support_points, neighbors_indices, features, K_points, K_values, query_order, rows_q, rows_s)
    Nq, Ns, H = q.shape[0], s.shape[0], idx.shape[1]
    K, Cin, Cout = W.shape
    off = _lib.tensor_arg(offsets, op + ": offsets", _F32, (Nq, K, 3), q.device)
    mod = _lib.tensor_arg(modulations, op + ": modulations", _F32, (Nq, K), q.device, optional=True)
    scale, shift, alpha = _epilogue_args(epilogue, op, Cout, q.device)
    L = _lib.lib()
    ws = _lib.workspace(L.d3f_kpconv_workspace_bytes(Nq, Ns, H, K, Cin, Cout), q.device)
    out = torch.empty((Nq, Cout), dtype=torch.float32, device=q.device)
    _lib.check(L.d3f_kpconv_deform_forward(_lib.ptr(q), _lib.ptr(s), _lib.ptr(idx), _lib.ptr(f), _lib.ptr(Kp),
                                           _lib.ptr(off), _lib.ptr(mod), _lib.ptr(W), _lib.ptr(packed_weight(W)), _lib.ptr(query_order), Nq, Ns, H, K, Cin, Cout,
                                           float(KP_extent), _INFLUENCE[KP_influence], _MODE[mode], _lib.ptr(scale),
                                           _lib.ptr(shift), None, alpha, _lib.ptr(out), _lib.ptr(ws), ws.numel(),
                                           _lib.stream(), _lib.ptr(rows_q), _lib.ptr(rows_s)),
               "d3f_kpconv_deform_forward")
    return out


def _kernel_points(K_radius, num_kpoints, device, fixed):
    store = V.current_store()
    name = V.scoped("kernel_points")
    if store is not None and name in store:
        return store.get(name)
    if store is not None and len(store) > 0:
        # a checkpoint is active but lacks this KPConv's saved disposition: never synthesise silently
        raise KeyError("kernel points '%s' missing from the active ParamStore" % name)
    # no checkpoint at all: seeded stand-in for kernels/kernel_points.py:184-280 (random rotation + 1 % noise). The
    # seed is a stable hash of the variable name, so every process and every rank draws the same points.
    import zlib
    from .synth import kernel_points
    seed = zlib.crc32(name.encode("utf-8")) & 0x7FFFFFFF
    return torch.from_numpy(kernel_points(np.random.default_rng(seed), K_radius, num_kpoints)).to(device)


def KPConv(query_points, support_points, neighbors_indices, features, K_values, fixed="center", KP_extent=1.0,
           KP_influence="linear", aggregation_mode="sum", *, epilogue=None, query_order=None, rows_q=None,
           rows_s=None):
    """:102-158 -- kernel-point disposition of radius 1.5*KP_extent, then KPConv_ops."""
    K_radius = 1.5 * KP_extent
    num_kpoints = int(K_values.shape[0])
    K_points = _kernel_points(K_radius, num_kpoints, query_points.device, fixed)
    return KPConv_ops(query_points, support_points, neighbors_indices, features, K_points, K_values, KP_extent,
                      KP_influence, aggregation_mode, epilogue=epilogue, query_order=query_order, rows_q=rows_q,
                      rows_s=rows_s)


def KPConv_deformable(query_points, support_points, neighbors_indices, features, K_values, fixed="center",
                      KP_extent=1.0, KP_influence="linear", aggregation_mode="sum", modulated=False, *,
                      epilogue=None, query_order=None, rows_q=None, rows_s=None):
    """:258-376 -- rigid KPConv producing 3K (4K if modulated) offsets (+ bias), then the deformed conv."""
    K_radius = 1.5 * KP_extent
    num_kpoints = int(K_values.shape[0])
    points_dim = int(query_points.shape[1])
    K_points = _kernel_points(K_radius, num_kpoints, query_points.device, fixed)
    store = V.current_store()
    offset_dim = (points_dim + 1) * num_kpoints if modulated else points_dim * num_kpoints
    w0_name, b0_name = V.scoped("offset_conv_weights"), V.scoped("offset_conv_bias")
    if store is not None and w0_name in store:
        K_values0, b0 = store.get(w0_name), store.get(b0_name)
    else:                                                    # the reference initialises both to zero (:327-328)
        K_values0 = torch.zeros((num_kpoints, K_values.shape[1], offset_dim), device=query_points.device)
        b0 = torch.zeros((offset_dim,), device=query_points.device)
    features0 = KPConv_ops(query_points, support_points, neighbors_indices, features, K_points, K_values0, KP_extent,
                           KP_influence, aggregation_mode, bias=b0, query_order=query_order, rows_q=rows_q,
                           rows_s=rows_s)
    if modulated:
        offsets = features0[:, :points_dim * num_kpoints].reshape(-1, num_kpoints, points_dim)
        modulations = 2 * torch.sigmoid(features0[:, points_dim * num_kpoints:])
    else:
        offsets = features0.reshape(-1, num_kpoints, points_dim)
        modulations = None
    offsets = offsets * KP_extent
    return KPConv_deform_ops(query_points, support_points, neighbors_indices, features, K_points, offsets,
                             modulations, K_values, KP_extent, KP_influence, aggregation_mode, epilogue=epilogue,
                             query_order=query_order, rows_q=rows_q, rows_s=rows_s)
