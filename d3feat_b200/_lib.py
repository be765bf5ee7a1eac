"""ctypes binding of libd3feat_b200.so (the C ABI of include/d3feat_b200.h).

There is no CPU fallback and no second backend: if the shared library is missing or a call fails the
error is raised here. PyTorch tensors are only containers for device memory; every call is enqueued on
torch's current CUDA stream.
"""
import ctypes as C
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
# D3F_LIB: alternative build of the same library (kernel-tuning experiments); never a different backend
LIB_PATH = os.environ.get("D3F_LIB") or os.path.join(_HERE, "libd3feat_b200.so")

# every symbol include/d3feat_b200.h declares: (name, restype, argtypes)
_P, _I, _F, _Z, _LL = C.c_void_p, C.c_int, C.c_float, C.c_size_t, C.c_longlong
_D, _U64 = C.c_double, C.c_uint64
SYMBOLS = [
    ("d3f_version", _I, []),
    ("d3f_last_error", C.c_char_p, []),
    ("d3f_launch_count", _LL, []),
    ("d3f_bbox", _I, [_P, _I, _P, _P]),
    ("d3f_grid_subsample_workspace_bytes", _Z, [_I, _I]),
    ("d3f_grid_subsample", _I, [_P, _P, _I, _I, _F, _P, _I, _P, _I, _P, _P, _P, _P, _P, _P, _P, _Z, _P]),
    ("d3f_voxel_down_sample_workspace_bytes", _Z, [_I, _I]),
    ("d3f_voxel_down_sample", _I, [_P, _P, _I, _I, _P, _D, _P, _P, _P, _P, _I, _P, _P, _Z, _P]),
    ("d3f_radius_neighbors_workspace_bytes", _Z, [_I, _I, _F, _P]),
    ("d3f_radius_neighbors_build", _I, [_P, _P, _I, _I, _F, _P, _P, _Z, _P]),
    ("d3f_radius_neighbors_count", _I, [_P, _P, _I, _P, _P, _I, _I, _F, _P, _P, _P, _P, _P]),
    ("d3f_radius_neighbors_fill", _I, [_P, _P, _I, _P, _P, _I, _I, _F, _P, _P, _I, _I, _P, _P]),
    ("d3f_kpconv_workspace_bytes", _Z, [_I, _I, _I, _I, _I, _I]),
    ("d3f_pyramid_workspace_bytes", _Z, [_I, _P, _P, _P]),
    ("d3f_pyramid_build", _I, [_P, _P, _I, _I, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _Z, _P, _P, _P, _P]),
    ("d3f_packed_weight_floats", _Z, [_I, _I]),
    ("d3f_pack_weight", _I, [_P, _I, _I, _P, _P]),
    ("d3f_radius_neighbors_order", _I, [_P, _I, _I, _F, _P, _P, _P]),
    ("d3f_kpconv_forward", _I, [_P, _P, _P, _P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _F, _I, _I, _I, _P, _P, _P, _F, _P,
                                _P, _Z, _P, _P, _P]),
    ("d3f_kpconv_deform_forward", _I, [_P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _F, _I, _I, _P, _P,
                                       _P, _F, _P, _P, _Z, _P, _P, _P]),
    ("d3f_unary_forward", _I, [_P, _P, _P, _I, _I, _I, _P, _P, _P, _P, _F, _P, _P, _P]),
    ("d3f_kpconv_backward_workspace_bytes", _Z, [_I, _I, _I, _I, _I, _I, _I]),
    ("d3f_kpconv_reverse_width", _I, [_P, _I, _I, _I, C.POINTER(C.c_int), _P, _Z, _P, _P, _P]),
    ("d3f_kpconv_backward", _I, [_P, _P, _P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _I, _F, _I, _I, _I, _I, _P, _P, _P,
                                 _Z, _P, _P, _P]),
    ("d3f_unary_backward_workspace_bytes", _Z, [_I, _I, _I]),
    ("d3f_unary_backward", _I, [_P, _P, _P, _I, _I, _I, _I, _P, _P, _P, _Z, _P, _P]),
    ("d3f_ind_max_pool_workspace_bytes", _Z, [_I]),
    ("d3f_ind_max_pool", _I, [_P, _P, _I, _I, _I, _I, _P, _P, _Z, _P, _P, _P]),
    ("d3f_closest_pool", _I, [_P, _P, _I, _I, _I, _I, _P, _P, _P, _P]),
    ("d3f_l2_normalize", _I, [_P, _I, _I, _F, _P, _P, _P]),
    ("d3f_unary_pair_forward", _I, [_P, _I, _P, _I, _P, _I, _I, _P, C.c_float, _P, _P, _P]),
    ("d3f_detection_scores_workspace_bytes", _Z, [_I, _I]),
    ("d3f_detection_scores", _I, [_P, _P, _P, _I, _I, _I, _I, _P, _P, _Z, _P, _P]),
    ("d3f_affine_leaky", _I, [_P, _I, _I, _P, _P, _P, _F, _P, _P, _P]),
    ("d3f_batch_norm_train_workspace_bytes", _Z, [_I, _I]),
    ("d3f_batch_norm_train_forward", _I, [_P, _I, _I, _P, _P, _P, _P, _F, _F, _P, _F, _P, _P, _P, _P, _Z, _P]),
    ("d3f_batch_norm_train_backward", _I, [_P, _P, _P, _I, _I, _P, _P, _P, _F, _P, _P, _P, _P, _P, _Z, _P]),
    ("d3f_ind_max_pool_backward_workspace_bytes", _Z, [_I, _I, _I, _I]),
    ("d3f_ind_max_pool_backward", _I, [_P, _P, _P, _P, _I, _I, _I, _I, _P, _P, _Z, _P]),
    ("d3f_gather_rows_backward_workspace_bytes", _Z, [_I, _I]),
    ("d3f_gather_rows_backward", _I, [_P, _P, _I, _I, _I, _P, _P, _Z, _P]),
    ("d3f_l2_normalize_backward", _I, [_P, _P, _I, _I, _F, _P, _P]),
    ("d3f_detection_scores_backward_workspace_bytes", _Z, [_I, _I, _I, _I]),
    ("d3f_detection_scores_backward", _I, [_P, _P, _P, _P, _I, _I, _I, _I, _P, _P, _Z, _P]),
    ("d3f_select_keypoints_workspace_bytes", _Z, [_I, _I]),
    ("d3f_select_keypoints", _I, [_P, _P, _I, _I, _I, _P, _P, _I, _P, _P, _P, _P, _P, _P, _P, _Z, _P, _P]),
    ("d3f_sample_keypoints_workspace_bytes", _Z, [_I]),
    ("d3f_sample_keypoints", _I, [_P, _I, _I, _I, _U64, _P, _P, _I, _P, _P, _P, _P, _P, _P, _P, _Z, _P, _P]),
    ("d3f_match_descriptors_workspace_bytes", _Z, [_I, _I]),
    ("d3f_match_descriptors", _I, [_P, _P, _I, _I, _I, _P, _I, _P, _P, _P, _P, _P, _P, _P, _Z, _P]),
    ("d3f_register_pairs_workspace_bytes", _Z, [_I, _I, _I, _I]),
    ("d3f_register_pairs", _I, [_P, _P, _I, _I, _P, _P, _I, _P, _I, _I, _I, _I, _D, _D, _U64, _P, _P, _P, _P, _P, _Z,
                                _P]),
    ("d3f_icp_pairs_workspace_bytes", _Z, [_I, _I, _I, _D, _P]),
    ("d3f_icp_pairs", _I, [_P, _P, _I, _I, _P, _P, _P, _I, _P, _D, _I, _D, _D, _P, _P, _P, _P, _P, _P, _Z, _P]),
    ("d3f_pair_correspondences_workspace_bytes", _Z, [_I, _I, _I, _D, _P]),
    ("d3f_pair_correspondences_count", _I, [_P, _P, _I, _I, _P, _P, _I, _P, _D, _I, _P, _P, _P, _P, _Z, _P]),
    ("d3f_pair_correspondences_fill", _I, [_P, _I, _I, _P, _P, _I, _P, _D, _I, _I, _P, _P, _Z, _P]),
    ("d3f_sample_correspondences_workspace_bytes", _Z, [_I, _I]),
    ("d3f_sample_correspondences", _I, [_P, _P, _I, _I, _P, _I, _I, _I, _U64, _P, _P, _P, _P, _Z, _P]),
    ("d3f_augment_pairs_workspace_bytes", _Z, [_I, _I]),
    ("d3f_augment_pairs", _I, [_P, _P, _I, _I, _P, _I, _P, _U64, _D, _I, _I, _D, _D, _D, _I, _P, _P, _P, _P, _P, _P, _P,
                               _P, _Z, _P]),
    ("d3f_evaluate_pairs_workspace_bytes", _Z, [_I, _I]),
    ("d3f_evaluate_pairs", _I, [_P, _P, _I, _I, _P, _P, _I, _P, _I, _P, _P, _P, _P, _I, _P, _I, _D, _D, _D, _D, _D, _D,
                                _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _Z, _P]),
    ("d3f_momentum_clip_workspace_bytes", _Z, [_I, _LL]),
    ("d3f_momentum_clip_update", _I, [_P, _I, _LL, _F, _F, _F, _P, _Z, _P]),
    ("d3f_rank_mean", _I, [_P, _I, _LL, _P, _P]),
    ("d3f_kernel_point_optimize", _I, [_P, _I, _I, _I, _I, _P, _P, _P, _P]),
]

_lib = None


class D3FError(RuntimeError):
    pass


def lib():
    """Load the library (once). Raises if it has not been built: there is no fallback path."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise D3FError(
                "libd3feat_b200.so is missing at %s -- build it with `python -c 'import __graft_entry__ as g; "
                "g.build()'` (nvcc, sm_90a). d3feat_b200 has no CPU or PyTorch fallback." % LIB_PATH)
        l = C.CDLL(LIB_PATH)
        for name, res, args in SYMBOLS:
            fn = getattr(l, name)  # AttributeError if the .so does not export a declared symbol
            fn.restype = res
            fn.argtypes = args
        _lib = l
    return _lib


def check(rc, what):
    if rc != 0:
        msg = lib().d3f_last_error().decode("utf-8", "replace")
        if rc == -1:
            raise ValueError("%s: %s" % (what, msg))
        raise D3FError("%s failed (%d): %s" % (what, rc, msg))


def stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def ptr(t):
    """Device (or host) address of a contiguous tensor; None -> NULL."""
    if t is None:
        return None
    assert t.is_contiguous(), "tensor must be contiguous"
    return C.c_void_p(t.data_ptr())


DEVICE_TYPE = "cuda"     # where the kernels read their arguments


def _describe(t):
    if not torch.is_tensor(t):
        return type(t).__name__
    return "%s %s on %s" % (str(t.dtype).replace("torch.", ""), list(t.shape), t.device)


def tensor_arg(t, name, dtype, shape=None, device=None, optional=False):
    """The tensor argument `name` ("<op>: <argument>") of a hot-path op, contiguous, or ValueError: it must be a
    `dtype` tensor on a CUDA device (`device`, when the call has already seen a tensor) whose shape matches `shape`,
    a tuple with None for a free dimension. Nothing is converted: a silent .to(int32) here would be a hidden copy per
    call, and a wrong dtype or a host address read by a kernel is a wrong result or a fault. Only attributes are read
    (no launch, no synchronisation); .contiguous() copies a strided view and returns anything else as it is."""
    if t is None and optional:
        return None
    ok = torch.is_tensor(t) and t.dtype == dtype
    if ok:
        dev = t.device
        ok = dev.type == DEVICE_TYPE and (device is None or dev == device)
    if ok and shape is not None:
        got = t.shape
        ok = len(got) == len(shape) and all(e is None or e == g for e, g in zip(shape, got))
    if not ok:
        want = "" if shape is None else " of shape [%s]" % ", ".join("*" if e is None else str(int(e)) for e in shape)
        raise ValueError("%s must be a %s CUDA tensor%s%s, got %s" % (
            name, str(dtype).replace("torch.", ""), want, "" if device is None else " on %s" % device, _describe(t)))
    return t.contiguous()


def row_count_arg(t, name, device):
    """An optional device row count: one int32 element (tensor_arg otherwise)."""
    t = tensor_arg(t, name, torch.int32, None, device, optional=True)
    if t is not None and t.numel() != 1:
        raise ValueError("%s must hold one int32 element, got %s" % (name, _describe(t)))
    return t


def publish_ready(device):
    """Whether a lazily computed cache entry (packed weight image, folded batch norm) that the current stream has just
    been given to produce may be published. A later hit uses the entry from any thread and stream with no ordering
    against its producer, so the producer must have finished: the current stream is synchronised once, on the miss,
    and a hit never waits. While the current stream is captured into a CUDA graph the entry only exists once the graph
    has been replayed: False, and the caller uses it for this call without publishing it (the graph then carries the
    producer; an eager warm-up before the capture keeps it out)."""
    if device.type != "cuda":
        return True
    if torch.cuda.is_current_stream_capturing():
        return False
    torch.cuda.current_stream(device).synchronize()
    return True


def workspace(nbytes, device):
    return torch.empty((max(int(nbytes), 256),), dtype=torch.uint8, device=device)


def f32(t, device):
    if not torch.is_tensor(t):
        t = torch.as_tensor(t, dtype=torch.float32)
    return t.to(device=device, dtype=torch.float32).contiguous()


def i32(t, device):
    if not torch.is_tensor(t):
        t = torch.as_tensor(t, dtype=torch.int32)
    return t.to(device=device, dtype=torch.int32).contiguous()


def launch_count():
    return int(lib().d3f_launch_count())
