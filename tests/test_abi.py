"""CPU: the C-ABI shared library loads and exports every symbol include/d3feat_b200.h declares, and the
Python binding table covers exactly that set (no compute calls: there is no GPU here)."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "d3feat_b200.h")


def header_symbols():
    src = open(HEADER).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(d3f_[a-z0-9_]+)\s*\(", src)))


@pytest.fixture(scope="module")
def built_lib():
    from d3feat_b200 import build
    path = build.build()
    return ctypes.CDLL(path)


def test_header_declares_the_expected_entry_points():
    syms = header_symbols()
    for must in ("d3f_grid_subsample", "d3f_radius_neighbors_build", "d3f_radius_neighbors_count",
                 "d3f_radius_neighbors_fill", "d3f_kpconv_forward", "d3f_kpconv_deform_forward",
                 "d3f_unary_forward", "d3f_ind_max_pool", "d3f_closest_pool", "d3f_last_error"):
        assert must in syms


def test_library_exports_every_declared_symbol(built_lib):
    for s in header_symbols():
        assert hasattr(built_lib, s), "libd3feat_b200.so does not export %s" % s


def test_binding_table_matches_header(built_lib):
    from d3feat_b200 import _lib
    bound = sorted(n for n, _, _ in _lib.SYMBOLS)
    assert bound == header_symbols()
    _lib.lib()          # binds argtypes / restypes for all of them
    assert _lib.lib().d3f_version() >= 100
    assert _lib.launch_count() == 0


def test_invalid_arguments_return_codes_without_a_gpu(built_lib):
    """Argument validation happens before any CUDA call, so it can be exercised on the CPU box."""
    built_lib.d3f_last_error.restype = ctypes.c_char_p
    built_lib.d3f_kpconv_forward.restype = ctypes.c_int
    rc = built_lib.d3f_unary_forward(None, None, None, ctypes.c_int(-1), ctypes.c_int(4), ctypes.c_int(4), None, None,
                                     None, None, ctypes.c_float(-1.0), None, None, None)
    assert rc == -1
    assert b"bad shape" in built_lib.d3f_last_error()
    built_lib.d3f_radius_neighbors_workspace_bytes.restype = ctypes.c_size_t
    assert built_lib.d3f_radius_neighbors_workspace_bytes(ctypes.c_int(10), ctypes.c_int(1), ctypes.c_float(0.1),
                                                          None) == 0


@pytest.mark.parametrize("B", [0, 1025])
def test_batch_size_checked_before_any_cuda_call(built_lib, B):
    """Grid subsampling, the radius-neighbour build / count / fill and the pyramid take 1 to 1024 clouds; any other
    number is refused before a kernel or a CUDA call (the pointers are never dereferenced)."""
    from d3feat_b200._lib import SYMBOLS
    lib = built_lib
    lib.d3f_last_error.restype = ctypes.c_char_p
    names = ("d3f_grid_subsample", "d3f_radius_neighbors_build", "d3f_radius_neighbors_count",
             "d3f_radius_neighbors_fill", "d3f_pyramid_build")
    for name in names:
        fn = getattr(lib, name)
        fn.restype, fn.argtypes = [(r, a) for n, r, a in SYMBOLS if n == name][0]
    fake = ctypes.c_void_p(256)
    bbox = (ctypes.c_float * 6)(0, 0, 0, 1, 1, 1)
    ptrs = (ctypes.c_void_p * 8)()
    caps = (ctypes.c_int * 8)(*([100] * 8))
    calls = {
        "d3f_grid_subsample": lambda: lib.d3f_grid_subsample(fake, fake, B, 100, 0.1, None, 0, None, 0, bbox, fake, None,
                                                             None, fake, fake, fake, 1 << 30, None),
        "d3f_radius_neighbors_build": lambda: lib.d3f_radius_neighbors_build(fake, fake, B, 100, 0.1, bbox, fake, 1 << 30,
                                                                             None),
        "d3f_radius_neighbors_count": lambda: lib.d3f_radius_neighbors_count(fake, fake, 100, fake, fake, B, 100, 0.1,
                                                                             bbox, fake, fake, fake, None),
        # zero columns: nothing to write, but the batch size is still checked
        "d3f_radius_neighbors_fill": lambda: lib.d3f_radius_neighbors_fill(fake, fake, 100, fake, fake, B, 100, 0.1, bbox,
                                                                           fake, 0, 100, fake, None),
        "d3f_pyramid_build": lambda: lib.d3f_pyramid_build(fake, fake, B, 100, fake, bbox, ptrs, ptrs, ptrs, ptrs, ptrs,
                                                           caps, None, fake, 1 << 30, None, fake, fake, None),
    }
    for name in names:
        assert calls[name]() == -1, name
        assert (b"B=%d" % B) in lib.d3f_last_error(), (name, lib.d3f_last_error())


def test_missing_library_fails_loudly(monkeypatch, tmp_path):
    from d3feat_b200 import _lib
    monkeypatch.setattr(_lib, "_lib", None)
    monkeypatch.setattr(_lib, "LIB_PATH", str(tmp_path / "nope.so"))
    with pytest.raises(_lib.D3FError):
        _lib.lib()
