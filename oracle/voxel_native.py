"""TEST INFRASTRUCTURE ONLY -- ctypes access to the C restatement of voxel down-sampling (oracle/voxel_oracle.c),
compiled into oracle/libvoxel_oracle.so with the flags of oracle/Makefile (-O2 -ffp-contract=off). Not part of the
product path."""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "voxel_oracle.c")
_LIB = os.path.join(_HERE, "libvoxel_oracle.so")

_f32p = np.ctypeslib.ndpointer(np.float32, flags="C_CONTIGUOUS")
_i32p = np.ctypeslib.ndpointer(np.int32, flags="C_CONTIGUOUS")


def build():
    if os.path.exists(_LIB) and os.path.getmtime(_LIB) >= os.path.getmtime(_SRC):
        return _LIB
    cc = os.environ.get("CC", "gcc")
    subprocess.check_call([cc, "-std=c11", "-O2", "-ffp-contract=off", "-fPIC", "-shared", _SRC, "-o", _LIB, "-lm"])
    return _LIB


_port = None


def port():
    global _port
    if _port is None:
        lib = C.CDLL(build())
        lib.orc_voxel_down_sample.restype = C.c_int
        lib.orc_voxel_down_sample.argtypes = [_f32p, C.c_int, _i32p, C.c_int, C.c_double, _f32p, _i32p]
        _port = lib
    return _port


def port_voxel_down_sample(points, lengths, voxel_size):
    """Open3D 0.7 voxel_down_sample of every cloud of a stack, canonical order -> (points [M,3] f32, lengths [B] i32).
    voxel_size is used as the Python float (a double) it is given as."""
    pts = np.ascontiguousarray(points, np.float32).reshape(-1, 3)
    lens = np.ascontiguousarray(lengths, np.int32).reshape(-1)
    out = np.empty((max(pts.shape[0], 1), 3), np.float32)
    out_len = np.zeros((lens.shape[0],), np.int32)
    M = port().orc_voxel_down_sample(pts, pts.shape[0], lens, lens.shape[0], float(voxel_size), out, out_len)
    return out[:M].copy(), out_len
