"""In-tree build of libd3feat_b200.so (nvcc, sm_90a only). No JIT cache: the .so sits next to this file
so that it travels to the GPU box with the repository snapshot."""
import hashlib
import os
import subprocess
import sys

_HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(_HERE, "csrc")
LIB = os.path.join(_HERE, "libd3feat_b200.so")
_STAMP = os.path.join(_HERE, "csrc", ".build_stamp")

SOURCES = ["api.cu", "sort.cu", "grid.cu", "neighbors.cu", "kpconv.cu", "kpconv_fused.cu", "gemm.cu", "pool.cu", "tc_gemm.cu", "pyramid.cu",
           "keypoints.cu", "matching.cu", "registration.cu", "icp.cu", "evaluation.cu", "voxel.cu", "kpconv_grad.cu", "train_ops.cu",
           "correspond.cu", "optim.cu", "kernel_points.cu"]

NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-lineinfo",
              "-Xcompiler", "-fPIC", "-Xptxas", "-v", "--expt-relaxed-constexpr"]


def _nvcc():
    for c in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if c and (os.path.isabs(c) and os.path.exists(c) or not os.path.isabs(c)):
            return c
    return "nvcc"


def _digest():
    h = hashlib.sha256()
    for root in (CSRC, os.path.join(_HERE, "..", "include")):
        for f in sorted(os.listdir(root)):
            if f.endswith((".cu", ".cuh", ".h")):
                with open(os.path.join(root, f), "rb") as fh:
                    h.update(f.encode())
                    h.update(fh.read())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def build(force=False, verbose=False):
    """Compile every .cu for sm_90a and link the shared library. Returns the path of the .so."""
    srcs = [s for s in SOURCES if os.path.exists(os.path.join(CSRC, s))]
    dig = _digest()
    if not force and os.path.exists(LIB) and os.path.exists(_STAMP) and open(_STAMP).read().strip() == dig:
        return LIB
    objdir = os.path.join(_HERE, "build")
    os.makedirs(objdir, exist_ok=True)
    procs = []
    objs = []
    for s in srcs:
        o = os.path.join(objdir, s.replace(".cu", ".o"))
        objs.append(o)
        cmd = [_nvcc()] + NVCC_FLAGS + ["-c", os.path.join(CSRC, s), "-o", o]
        procs.append((s, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    log = []
    failed = False
    for s, p in procs:
        out, _ = p.communicate()
        log.append("==== %s ====\n%s" % (s, out))
        if p.returncode != 0:
            failed = True
    with open(os.path.join(objdir, "ptxas.log"), "w") as fh:
        fh.write("\n".join(log))
    if failed or verbose:
        sys.stderr.write("\n".join(log) + "\n")
    if failed:
        raise RuntimeError("nvcc failed (see output above)")
    cmd = [_nvcc(), "-shared", "-o", LIB] + objs + ["-lcudart", "-lcuda"]
    subprocess.check_call(cmd)
    with open(_STAMP, "w") as fh:
        fh.write(dig)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
