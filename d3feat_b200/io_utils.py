"""Host-side formats either side of the hot path (SURVEY.md §8 f3/f4): the session's parameters.txt, PLY point
clouds, and the per-fragment arrays the reference's offline evaluation consumes.

  * load_config      -- utils/config.py:Config.load (parameters.txt -> attributes; only the keys the path reads)
  * save_config      -- utils/config.py:Config.save for those keys and the trainer's schedule (trainer.Trainer)
  * write_ply_points -- utils/ply.py:write_ply of x/y/z (the trainer's kernel_points/epoch*/ files)
  * read_ply_points  -- utils/ply.py:read_ply, vertex x/y/z of ascii / binary PLY files
  * select_keypoints -- utils/tester.py:209-213 (3DMatch: all points, ascending score) and :283-290 (KITTI: top-k)
  * write_fragment   -- utils/tester.py:226-228: descriptors/<scene>/cloud_bin_N.D3Feat.npy,
                        keypoints/<scene>/cloud_bin_N.npy, scores/<scene>/cloud_bin_N.npy, the layout
                        geometric_registration/evaluate.py:39-50 reads back (get_keypts / get_desc / get_scores)
  * load_log / load_info / truth_for_pairs -- a 3DMatch scene's gt.log / gt.info as evaluation.GroundTruth; gt.log
                        holds target-to-source poses, the truth is their inverse, source to target
"""
import os

import numpy as np

from .synth import Config

_INT_KEYS = ("num_layers", "first_features_dim", "in_features_dim", "in_points_dim", "num_kernel_points", "num_classes",
             "use_batch_norm", "modulated", "input_threads", "batch_num")
_FLOAT_KEYS = ("first_subsampling_dl", "density_parameter", "KP_extent", "batch_norm_momentum", "in_radius")
_STR_KEYS = ("dataset", "fixed_kernel_points", "KP_influence", "convolution_mode")


def load_config(path):
    """path: a results/Log_*/ directory or its parameters.txt."""
    if os.path.isdir(path):
        path = os.path.join(path, "parameters.txt")
    kw = {}
    with open(path) as fh:
        for line in fh:
            line = line.strip()
            if not line or line.startswith("#") or " = " not in line:
                continue
            key, val = line.split(" = ", 1)
            if key == "architecture":
                kw[key] = val.split()
            elif key in _INT_KEYS:
                kw[key] = int(val)
            elif key in _FLOAT_KEYS:
                kw[key] = float(val)
            elif key in _STR_KEYS:
                kw[key] = val
    if "architecture" not in kw:
        raise ValueError("%s: no architecture line" % path)
    for k in ("use_batch_norm", "modulated"):
        if k in kw:
            kw[k] = bool(kw[k])
    return Config(**kw)


def save_config(config, path, dataset=None):
    """utils/config.py:Config.save for the keys load_config reads (and the trainer's own: the learning-rate schedule,
    max_epoch, epoch_steps, validation_size, snapshot_gap) in the reference's line formats and section layout: writes
    path/parameters.txt. A key the config does not have is left out; dataset fills in a config without one."""
    def has(k):
        return getattr(config, k, None) is not None

    lines = ["# -----------------------------------#", "# Parameters of the training session #",
             "# -----------------------------------#", "", "# Input parameters", "# ****************", ""]
    fmt = dict(in_points_dim="{:d}", in_features_dim="{:d}", in_radius="{:.3f}", input_threads="{:d}",
               num_layers="{:d}", first_features_dim="{:d}", use_batch_norm="{:d}", batch_norm_momentum="{:.3f}",
               first_subsampling_dl="{:.3f}", num_kernel_points="{:d}", density_parameter="{:.3f}",
               fixed_kernel_points="{:s}", KP_extent="{:.3f}", KP_influence="{:s}", convolution_mode="{:s}",
               modulated="{:d}", learning_rate="{:f}", momentum="{:f}", grad_clip_norm="{:f}", weights_decay="{:f}",
               batch_num="{:d}", max_epoch="{:d}", epoch_steps="{:d}", validation_size="{:d}", snapshot_gap="{:d}")

    def put(*keys):
        for k in keys:
            if has(k):
                v = getattr(config, k)
                lines.append((k + " = " + fmt[k]).format(int(v) if fmt[k] == "{:d}" else v))

    name = getattr(config, "dataset", None) or dataset
    if name is not None:
        lines.append("dataset = {:s}".format(name))
    put("in_points_dim", "in_features_dim", "in_radius", "input_threads")
    lines += ["", "# Model parameters", "# ****************", "",
              "architecture =" + "".join(" {:s}".format(a) for a in config.architecture)]
    put("num_layers", "first_features_dim", "use_batch_norm", "batch_norm_momentum")
    lines += ["", "# KPConv parameters", "# *****************", ""]
    put("first_subsampling_dl", "num_kernel_points", "density_parameter", "fixed_kernel_points", "KP_extent",
        "KP_influence", "convolution_mode", "modulated")
    lines += ["", "# Training parameters", "# *******************", ""]
    put("learning_rate", "momentum")
    if getattr(config, "lr_decays", None):
        lines.append("lr_decay_epochs =" + "".join(" {:d}:{:f}".format(e, d) for e, d in config.lr_decays.items()))
    put("grad_clip_norm", "weights_decay", "batch_num", "max_epoch", "epoch_steps", "validation_size", "snapshot_gap")
    os.makedirs(path, exist_ok=True)
    out = os.path.join(path, "parameters.txt")
    with open(out, "w") as fh:
        fh.write("\n".join(lines) + "\n")
    return out


def write_ply_points(path, points):
    """float32 [N,3] points as a binary little-endian PLY with vertex x/y/z (utils/ply.py:write_ply's layout)."""
    pts = np.ascontiguousarray(points, np.float32).reshape(-1, 3)
    head = "ply\nformat binary_little_endian 1.0\nelement vertex %d\nproperty float x\nproperty float y\n" \
           "property float z\nend_header\n" % pts.shape[0]
    with open(path, "wb") as fh:
        fh.write(head.encode("ascii"))
        fh.write(pts.astype("<f4").tobytes())


_PLY_TYPES = {"char": "i1", "int8": "i1", "uchar": "u1", "uint8": "u1", "short": "i2", "int16": "i2", "ushort": "u2",
              "uint16": "u2", "int": "i4", "int32": "i4", "uint": "u4", "uint32": "u4", "float": "f4",
              "float32": "f4", "double": "f8", "float64": "f8"}


def read_ply_points(path):
    """float32 [N,3] vertex positions of a PLY file (ascii, binary little- or big-endian)."""
    with open(path, "rb") as fh:
        if fh.readline().strip() != b"ply":
            raise ValueError("%s: not a PLY file" % path)
        fmt = None
        n_vertex = None
        props = []
        in_vertex = False
        while True:
            line = fh.readline()
            if not line:
                raise ValueError("%s: truncated PLY header" % path)
            tok = line.decode("ascii", "replace").split()
            if not tok:
                continue
            if tok[0] == "format":
                fmt = tok[1]
            elif tok[0] == "element":
                in_vertex = tok[1] == "vertex"
                if in_vertex:
                    n_vertex = int(tok[2])
            elif tok[0] == "property" and in_vertex:
                if tok[1] == "list":
                    raise ValueError("%s: list property on vertices" % path)
                props.append((tok[2], _PLY_TYPES[tok[1]]))
            elif tok[0] == "end_header":
                break
        if n_vertex is None or fmt is None:
            raise ValueError("%s: PLY header without format / vertex element" % path)
        if fmt == "ascii":
            data = np.loadtxt(fh, max_rows=n_vertex, ndmin=2)
            cols = [p[0] for p in props]
            return np.ascontiguousarray(data[:, [cols.index(a) for a in "xyz"]], np.float32)
        order = "<" if fmt == "binary_little_endian" else ">"
        rec = np.fromfile(fh, dtype=[(n, order + t) for n, t in props], count=n_vertex)
    return np.ascontiguousarray(np.stack([rec["x"], rec["y"], rec["z"]], 1), np.float32)


def select_keypoints(scores, num_keypts=None):
    """Indices of the detected keypoints of ONE cloud. scores: [N,1] or [N].
    num_keypts=None: every point in ascending score order (what the 3DMatch tester dumps; the evaluation takes the
    last 250 rows, evaluate.py:47-50). num_keypts=k: the k highest scores, ascending (the KITTI tester)."""
    s = np.asarray(scores).reshape(-1, 1)
    order = np.argsort(s, axis=0).reshape(-1)          # same call as the reference: identical tie order
    return order if num_keypts is None else order[-num_keypts:]


def write_fragment(root, scene, num_frag, points, descriptors, scores, num_keypts=None):
    """Writes the three arrays of one fragment, rows sorted by detection score. Returns the paths."""
    ids = select_keypoints(scores, num_keypts)
    paths = []
    for sub, name, arr in (("descriptors", "cloud_bin_{}.D3Feat".format(num_frag), np.asarray(descriptors)[ids]),
                           ("keypoints", "cloud_bin_{}".format(num_frag), np.asarray(points)[ids]),
                           ("scores", "cloud_bin_{}".format(num_frag), np.asarray(scores)[ids])):
        d = os.path.join(root, sub, scene)
        os.makedirs(d, exist_ok=True)
        p = os.path.join(d, name + ".npy")
        np.save(p, arr.astype(np.float32))
        paths.append(p)
    return paths


def _load_blocks(path, rows):
    """Choi's trajectory format: blocks of a header line `i j n_frag` and `rows` lines of floats."""
    with open(path) as fh:
        lines = [ln.split() for ln in fh if ln.strip()]
    if len(lines) % (rows + 1):
        raise ValueError("%s: %d non-empty lines are not blocks of 1 + %d" % (path, len(lines), rows))
    n = len(lines) // (rows + 1)
    ids = np.zeros((n, 3), np.int64)
    mats = np.zeros((n, rows, rows))
    for b in range(n):
        head = lines[b * (rows + 1)]
        ids[b] = [int(x) for x in head[:3]]
        mats[b] = [[float(x) for x in lines[b * (rows + 1) + 1 + r][:rows]] for r in range(rows)]
    return ids, mats


def load_log(path):
    """(ids [M,3] int64 (i, j, n_frag), T [M,4,4] float64) of a gt.log (geometric_registration/utils.py:loadlog).
    T maps fragment j onto fragment i (target to source): the reference transforms the target by it."""
    return _load_blocks(path, 4)


def load_info(path):
    """(ids [M,3] int64 (i, j, n_frag), info [M,6,6] float64) of a gt.info: Choi's information matrices, read by
    3dmatch/evaluate.m for mrEvaluateRegistration."""
    return _load_blocks(path, 6)


def counts_for_recall(i, j):
    """Registration recall scores only non-consecutive fragments (mrEvaluateRegistration.m: j - i > 1)."""
    return j - i > 1


def truth_for_pairs(log, info, pairs):
    """evaluation.GroundTruth of fragment pairs [(i, j), ...] (the cloud ids of a scene batch) from load_log's and
    load_info's results (info may be None). A pair in the log gets flags bit 0 and G = inv(T_log), the source-to-target
    pose (t ~ R s + t); it also gets bit 1 when j - i > 1 and info is given. Other pairs get flags 0 and the
    identity."""
    from .evaluation import GroundTruth
    ids, T = log
    pairs = np.asarray(pairs, np.int64).reshape(-1, 2)
    P = pairs.shape[0]
    at = {(int(i), int(j)): b for b, (i, j, _) in enumerate(ids)}
    at_info = None if info is None else {(int(i), int(j)): b for b, (i, j, _) in enumerate(info[0])}
    pose = np.tile(np.eye(4), (P, 1, 1))
    inf = None if info is None else np.zeros((P, 6, 6))
    flags = np.zeros(P, np.int32)
    for p, (i, j) in enumerate(pairs.tolist()):
        b = at.get((i, j))
        if b is None:
            continue
        pose[p] = np.linalg.inv(T[b])
        flags[p] = 1
        if at_info is not None and (i, j) in at_info and counts_for_recall(i, j):
            inf[p] = info[1][at_info[(i, j)]]
            flags[p] |= 2
    return GroundTruth(pose, inf, flags)
