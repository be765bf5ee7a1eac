"""The hot-path ops refuse an illegal tensor argument with a ValueError that names it, before anything is launched.

A kernel reads what it is given: int64 indices are read as int32 pairs, float64 features bit by bit, a host address
faults, a short vector is read out of bounds. So every wrapper checks dtype, device, rank and the shapes of a call
against each other (_lib.tensor_arg) and converts nothing.

Every negative case runs with the library replaced by a stub whose every symbol raises: a missing check cannot reach the
GPU, it fails here. In "host" mode the ops are told their device type is "cpu" (the checks only read attributes), so CPU
tensors stand in for device tensors, a meta tensor for one on the wrong device, and the whole table runs on any machine.
In "cuda" mode (gpu marker) the same table runs on real CUDA tensors with a CPU tensor as the wrong device -- still
under the stub. The positive cases then run every op of the table for real, with the legal arguments.
"""
import numpy as np
import pytest
import torch

F, I = "f", "i"
S = dict(N=6, Nq=5, Ns=7, H=4, K=15, Cin=32, Cout=32, C1=32, C2=8, B=2, D=32, N2=3)
WRONG = {F: [torch.float64, torch.float16, torch.bfloat16, torch.int32],
         I: [torch.int64, torch.int16, torch.float32]}


class Arg:
    def __init__(self, key, kind, shape, optional=False, msg=None, hi=None, any_rank=False, value=None):
        self.key, self.kind, self.shape, self.optional = key, kind, shape, optional
        self.msg = msg or key            # the name the error message uses
        self.hi = hi                     # index tensors: values in [0, S[hi]]
        self.any_rank = any_rank         # no rank case: a row count is one element of any rank
        self.value = value               # fixed content (lengths, row counts)


def count(key, n):
    return Arg(key, I, (1,), optional=True, any_rank=True, value=lambda: [S[n]])


def _lengths(total):
    return lambda: [S[total] - S[total] // 2, S[total] // 2]


def _co():
    from d3feat_b200 import convolution_ops
    return convolution_ops


def _nb():
    from d3feat_b200 import network_blocks
    return network_blocks


def _grid(a, real):
    from d3feat_b200 import tf_custom_ops as ops
    if real:
        return ops.NeighborGrid(a["supports"], a["s_batches"], 0.3)
    g = object.__new__(ops.NeighborGrid)          # what count / fill read of a built grid, without building one
    g.s, g.sb, g.B, g.Ns, g.radius, g.ws, g._bbp = a["supports"], a["s_batches"], S["B"], S["Ns"], 0.3, None, None
    return g


def _select(a, real):
    from d3feat_b200.keypoints import select_keypoints
    return select_keypoints(a["scores"], a["lengths"], 2, points=a["points"], descriptors=a["descriptors"],
                            rows=a["rows"]).index


KP = [Arg("query_points", F, ("Nq", 3)), Arg("support_points", F, ("Ns", 3)),
      Arg("neighbors_indices", I, ("Nq", "H"), hi="Ns"), Arg("features", F, ("Ns", "Cin")),
      Arg("K_values", F, ("K", "Cin", "Cout")), Arg("K_points", F, ("K", 3))]
KP_TAIL = [Arg("query_order", I, ("Nq",), optional=True, value=lambda: list(range(S["Nq"]))[::-1]),
           count("rows_q", "Nq"), count("rows_s", "Ns"),
           Arg("scale", F, ("Cout",), msg="epilogue scale"), Arg("shift", F, ("Cout",), msg="epilogue shift")]
GRID = [Arg("supports", F, ("Ns", 3)), Arg("s_batches", I, ("B",), value=_lengths("Ns"))]
QUERIES = [Arg("queries", F, ("Nq", 3)), Arg("q_batches", I, ("B",), value=_lengths("Nq"))]

# op -> (arguments in the order the wrapper checks them, call(a, real) -> result tensor, fixed arguments)
OPS = {
    "unary_convolution": (
        [Arg("features", F, ("N", "Cin")), Arg("K_values", F, ("Cin", "Cout")),
         Arg("scale", F, ("Cout",), msg="epilogue scale"), Arg("shift", F, ("Cout",), msg="epilogue shift"),
         Arg("residual", F, ("N", "Cout"), optional=True), count("rows", "N")],
        lambda a, real: _co().unary_convolution(a["features"], a["K_values"], epilogue=(a["scale"], a["shift"], 0.2),
                                                residual=a["residual"], rows=a["rows"]), []),
    "unary_pair_convolution": (
        [Arg("x1", F, ("N", "C1")), Arg("x2", F, ("N", "C2")), Arg("w1", F, ("C1", "Cout")),
         Arg("w2", F, ("C2", "Cout")), Arg("s1", F, ("Cout",), msg="affine1 scale"),
         Arg("t1", F, ("Cout",), msg="affine1 shift"), Arg("s2", F, ("Cout",), msg="affine2 scale"),
         Arg("t2", F, ("Cout",), msg="affine2 shift"), count("rows", "N")],
        lambda a, real: _co().unary_pair_convolution(a["x1"], a["w1"], (a["s1"], a["t1"]), a["x2"], a["w2"],
                                                     (a["s2"], a["t2"]), 0.2, rows=a["rows"]), []),
    "KPConv_ops": (
        KP + KP_TAIL + [Arg("bias", F, ("Cout",), optional=True)],
        lambda a, real: _co().KPConv_ops(*[a[x.key] for x in KP[:4]], a["K_points"], a["K_values"], 0.3, "linear", "sum",
                                         epilogue=(a["scale"], a["shift"], 0.2), bias=a["bias"],
                                         query_order=a["query_order"], rows_q=a["rows_q"], rows_s=a["rows_s"]), []),
    "KPConv_deform_ops": (
        KP + KP_TAIL[:3] + [Arg("offsets", F, ("Nq", "K", 3)), Arg("modulations", F, ("Nq", "K"), optional=True)]
        + KP_TAIL[3:],
        lambda a, real: _co().KPConv_deform_ops(
            a["query_points"], a["support_points"], a["neighbors_indices"], a["features"], a["K_points"], a["offsets"],
            a["modulations"], a["K_values"], 0.3, "linear", "sum", epilogue=(a["scale"], a["shift"], 0.2),
            query_order=a["query_order"], rows_q=a["rows_q"], rows_s=a["rows_s"]), []),
    "packed_weight": (
        [Arg("weights", F, ("Cin", "Cout"), any_rank=True)],        # [K, N] or [K, Cin, Cout]
        lambda a, real: _co().packed_weight(a["weights"]), []),
    "ind_max_pool": (
        [Arg("x", F, ("N", "Cin")), Arg("inds", I, ("N2", "H"), hi="N"), count("rows_x", "N"), count("rows_out", "N2")],
        lambda a, real: _nb().ind_max_pool(a["x"], a["inds"], rows_x=a["rows_x"], rows_out=a["rows_out"]), []),
    "closest_pool": (
        [Arg("x", F, ("N", "Cin")), Arg("inds", I, ("N2", "H"), hi="N"), count("rows_x", "N"), count("rows_out", "N2")],
        lambda a, real: _nb().closest_pool(a["x"], a["inds"], rows_x=a["rows_x"], rows_out=a["rows_out"]), []),
    "affine_leaky": (
        [Arg("x", F, ("N", "Cin")), Arg("scale", F, ("Cin",), optional=True), Arg("shift", F, ("Cin",), optional=True),
         Arg("residual", F, ("N", "Cin"), optional=True), count("rows", "N")],
        lambda a, real: _nb()._affine_leaky(a["x"], a["scale"], a["shift"], a["residual"], 0.2, a["rows"]), []),
    "l2_normalize": (
        [Arg("features", F, ("N", "D")), count("rows", "N")],
        lambda a, real: _nb().l2_normalize(a["features"], rows=a["rows"]), []),
    "detection_scores": (
        [Arg("features", F, ("N", "D")), Arg("neighbors", I, ("N", "H"), hi="N"),
         Arg("lengths", I, ("B",), value=_lengths("N")), count("rows", "N")],
        lambda a, real: _nb().detection_scores(a["features"], a["neighbors"], a["lengths"], rows=a["rows"]), []),
    "NeighborGrid": (GRID, lambda a, real: _grid(a, True).order(), []),
    "NeighborGrid.count": (QUERIES, lambda a, real: _grid(a, real).count(a["queries"], a["q_batches"])[0], GRID),
    "NeighborGrid.fill": (QUERIES, lambda a, real: _grid(a, real).fill(a["queries"], a["q_batches"], 3, S["Ns"]), GRID),
    "select_keypoints": (
        [Arg("scores", F, ("N",), any_rank=True), Arg("points", F, ("N", 3), optional=True),
         Arg("descriptors", F, ("N", "D"), optional=True), count("rows", "N")],
        _select, [Arg("lengths", I, ("B",), value=_lengths("N"))]),
}

TORCH = {F: torch.float32, I: torch.int32}


def dims(shape):
    return tuple(d if isinstance(d, int) else S[d] for d in shape)


def tensor(arg, dev, rng, shape=None, dtype=None):
    shape = dims(arg.shape) if shape is None else shape
    if arg.value is not None and shape == dims(arg.shape):
        a = np.asarray(arg.value(), np.int32)
    elif arg.kind == F:
        a = np.asarray(rng.normal(size=shape), np.float32)
    else:
        a = np.asarray(rng.integers(0, (S[arg.hi] if arg.hi else 3) + 1, size=shape), np.int32)
    return torch.from_numpy(a).to(dtype or TORCH[arg.kind]).to(dev)


def arguments(op, dev):
    rng = np.random.default_rng(len(op))
    args, _, fixed = OPS[op]
    return {a.key: tensor(a, dev, rng) for a in args + fixed}


def negative_cases():
    """(op, argument, case, name the message must hold): per argument the wrong device, None, the wrong dtypes,
    rank +- 1, and every dimension off by one. A dimension an earlier argument (or a literal) fixed is this argument's
    fault; one it is the first to name is legal by itself and must be caught at the later argument that shares it."""
    out = []
    for op, (args, _, fixed) in OPS.items():
        seen = {d for f in fixed for d in f.shape}
        for n, a in enumerate(args):
            own = "%s: %s " % (op, a.msg)
            out.append((op, a.key, "device", own))
            if not a.optional:
                out.append((op, a.key, "none", own))
            out += [(op, a.key, str(dt).replace("torch.", ""), own) for dt in WRONG[a.kind]]
            if not a.any_rank:
                out += [(op, a.key, "rank+1", own), (op, a.key, "rank-1", own)]
            for i, d in enumerate(a.shape):
                if isinstance(d, int) or d in seen:
                    out.append((op, a.key, "dim%d+1" % i, own))
                elif any(d in b.shape for b in args[n + 1:]):
                    out.append((op, a.key, "dim%d+1" % i, op + ": "))
            seen |= set(a.shape)
    return out


NEGATIVE = negative_cases()


def mutate(arg, case, dev, wrong_dev, rng):
    shape = dims(arg.shape)
    if case == "none":
        return None
    if case == "device":
        return torch.empty(shape, dtype=TORCH[arg.kind], device=wrong_dev)
    if case == "rank+1":
        return tensor(arg, dev, rng, (1,) + shape)
    if case == "rank-1":
        return tensor(arg, dev, rng, shape[1:])
    if case.startswith("dim"):
        i = int(case[3:-2])
        return tensor(arg, dev, rng, shape[:i] + (shape[i] + 1,) + shape[i + 1:])
    return tensor(arg, dev, rng, dtype=getattr(torch, case))


class Stub:
    def __getattr__(self, symbol):
        raise AssertionError("reached the library with a bad argument: %s" % symbol)


def run_negative(monkeypatch, dev, wrong_dev, op, key, case, name):
    from d3feat_b200 import _lib
    monkeypatch.setattr(_lib, "lib", lambda: Stub())
    args, call, _ = OPS[op]
    a = arguments(op, dev)
    a[key] = mutate(next(x for x in args if x.key == key), case, dev, wrong_dev, np.random.default_rng(1))
    with pytest.raises(ValueError) as e:
        call(a, False)
    assert name in str(e.value) + " ", "the message does not name the argument: %s" % e.value


IDS = ["%s-%s-%s" % c[:3] for c in NEGATIVE]


@pytest.mark.parametrize("op,key,case,name", NEGATIVE, ids=IDS)
def test_bad_argument_is_refused_host(monkeypatch, op, key, case, name):
    from d3feat_b200 import _lib
    monkeypatch.setattr(_lib, "DEVICE_TYPE", "cpu")
    run_negative(monkeypatch, torch.device("cpu"), torch.device("meta"), op, key, case, name)


@pytest.mark.gpu
@pytest.mark.parametrize("op,key,case,name", NEGATIVE, ids=IDS)
def test_bad_argument_is_refused_cuda(cuda, monkeypatch, op, key, case, name):
    run_negative(monkeypatch, cuda, torch.device("cpu"), op, key, case, name)


@pytest.mark.parametrize("op", sorted(OPS))
def test_legal_arguments_pass_the_checks_host(monkeypatch, op):
    """The stub is reached, i.e. no check refuses the legal call (an over-eager check fails here on any machine)."""
    from d3feat_b200 import _lib
    monkeypatch.setattr(_lib, "DEVICE_TYPE", "cpu")
    monkeypatch.setattr(_lib, "lib", lambda: Stub())
    with pytest.raises(AssertionError, match="reached the library"):
        OPS[op][1](arguments(op, torch.device("cpu")), False)


# ---- positive: the real library, legal arguments --------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("op", sorted(OPS))
def test_legal_arguments_run(cuda, op):
    """With the library in place the table's legal call runs, with and without its optional arguments, and the two
    agree where the optional ones are no-ops (full row counts, the identity is not assumed for the others)."""
    args, call, _ = OPS[op]
    a = arguments(op, cuda)
    full = call(a, True)
    assert torch.isfinite(full.float()).all()
    b = dict(a)
    for x in args:
        if x.optional and x.any_rank:
            b[x.key] = None                       # no device row count = every row
    assert torch.equal(call(b, True), full)
    for x in args:
        if x.optional:
            b[x.key] = None
    assert call(b, True).shape == full.shape


@pytest.mark.gpu
def test_empty_inputs_still_pass(cuda):
    co, nb = _co(), _nb()
    z = lambda *s, dt=torch.float32: torch.zeros(s, dtype=dt, device=cuda)
    assert co.unary_convolution(torch.empty((0, 32), device=cuda), z(32, 16)).shape == (0, 16)
    Kp, W = z(15, 3), z(15, 32, 16)
    out = co.KPConv_ops(z(0, 3), z(7, 3), z(0, 4, dt=torch.int32), z(7, 32), Kp, W, 0.3, "linear", "sum")
    assert out.shape == (0, 16)
    out = co.KPConv_ops(z(5, 3), z(0, 3), z(5, 4, dt=torch.int32), z(0, 32), Kp, W, 0.3, "linear", "sum")
    assert out.shape == (5, 16) and bool((out == 0).all())
    out = co.KPConv_deform_ops(z(0, 3), z(7, 3), z(0, 4, dt=torch.int32), z(7, 32), Kp, z(0, 15, 3), z(0, 15), W, 0.3,
                               "linear", "sum")
    assert out.shape == (0, 16)
    assert nb.closest_pool(z(6, 8), z(0, 3, dt=torch.int32)).shape == (0, 8)
    assert nb.ind_max_pool(z(6, 8), z(0, 3, dt=torch.int32)).shape == (0, 8)
    assert nb.l2_normalize(z(0, 32)).shape == (0, 32)
