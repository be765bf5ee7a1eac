"""GPU: the kernel-point optimiser (csrc/kernel_points.cu) bit for bit against its restatement
(oracle/kernel_points_np.py): final points, every saved gradient norm and the iteration count, for K in
{1, 2, 4, 7, 15, 32, 64}, the three fixings and 1 or 100 tries (8 tries for K >= 32, where the host restatement of 100
tries takes minutes, except K = 64 'center' with 100 tries, load_kernels' largest problem), and for more tries than
the CTA has threads (K = 4 with 1600 tries, K = 3 with 2000, K = 1 with 6400). It reproduces the reference's own runs
(tests/golden/kernel_dispositions.npz), gives the same bits across calls and streams, and refuses oversized problems
before any launch. A store from training.initial_params runs the inference network and a short training run, whose
snapshot keeps the initial kernel points."""
import os

import numpy as np
import pytest
import torch

from oracle import kernel_points_np as O

pytestmark = pytest.mark.gpu

CASES = [(K, fixed, T) for K in (1, 2, 4, 7, 15, 32, 64) for fixed in ("none", "center", "verticals")
         for T in ((1, 100) if K <= 15 else (1, 8))]
# more tries than the CTA has threads, up to the full 6400 points (the 200 KB shared-memory configuration)
CASES += [(4, fixed, 1600) for fixed in ("none", "center", "verticals")] + [(3, "none", 2000), (1, "none", 6400),
                                                                            (64, "center", 100)]


def initial(K, T, fixed, seed):
    p = np.random.default_rng(seed).uniform(-0.7, 0.7, (T, K, 3))
    return O.fix_points(p, fixed)


def run(x, fixed):
    from d3feat_b200 import kernel_points as kp
    p, saved, n = kp.optimize(x, fixed)
    torch.cuda.synchronize()
    return p.cpu().numpy(), saved.cpu().numpy(), int(n)


def bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.uint64)


@pytest.mark.parametrize("K,fixed,T", CASES)
def test_bit_exact_against_the_restatement(cuda, K, fixed, T):
    x = initial(K, T, fixed, 1000 * K + T)
    p, saved, n = run(x, fixed)
    rp, rsaved, rn = O.optimize(x, fixed)
    assert n == rn
    assert np.array_equal(bits(saved), bits(rsaved))
    assert np.array_equal(bits(p), bits(rp))
    if K <= O.first_moving(fixed, K):
        assert n == 0 and np.array_equal(bits(p), bits(x))


@pytest.mark.parametrize("case", ["center_7", "center_15", "center_32", "none_15", "verticals_15"])
def test_reproduces_the_reference_runs(cuda, golden, case):
    from d3feat_b200 import kernel_points as kp
    z = golden("kernel_dispositions.npz")
    fixed = case.split("_")[0]
    init = z[case + "|initial"]
    points, saved = kp.kernel_point_optimization(1.0, init.shape[1], num_kernels=init.shape[0], fixed=fixed,
                                                 initial=init)
    n = int(z[case + "|iterations"])
    assert saved[n - 1].all() and not saved[n:].any()
    np.testing.assert_allclose(saved[z[case + "|rows"]], z[case + "|saved"], rtol=0, atol=1e-12)
    np.testing.assert_allclose(points, z[case + "|points"], rtol=0, atol=1e-12)
    assert int(np.argmin(saved[-1])) == int(z[case + "|best_k"])


def test_same_bits_across_calls_and_streams(cuda):
    from d3feat_b200 import kernel_points as kp
    x = torch.from_numpy(initial(15, 100, "center", 5)).to(cuda)
    ref = [t.clone() for t in kp.optimize(x, "center")]
    streams = [torch.cuda.Stream(cuda) for _ in range(2)]
    outs = []
    for s in streams:
        with torch.cuda.stream(s):
            s.wait_stream(torch.cuda.current_stream(cuda))
            outs.append(kp.optimize(x, "center"))
    torch.cuda.synchronize()
    for out in outs:
        for a, b in zip(out, ref):
            assert torch.equal(a.view(torch.int64) if a.dtype == torch.float64 else a,
                               b.view(torch.int64) if b.dtype == torch.float64 else b)


def test_oversized_problems_are_refused_before_any_launch(cuda):
    from d3feat_b200 import _lib, kernel_points as kp
    n0 = _lib.launch_count()
    with pytest.raises(ValueError):
        kp.optimize(torch.zeros((101, 64, 3), dtype=torch.float64, device=cuda), "center")
    dummy = torch.zeros(16, dtype=torch.float64, device=cuda)
    for T, K, dim, fixed in ((100, 65, 3, 1), (6401, 1, 3, 0), (1, 15, 2, 1), (1, 15, 3, 3), (0, 15, 3, 1)):
        rc = _lib.lib().d3f_kernel_point_optimize(_lib.ptr(dummy), T, K, dim, fixed, _lib.ptr(dummy),
                                                  _lib.ptr(dummy), _lib.ptr(dummy), _lib.stream())
        assert rc == -1, (T, K, dim, fixed)
    assert _lib.launch_count() == n0


def test_initial_store_runs_the_network_and_a_training_run(cuda, tmp_path):
    from d3feat_b200 import tf_checkpoint as ck, trainer, training
    from d3feat_b200.encoder import KPFCNN
    from d3feat_b200.variables import ParamStore
    from test_gpu_trainer import ANC_TO_POS, LIMITS, clouds, make_config

    cfg = make_config(max_epoch=1)
    params = training.initial_params(cfg, seed=4)
    pts, lens = clouds(cuda)
    out = KPFCNN(cfg, params, LIMITS, device=cuda)(pts[:3000].cpu().numpy(), lens[:2])
    assert all(torch.isfinite(f).all() for f in out["F"])

    run_dir = str(tmp_path / "run")
    store = ParamStore(params, cuda)
    sched = trainer.ThreeDMatchSchedule(pts, lens, ANC_TO_POS, seed=1)
    tr = trainer.Trainer(cfg, store, LIMITS, sched, lambda epoch, i: sched(epoch, i), saving_path=run_dir, seed=3)
    tr.train()
    torch.cuda.synchronize()
    lines = open(os.path.join(run_dir, "training.txt")).read().splitlines()[1:]
    assert lines
    for line in lines:
        vals = [float(tok) for tok in line.replace(",", " ").split() if _is_float(tok)]
        assert vals and np.isfinite(vals).all(), line
    snap = ck.load_params(os.path.join(run_dir, "snapshots", "snap-1"))
    kps = [n for n in params if n.endswith("/kernel_points")]
    assert kps
    for n in kps:
        assert np.array_equal(snap[n].view(np.uint32), params[n].view(np.uint32)), n
    assert any(not np.array_equal(snap[n], params[n]) for n in params if n.endswith("/weights"))


def _is_float(tok):
    try:
        float(tok)
        return True
    except ValueError:
        return False
