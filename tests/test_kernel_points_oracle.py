"""The kernel-point optimiser's restatement against the reference's own runs, and the host side of new-run
initialisation (kernel_points.py, training.initial_params) with the optimiser replaced by that restatement.

tests/golden/kernel_dispositions.npz holds runs of kernels/kernel_points.py:41-181 with 100 tries (written by
scripts/make_golden_kernel_points.py): the initial points the reference drew, sampled rows of its gradient-norm
history, its stop iteration, every try's final points and the try load_kernels keeps.
"""
import hashlib

import numpy as np
import pytest
import torch

from d3feat_b200 import kernel_points as kp, synth, training
from oracle import kernel_points_np as O
from test_checkpoint_io import released_snapshot

GOLDEN_CASES = ("center_7", "center_15", "center_32", "none_15", "verticals_15")


@pytest.fixture
def oracle_optimizer(monkeypatch):
    """kernel_points.optimize computed by the restatement (its contract) on the host; a fresh disposition cache."""
    def optimize(initial, fixed="center"):
        p, saved, n = O.optimize(np.asarray(initial, dtype=np.float64), fixed)
        return torch.from_numpy(p), torch.from_numpy(saved), torch.tensor(n, dtype=torch.int32)
    monkeypatch.setattr(kp, "optimize", optimize)
    monkeypatch.setattr(kp, "_cache", {})


@pytest.mark.parametrize("case", GOLDEN_CASES)
def test_restatement_reproduces_the_reference(golden, case):
    z = golden("kernel_dispositions.npz")
    fixed = case.split("_")[0]
    points, saved, n = O.kernel_point_optimization_debug(1.0, z[case + "|initial"], fixed)
    assert n == int(z[case + "|iterations"])
    assert not saved[n:].any() and saved[n - 1].all()
    np.testing.assert_allclose(saved[z[case + "|rows"]], z[case + "|saved"], rtol=0, atol=1e-12)
    np.testing.assert_allclose(points, z[case + "|points"], rtol=0, atol=1e-12)
    assert O.best_try(saved) == int(z[case + "|best_k"]) == 0     # stopped early: the last row is zero


def test_best_try_of_a_full_history_is_the_argmin():
    saved = np.zeros((O.MAX_ITER, 100))
    saved[:] = np.random.default_rng(0).uniform(1.0, 2.0, (O.MAX_ITER, 100))
    saved[-1, 37] = 0.5
    assert O.best_try(saved) == 37
    saved[-1] = 0
    assert O.best_try(saved) == 0


@pytest.mark.parametrize("fixed,K", [("center", 1), ("verticals", 1), ("verticals", 2), ("verticals", 3)])
def test_no_moving_point_runs_no_iteration(oracle_optimizer, fixed, K):
    init = np.random.default_rng(K).uniform(-0.5, 0.5, (4, K, 3))
    p, saved, n = O.optimize(O.fix_points(init, fixed), fixed)
    assert n == 0 and not saved.any()
    assert np.array_equal(p, O.fix_points(init, fixed))
    pts, saved = kp.kernel_point_optimization(2.0, K, num_kernels=4, fixed=fixed, seed=5)
    assert not saved.any() and pts.shape == (4, K, 3)
    assert not pts[:, 0].any()                                   # the centre stays at the origin
    if K > 1:                                                     # rescaled: mean |p| over points 1.. is 2.0
        np.testing.assert_allclose(np.abs(pts[:, 1:, 2]), 2.0, rtol=1e-9)   # |p| carries +1e-12
        assert not pts[:, 1:, :2].any()


def test_unknown_fixed_and_dimension_are_refused():
    with pytest.raises(ValueError):
        kp.kernel_point_optimization(1.0, 15, fixed="corner")
    with pytest.raises(ValueError):
        kp.kernel_point_optimization(1.0, 15, dimension=2)
    with pytest.raises(ValueError):
        kp.load_kernels(1.0, 15, 1, 3, "corner", disposition=np.zeros((15, 3)))
    with pytest.raises(ValueError):
        kp.load_kernels(1.0, 15, 1, 2, "center", disposition=np.zeros((15, 3)))
    with pytest.raises(ValueError):
        kp.optimize(np.zeros((101, 64, 3)), "center")            # T * K > 6400: refused before any launch
    with pytest.raises(ValueError):
        O.first_moving("corner", 15)


def test_initial_points_are_rejection_sampled_and_fixed():
    p = kp.initial_points(15, 100, 7, "none")
    sq = p * p
    assert p.shape == (100, 15, 3) and (((sq[..., 0] + sq[..., 1]) + sq[..., 2]) < 0.5).all()
    c = kp.initial_points(15, 100, 7, "center")
    assert not c[:, 0].any() and np.array_equal(c[:, 1:], p[:, 1:])
    v = kp.initial_points(15, 100, 7, "verticals")
    assert np.array_equal(v[:, 1], np.tile([0, 0, 2 / 3], (100, 1))) and np.array_equal(v[:, 3:], p[:, 3:])
    assert np.array_equal(kp.initial_points(15, 100, 7, "none"), p)
    assert not np.array_equal(kp.initial_points(15, 100, 8, "none"), p)


def test_rotations_are_proper_and_redrawn():
    redrawn = 0
    for n in range(3000):
        R, pairs = kp.rotation(11, n)
        assert np.abs(R.T @ R - np.eye(3)).max() < 5e-8        # the +1e-9 of :255-264 shortens u, v and w
        assert abs(np.linalg.det(R) - 1.0) < 5e-8
        assert abs(R[:, 0] @ R[:, 1]) < 5e-8                   # |u| = 1 - 1e-9: the +1e-9 of :255
        redrawn += pairs > 1
        # the pair kept is the first with |u.v| <= 0.99, as the oracle picks it from the same draws
        idx = np.uint64(((n << 20)) * 3) + np.arange(3 * pairs, dtype=np.uint64)
        u = kp.uniform(11, kp.ROTATION_U, idx).reshape(-1, 3) * 2 - 1
        v = kp.uniform(11, kp.ROTATION_V, idx).reshape(-1, 3) * 2 - 1
        assert np.array_equal(O.rotation(u, v), R)
    assert redrawn > 0                                           # about 1 % of the first pairs are redrawn
    d = np.random.default_rng(0).normal(size=(15, 3))
    got = kp.load_kernels(0.5, 15, 3, 3, "verticals", seed=4, disposition=d)
    for n in range(3):
        theta = kp.uniform(4, kp.THETA, np.arange(n, n + 1))[0] * 2 * np.pi
        assert np.array_equal(got[n], O.rotate(d, 0.5, O.vertical_rotation(theta)))


def _names_shapes(params):
    return {k: tuple(v.shape) for k, v in params.items()}


@pytest.mark.parametrize("arch", ["3dmatch", "kitti_deform"])
def test_initial_params_have_make_params_names(oracle_optimizer, arch):
    cfg = synth.Config() if arch == "3dmatch" else synth.Config(architecture=list(synth.ARCH_KITTI_DEFORM))
    p = training.initial_params(cfg, seed=0)
    m = synth.make_params(cfg, seed=0)
    assert list(p) == list(m) and _names_shapes(p) == _names_shapes(m)
    assert all(v.dtype == np.float32 for v in p.values())


def test_initial_params_have_the_released_snapshot_variables(oracle_optimizer, golden, tmp_path):
    from d3feat_b200 import io_utils, tf_checkpoint as ck
    z = golden("released_checkpoints.npz")
    released = {k: z[k] for k in z.files if k.startswith("contraloss54|")}
    prefix, entries = released_snapshot(released, "contraloss54", 54, tmp_path / "released")
    cfg = io_utils.load_config(__import__("os").path.dirname(prefix))
    p = training.initial_params(cfg, seed=0)
    want = {n[len("KernelPointNetwork/"):]: tuple(e["shape"]) for n, e in entries.items()}
    assert len(want) == len(p) == 196 and _names_shapes(p) == want


def test_initial_values_are_tf_initialisers(oracle_optimizer):
    cfg = synth.Config(architecture=list(synth.ARCH_KITTI_DEFORM))
    p = training.initial_params(cfg, seed=2)
    for k, v in p.items():
        if k.endswith("/gamma") or k.endswith("/moving_variance"):
            assert (v == 1).all(), k
        elif k.endswith("/beta") or k.endswith("/moving_mean") or "offset_conv" in k:
            assert not v.any(), k
        elif k.endswith("/weights"):
            std = np.float32(np.sqrt(2 / v.shape[-1]))
            assert np.array_equal(np.round(v.astype(np.float64) * 1000) / 1000, v.astype(np.float64).round(3)), k
            assert np.abs(np.round(v.astype(np.float64) * 1000) - v.astype(np.float64) * 1000).max() < 1e-3, k
            assert np.abs(v).max() <= 2 * std + 5e-4, k
            if v.size > 2000:
                assert 0.8 * std < v.std() < 0.95 * std, k       # N(0, std) truncated at 2 std: 0.88 std
    off = training.initial_params(synth.Config(use_batch_norm=False), seed=2)
    assert not any("batch_normalization" in k for k in off)
    assert not off["layer_0/simple_0/offset"].any() and off["layer_0/simple_0/offset"].shape == (64,)


def test_kernel_points_are_the_shared_disposition_rotated_with_noise(oracle_optimizer):
    cfg = synth.Config()
    p = training.initial_params(cfg, seed=0)
    D = kp.shared_disposition(cfg.num_kernel_points, "center", 0)
    kps = [(v, p[v.name]) for v in training.nb.variables(cfg) if v.kind == "kernel_points"]
    assert len(kps) == 10                                           # simple + nine resnetb conv2
    seen = set()
    for v, got in kps:
        ref = D * v.radius
        U, _, Vt = np.linalg.svd(got.astype(np.float64).T @ ref)      # Procrustes: got @ R ~ ref
        R = U @ Vt
        res = got.astype(np.float64) @ R - ref
        rms = np.sqrt(np.mean(res ** 2))
        assert 0.6 * 0.01 * v.radius < rms < 1.3 * 0.01 * v.radius, (v.name, rms / v.radius)
        seen.add(got.tobytes())
    assert len(seen) == len(kps)                                    # every KPConv has its own rotation and noise


def test_same_seed_same_bits(oracle_optimizer):
    cfg = synth.Config(architecture=list(synth.ARCH_ENCODER))
    a, b, c = (training.initial_params(cfg, seed=s) for s in (0, 0, 1))
    assert all(np.array_equal(a[k].view(np.uint32), b[k].view(np.uint32)) for k in a)
    assert all(not np.array_equal(a[k], c[k]) for k in a if k.endswith(("/weights", "/kernel_points")))


@pytest.mark.parametrize("arch,seed,trained_like,digest", [
    ("3dmatch", 3, True, "af8f3fd686802e7165a67e1770f208b6bf110435655496127d24a142d1fbf2f2"),
    ("3dmatch", 3, False, "fb909b0c946c1690571744a50a483c5ee57a526162baf91f2e4ff775b937991a"),
    ("kitti_deform_modulated", 3, True, "dea645107a609160eb47718c044db4b59243471f88d256a94b97a0a2783080c0"),
])
def test_make_params_is_unchanged(arch, seed, trained_like, digest):
    """Digests of make_params' names, shapes and bytes, in order, before it read the shared variable schedule."""
    cfg = synth.Config() if arch == "3dmatch" else synth.Config(architecture=list(synth.ARCH_KITTI_DEFORM),
                                                                 modulated=True)
    h = hashlib.sha256()
    for k, v in synth.make_params(cfg, seed=seed, trained_like_bn=trained_like).items():
        h.update(k.encode())
        h.update(str(v.shape).encode())
        h.update(v.tobytes())
    assert h.hexdigest() == digest
