"""GPU: one real training step, replayed op by op on the network's own activations against float64
(tests/_training_replay.py records it).

Two pairs, each with the neighbour limits pyramid.calibrate_neighbors gives their clouds, each run with the tensor-core
kernels and with the CUDA-core ones (convolution_ops.USE_TENSOR_CORES, the D3F_TENSOR_CORES switch):
  * 3DMatch: two 15 000-point room fragments in TRAINING_3DMATCH (level 1 spans several 2048-row blocks);
  * KITTI: a lidar-scan pair of 16 000 points each through training_data.training_pairs in TRAINING_KITTI, so the
    network sees the augmented points, lengths and keypoints training feeds it (tens of metres, strong density
    gradient).
The step runs with weights_decay = 0. Then:
  * the recorded calls per op kind equal _training_replay.expected_calls(config);
  * every trainable parameter's .grad equals, bit for bit, the weight / gamma / beta gradient its one op's direct entry
    point gives for the recorded upstream gradient;
  * every op's input gradients from the direct entry points (and batch norm's output, batch mean / invstd and moving
    statistics) are within TOL = 1e-5 x the element's magnitude of the float64 restatement on the same fp32 inputs
    (_oracle.assert_close): LeakyReLU branches pinned to the GPU's output, detection rows whose two best channels lie
    within 1e-5 checked against both channels (fewer than 0.1 % of the rows).
The worst ratio per op kind is printed (RATIO lines), and the float64 side's wall time.
"""
import time

import numpy as np
import pytest
import torch

import _training_replay as rp
from _oracle import TOL, assert_close

pytestmark = pytest.mark.gpu

N_3DMATCH = 15000
N_KITTI = 16000
_PAIRS = {}


def _rotz(th, t):
    T = np.eye(4)
    T[:3, :3] = [[np.cos(th), -np.sin(th), 0], [np.sin(th), np.cos(th), 0], [0, 0, 1]]
    T[:3, 3] = t
    return T


def make_pair(dataset, dev):
    """(config, points, lengths, anc, pos, backup) as one training step sees them (host arrays / device tensors)."""
    if dataset in _PAIRS:
        return _PAIRS[dataset]
    from d3feat_b200 import synth, training as T, training_data as td
    if dataset == "3dmatch":
        cfg = synth.Config(**dict(T.TRAINING_3DMATCH, weights_decay=0.0))
        a = synth.room_fragment(0, N_3DMATCH)
        M = _rotz(0.3, [0.5, -0.2, 0.1])
        b = (a.astype(np.float64) @ M[:3, :3].T + M[:3, 3]).astype(np.float32)
        pts = torch.from_numpy(np.concatenate([a, b])).to(dev)
        lens = torch.tensor([len(a), len(b)], dtype=torch.int32, device=dev)
        rng = np.random.default_rng(0)
        anc = rng.choice(len(a), cfg.keypts_num, replace=True).astype(np.int32)
        anc, pos = (torch.from_numpy(v).to(dev) for v in (anc, anc + len(a)))
        backup = pts
    else:
        cfg = synth.Config(**dict(T.TRAINING_KITTI, weights_decay=0.0))
        a = synth.lidar_scan(1, N_KITTI)
        M = _rotz(0.1, [2.0, 0.5, 0.0])
        b = (a.astype(np.float64) @ M[:3, :3].T + M[:3, 3]).astype(np.float32)
        tp = td.training_pairs(torch.from_numpy(np.concatenate([a, b])).to(dev),
                               torch.tensor([len(a), len(b)], dtype=torch.int32, device=dev),
                               torch.tensor([[0, 1]], dtype=torch.int32, device=dev),
                               torch.from_numpy(M[None]).to(dev), cfg, "kitti", seed=3)
        assert bool(tp.valid[0])
        pts, lens, anc, pos, backup = tp.pair(0)
    _PAIRS[dataset] = (cfg, pts, lens, anc, pos, backup)
    return _PAIRS[dataset]


def record(dev, dataset):
    from d3feat_b200 import pyramid, synth, training as T
    from d3feat_b200.encoder import KPFCNN
    from d3feat_b200.variables import ParamStore, use_params
    cfg, pts, lens, anc, pos, backup = make_pair(dataset, dev)
    host_pts, n = pts.cpu().numpy(), [int(v) for v in lens.tolist()]
    limits = pyramid.calibrate_neighbors(cfg, [host_pts[:n[0]], host_pts[n[0]:]], device=dev)
    store = ParamStore(synth.make_params(cfg, seed=0), dev)
    inputs = KPFCNN(cfg, store, limits, device=dev).build_inputs(pts, lens)
    params = T.trainable(store)
    rec = rp.Recorder()
    with rec.patched(), use_params(store):
        desc, scores = T.forward(inputs, cfg)
        loss, _, _, acc, _, _ = T.d3feat_loss(desc, scores, anc, pos, backup, cfg)
    loss.backward()
    torch.cuda.synchronize()
    assert torch.isfinite(loss).item() and float(acc) != -1.0
    rows = [int(p.shape[0]) for p in inputs["points"]]
    print("\n%s: rows per level %s, neighbour limits %s, loss %.6g" % (dataset, rows, limits, float(loss.detach())))
    return cfg, rec, params, rows


@pytest.mark.parametrize("tensor_cores", [True, False], ids=["tensor_cores", "cuda_cores"])
@pytest.mark.parametrize("dataset", ["3dmatch", "kitti"])
def test_training_step_replay(cuda, monkeypatch, dataset, tensor_cores):
    from d3feat_b200 import convolution_ops as co
    monkeypatch.setattr(co, "USE_TENSOR_CORES", tensor_cores)
    cfg, rec, params, rows = record(cuda, dataset)
    if dataset == "3dmatch":
        assert rows[1] > 2048
    assert rp.counts(rec.calls) == rp.expected_calls(cfg)
    tag = "%s %s" % (dataset, "tc" if tensor_cores else "cuda-core")
    seen = set()
    worst = {}
    t64 = 0.0
    n_amb = n_det = 0
    for r in rec.calls:
        what = "%s #%d %s" % (r["kind"], r["index"], r.get("scope", ""))
        assert r["grad_out"] is not None and r["grad_out"].shape == r["out"].shape, what
        d = rp.direct(r)
        # the step's .grad is the op's own gradient, bit for bit (each parameter is read by exactly one op)
        for p, gp in rp.param_grads(r, d):
            assert id(p) not in seen, what
            seen.add(id(p))
            assert p.grad is not None and torch.equal(p.grad, gp), what
        h = rp.host(r, d)
        t0 = time.perf_counter()
        refs = rp.reference(h)
        t64 += time.perf_counter() - t0
        for name, (ref, mag, alt) in sorted(refs.items()):
            got = h["gpu"][name]
            if r["kind"] == "det":
                rows_in = int(np.asarray(h["lengths"]).sum())
                got, ref, mag, alt = got[:rows_in], ref[:rows_in], mag[:rows_in], alt[:rows_in]
                n_amb, n_det = int(h["ambiguous"].sum()), rows_in
            ratio = assert_close(got, ref, mag, TOL, what="%s %s %s" % (tag, what, name), alt=alt)
            key = "%s %s" % (r["kind"], name)
            worst[key] = max(worst.get(key, 0.0), ratio)
        del d, h, refs
    assert seen == {id(p) for p in params}
    print("%s: detection rows checked against both channels: %d of %d" % (tag, n_amb, n_det))
    assert n_amb < 1e-3 * n_det
    print("%s: float64 side %.1f s; worst |err| / mag per op kind: %s" % (
        tag, t64, ", ".join("%s %.3g" % kv for kv in sorted(worst.items()))))
