"""The decoder half on the serving path, element by element against float64: the workload scripts/keypoint_bench.py
times (fragments 0..7 x 30 000 points, ARCH_3DMATCH, seed-0 parameters, 40 neighbour columns, k = 250).

Every decoder op is traced (tests/_trace.py) and checked on its own inputs: the nearest upsample (closest_pool)
exactly, the unary GEMMs over the concatenated skip features (K = 3072 / 1024 / 512 / 256) and the last unary (K = 64)
against |x| @ |w|, the detection scores against the oracle's magnitude mode. The l2 normalisation is inline in the decoder, so
the descriptors are checked against the float64 normalisation of the traced last-unary output (mag = |ref|). The
keypoints are the argsort oracle (tests/test_gpu_keypoints.py) applied to the GPU's scores, whose every element is
checked against float64 first: the selection is discontinuous in the scores, so this order matters.
"""
import numpy as np
import pytest
import torch

from oracle import kpconv_np as ok

from _oracle import TOL, assert_close
from _trace import record_ops, check_sampled_rows
from test_gpu_keypoints import bits, oracle as keypoint_oracle

pytestmark = pytest.mark.gpu

RTOL = 1e-4
LIMITS = [40, 40, 40, 40, 40]
K = 250
SAMPLED_ROWS = 2000


def t(a, dev):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


@pytest.fixture(scope="module")
def serving_workload(cuda):
    """What scripts/keypoint_bench.py builds: fragments 0..7 x 30 000 points, ARCH_3DMATCH, seed-0 parameters."""
    from d3feat_b200 import synth
    from d3feat_b200.encoder import KPFCNN
    cfg = synth.Config(architecture=synth.ARCH_3DMATCH)
    clouds = [synth.room_fragment(f, 30000) for f in range(8)]
    P = np.concatenate(clouds, 0)
    L = np.array([c.shape[0] for c in clouds], np.int32)
    enc = KPFCNN(cfg, synth.make_params(cfg, 0), LIMITS, device=cuda)
    return cfg, P, L, enc


def _decoder(records):
    """The records from the first nearest upsample on: 4 closest_pool, 4 unary + the last unary, the scores."""
    first = next(i for i, r in enumerate(records) if r["op"] == "closest_pool")
    dec = records[first:]
    ops = [r["op"] for r in dec]
    assert ops.count("closest_pool") == 4 and ops.count("unary") == 5 and ops[-1] == "detection_scores", ops
    assert [int(r["x"].shape[1]) for r in dec if r["op"] == "unary"] == [3072, 1024, 512, 256, 64]
    return dec


def _report(rep, what):
    worst = {}
    for op, _, _, r in rep:
        worst[op] = max(worst.get(op, 0.0), r)
    print("%s: largest |err|/mag per op: %s" % (what, ", ".join("%s %.3e" % kv for kv in sorted(worst.items()))))


def _check_dense(dec, desc, scores, n, what):
    """desc / scores: the GPU's [>= n, 32] / [>= n, 1]. Rows below n only: the l2 normalisation of the traced
    last-unary output, and every score element by element. Returns the GPU scores [n]."""
    rec = dec[-1]
    last_unary = dec[-2]
    assert last_unary["op"] == "unary" and rec["features"] is last_unary["out"]
    x = rec["features"][:n].cpu().numpy().astype(np.float64)
    ref = x / np.sqrt(np.maximum((x * x).sum(1, keepdims=True), 1e-10))
    assert_close(desc[:n].cpu().numpy(), ref, np.abs(ref), TOL, "%s l2_normalize" % what)
    nbr = rec["neighbors"][:n].cpu().numpy()
    assert nbr.min() >= 0 and nbr.max() <= n
    s = scores[:n].cpu().numpy()
    ref, mag, alt = ok.detection_scores(x, nbr, rec["lengths"].cpu().numpy(), magnitude=True)
    assert_close(s, ref, mag, TOL, "%s detection_scores (every row)" % what, alt=alt)
    return s.reshape(-1)


def _check_keypoints(kp, s, L, P, desc):
    idx, cnt = keypoint_oracle(s, L, K)
    assert np.array_equal(kp.index.cpu().numpy(), idx) and np.array_equal(kp.count.cpu().numpy(), cnt)
    assert (idx >= 0).all()
    assert np.array_equal(bits(kp.points.cpu().numpy()), bits(P[idx]))
    assert np.array_equal(bits(kp.descriptors.cpu().numpy()), bits(desc[idx]))
    assert np.array_equal(bits(kp.scores.cpu().numpy()), bits(s[idx]))


def test_serving_workload_decoder_vs_float64(cuda, serving_workload):
    """The eager exact path: enc(P, L, num_keypoints=250) under the trace."""
    cfg, P, L, enc = serving_workload
    with record_ops() as tr:
        out = enc(P, L, num_keypoints=K)
        torch.cuda.synchronize()
    n = P.shape[0]
    tr.records = _decoder(tr.records)
    rep = check_sampled_rows(tr, SAMPLED_ROWS, np.random.default_rng(3), RTOL, what="serving exact")
    _report(rep, "serving exact decoder")
    desc = out["descriptors"]
    assert tuple(desc.shape) == (n, 32) and tuple(out["scores"].shape) == (n, 1)
    s = _check_dense(tr.records, desc, out["scores"], n, "serving exact")
    _check_keypoints(out["keypoints"], s, L, out["inputs"]["points"][0].cpu().numpy(), desc.cpu().numpy())


def test_serving_static_pyramid_and_graph_detections_vs_float64(cuda, serving_workload):
    """The same batch on the static pyramid (capacity-sized launches sized as GraphPipeline.for_batch sizes them, level
    counts only in device memory), run eagerly: every op of the encoder and the decoder on rows below the device count,
    the descriptors, every score and the keypoints. Then GraphPipeline(decoder=True, keypoints=250), stepped twice on
    the batch, returns the eager static descriptors, scores and KeypointSet bit for bit."""
    from d3feat_b200 import pyramid as pyr
    from d3feat_b200.encoder import GraphPipeline
    from d3feat_b200.keypoints import select_keypoints
    cfg, P, L, enc = serving_workload
    Pd, Ld = t(P, cuda), t(L, cuda)
    pipe = GraphPipeline.for_batch(enc, Pd, Ld, decoder=True, keypoints=K)
    buf = pyr.PyramidBuffers(cfg, enc.limits, pipe.caps, pipe.n_clouds, cuda, bbox=pipe.bbox)
    n = P.shape[0]
    buf.points0[:n].copy_(Pd)
    buf.lengths0.copy_(Ld)
    buf.n0.fill_(n)
    inputs = enc.build_inputs_static(buf)
    with record_ops() as tr:
        F = enc.encode(inputs)
        desc, scores = enc.describe(inputs, F, with_scores=True)
        kp = select_keypoints(scores, inputs["lengths"][0], K, points=inputs["points"][0], descriptors=desc,
                              rows=inputs["rows"][0])
        torch.cuda.synchronize()
    assert int(inputs["status"].item()) == 0
    counts = inputs["counts"][:5].cpu().tolist()
    assert counts[0] == n and all(0 < c <= cap for c, cap in zip(counts, pipe.caps))
    assert desc.shape[0] == pipe.caps[0] > n
    assert all(r.get("rows_q") is not None for r in tr.records)      # every op ran capacity-sized
    dec = _decoder(tr.records)
    rep = check_sampled_rows(tr, SAMPLED_ROWS, np.random.default_rng(4), RTOL, min_kpconv=10, what="serving static")
    _report(rep, "serving static encoder + decoder")
    s = _check_dense(dec, desc, scores, n, "serving static")
    _check_keypoints(kp, s, L, inputs["points"][0][:n].cpu().numpy(), desc[:n].cpu().numpy())
    eager = [desc[:n].clone(), scores[:n].clone()] + [x.clone() for x in kp]
    pipe.prime(Pd, Ld)
    got = []
    for i in range(2):
        res, cnt = pipe.step(Pd, Ld) if i == 0 else pipe.step()
        got.append(([res.descriptors[:n].clone(), res.scores[:n].clone()] + [x.clone() for x in res.keypoints],
                    cnt.clone()))
    pipe.check()
    names = ["descriptors", "scores"] + ["keypoints." + f for f in kp._fields]
    for i, (res, cnt) in enumerate(got):
        assert cnt[:5].cpu().tolist() == counts
        for name, a, b in zip(names, res, eager):
            assert a.shape == b.shape and torch.equal(a.view(torch.int32), b.view(torch.int32)), (i, name)
