"""GPU: d3f_momentum_clip_update (training.MomentumClip) bit for bit against oracle/optim_np.py over every trainable
tensor of the 3DMatch store, across streams, in a CUDA graph, and after a real training step; d3f_rank_mean against
the oracle."""
import numpy as np
import pytest
import torch

from oracle import optim_np as oo

pytestmark = pytest.mark.gpu

LIMITS = [34, 34, 34, 34, 34]


def bits(t):
    a = t.detach().cpu().numpy() if torch.is_tensor(t) else np.asarray(t)
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def same(a, b):
    """Bitwise equal, NaN equal to any NaN (the GPU's fp64 -> fp32 conversion gives the canonical NaN)."""
    a, b = bits(a), bits(b)
    nan_a, nan_b = (a & 0x7fffffff) > 0x7f800000, (b & 0x7fffffff) > 0x7f800000
    return np.array_equal(nan_a, nan_b) and np.array_equal(a[~nan_a], b[~nan_b])


def store_tensors(dev):
    """Every trainable tensor of the 3DMatch architecture, plus tensors of 1 and 2049 elements and a zero one."""
    from d3feat_b200 import synth, training as T
    cfg = synth.Config(**T.TRAINING_3DMATCH)
    params = synth.make_params(cfg, seed=0)
    names = [n for n in sorted(params) if n.rsplit("/", 1)[-1] in T.TRAINABLE]
    ts = [torch.from_numpy(np.ascontiguousarray(params[n], np.float32)).to(dev) for n in names]
    rng = np.random.default_rng(5)
    for shape in ((1,), (2049,), (3, 683), (4097,)):
        ts.append(torch.from_numpy(rng.normal(size=shape).astype(np.float32)).to(dev))
    return cfg, ts


def grads_for(ts, step, dev):
    """Gradients whose norms span 1e-3 .. 1e4 (clip active and inactive at 100); tensor 3 is zero every step."""
    rng = np.random.default_rng(100 + step)
    out = []
    for i, t in enumerate(ts):
        scale = 10.0 ** rng.uniform(-3, 4) / np.sqrt(t.numel())
        g = (rng.normal(size=tuple(t.shape)) * scale).astype(np.float32)
        if i == 3:
            g[...] = 0
        out.append(torch.from_numpy(g).to(dev))
    return out


def oracle_steps(vars0, grads, lr, m, clips):
    v = [x.copy() for x in vars0]
    a = [np.zeros_like(x) for x in vars0]
    for s, c in enumerate(clips):
        for i in range(len(v)):
            v[i], a[i] = oo.momentum_clip_update(v[i], a[i], grads[s][i], lr, m, c)
    return v, a


def test_twenty_updates_bit_exact_against_the_oracle(cuda):
    from d3feat_b200 import training as T, _lib
    cfg, ts = store_tensors(cuda)
    n_el = sum(t.numel() for t in ts)
    print("3DMatch store: %d trainable tensors, %d elements (+ the 1 / 2049 / 3x683 / 4097 extras)" % (
        len(ts) - 4, n_el - 1 - 2049 - 3 * 683 - 4097))
    vars0 = [t.cpu().numpy() for t in ts]
    lr, m = cfg.learning_rate, cfg.momentum
    clips = [cfg.grad_clip_norm] * 18 + [0.0, -1.0]              # the last two steps without clipping
    grads = [[g.cpu().numpy() for g in grads_for(ts, s, cuda)] for s in range(len(clips))]
    opt = T.MomentumClip(ts, lr, m, cfg.grad_clip_norm)
    for p in ts:
        p.grad = torch.zeros_like(p)
    n_clipped = 0
    for s, c in enumerate(clips):
        gs = grads_for(ts, s, cuda)
        if s == 7:
            ts[5].grad = gs[5].clone()          # a gradient that moves: the table is rebuilt
        for p, g in zip(ts, gs):
            p.grad.copy_(g)
        opt.clip_norm = c
        n0 = _lib.launch_count()
        opt.step()
        assert _lib.launch_count() - n0 == (2 if c > 0 else 1)
        n_clipped += sum(oo.clip_norm_max(g, c) > np.float32(c) for g in grads[s]) if c > 0 else 0
    torch.cuda.synchronize()
    v, a = oracle_steps(vars0, grads, lr, m, clips)
    print("clipped gradients over the run: %d of %d" % (n_clipped, 18 * len(ts)))
    assert 0 < n_clipped < 18 * len(ts)
    for i, t in enumerate(ts):
        assert np.array_equal(bits(t), bits(v[i])), "var %d (%d elements)" % (i, t.numel())
        assert np.array_equal(bits(opt.state[i]), bits(a[i])), "accum %d" % i


def test_identical_across_streams_and_direct_entry_point(cuda):
    from d3feat_b200 import training as T
    cfg, ts0 = store_tensors(cuda)
    gs = [grads_for(ts0, s, cuda) for s in range(3)]
    results = []
    for stream in (None, torch.cuda.Stream(cuda), "direct"):
        ts = [t.clone() for t in ts0]
        acc = [torch.zeros_like(t) for t in ts]
        opt = T.MomentumClip(ts, cfg.learning_rate, cfg.momentum, cfg.grad_clip_norm)
        if isinstance(stream, torch.cuda.Stream):
            stream.wait_stream(torch.cuda.current_stream())     # ts, acc, state and gs come from the default stream
        with torch.cuda.stream(stream if isinstance(stream, torch.cuda.Stream) else torch.cuda.current_stream()):
            for s in range(3):
                if stream == "direct":
                    T.momentum_clip_update(ts, acc, gs[s], cfg.learning_rate, cfg.momentum, cfg.grad_clip_norm)
                else:
                    for p, g in zip(ts, gs[s]):
                        p.grad = g
                    opt.step()
        torch.cuda.synchronize()
        results.append([bits(t) for t in ts] + [bits(a) for a in (acc if stream == "direct" else opt.state)])
    for r in results[1:]:
        assert all(np.array_equal(x, y) for x, y in zip(results[0], r))


def test_cuda_graph_replay_equals_eager(cuda):
    from d3feat_b200 import training as T
    cfg, ts = store_tensors(cuda)
    opt = T.MomentumClip(ts, cfg.learning_rate, cfg.momentum, cfg.grad_clip_norm)
    for p, g in zip(ts, grads_for(ts, 0, cuda)):
        p.grad = g
    side = torch.cuda.Stream(cuda)
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        opt.step()                                         # warm-up: builds the table outside the capture
    torch.cuda.current_stream().wait_stream(side)
    for p, g in zip(ts, grads_for(ts, 1, cuda)):
        p.grad.copy_(g)
    snap = [t.detach().clone() for t in ts] + [a.clone() for a in opt.state]

    def restore():
        for t, x in zip(ts + opt.state, snap):
            t.detach().copy_(x)

    opt.step()
    torch.cuda.synchronize()
    eager = [bits(t) for t in ts + opt.state]
    restore()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        opt.step()
    restore()
    torch.cuda.synchronize()
    graph.replay()
    torch.cuda.synchronize()
    assert all(np.array_equal(x, bits(t)) for x, t in zip(eager, ts + opt.state))


def test_replaced_accumulators_and_parameter_storage_are_used(cuda):
    """Replacing opt.state[k] (restored slots), the whole state list, or a parameter's storage (p.data = ...) between
    steps moves addresses the cached table holds: the next step must update the new tensors, as the oracle does, and
    leave the replaced ones alone."""
    from d3feat_b200 import training as T
    cfg, ts = store_tensors(cuda)
    lr, m, c = cfg.learning_rate, cfg.momentum, cfg.grad_clip_norm
    opt = T.MomentumClip(ts, lr, m, c)
    v = [t.cpu().numpy() for t in ts]
    a = [np.zeros_like(x) for x in v]
    for p in ts:
        p.grad = torch.zeros_like(p)
    rng = np.random.default_rng(11)
    k, j = 7, len(ts) - 3
    for s in range(4):
        gs = grads_for(ts, s, cuda)
        for p, g in zip(ts, gs):
            p.grad.copy_(g)
        old = None
        if s == 1:                                         # restored slot for tensor k
            loaded = rng.normal(size=tuple(ts[k].shape)).astype(np.float32) * 0.01
            old = opt.state[k]
            opt.state[k] = torch.from_numpy(loaded).to(cuda)
            a[k] = loaded
        elif s == 2:                                       # new storage for parameter j
            fresh = rng.normal(size=tuple(ts[j].shape)).astype(np.float32)
            old = ts[j].data
            ts[j].data = torch.from_numpy(fresh).to(cuda)
            v[j] = fresh
        elif s == 3:                                       # the whole state list replaced by copies
            opt.state = [x.clone() for x in opt.state]
        before = None if old is None else old.clone()
        opt.step()
        torch.cuda.synchronize()
        if old is not None:
            assert torch.equal(old, before)                # the replaced tensor is not written
        for i in range(len(ts)):
            v[i], a[i] = oo.momentum_clip_update(v[i], a[i], gs[i].cpu().numpy(), lr, m, c)
        for i, t in enumerate(ts):
            assert np.array_equal(bits(t), bits(v[i])), (s, i)
            assert np.array_equal(bits(opt.state[i]), bits(a[i])), (s, i)
    opt.state = opt.state[:-1]
    with pytest.raises(ValueError, match=r"MomentumClip.step: %d accumulators in state for %d parameters" % (
            len(ts) - 1, len(ts))):
        opt.step()


def test_table_is_not_rebuilt_during_capture(cuda, monkeypatch):
    """A step whose table would have to be rebuilt while the stream is captured refuses before any launch (the capture
    is simulated: no graph is recorded); the direct entry point, which builds a table every call, refuses too."""
    from d3feat_b200 import training as T, _lib
    cfg, ts = store_tensors(cuda)
    opt = T.MomentumClip(ts, cfg.learning_rate, cfg.momentum, cfg.grad_clip_norm)
    for p, g in zip(ts, grads_for(ts, 0, cuda)):
        p.grad = g
    before = [t.clone() for t in ts]
    monkeypatch.setattr(torch.cuda, "is_current_stream_capturing", lambda: True)
    n0 = _lib.launch_count()
    with pytest.raises(RuntimeError, match="run one eager step"):
        opt.step()
    with pytest.raises(RuntimeError, match="during CUDA graph capture"):
        T.momentum_clip_update(ts, opt.state, [p.grad for p in ts], 0.1, 0.9, 1.0)
    assert _lib.launch_count() == n0
    assert all(torch.equal(t, b) for t, b in zip(ts, before))


def test_after_a_real_training_step(cuda):
    from d3feat_b200 import synth, training as T
    from d3feat_b200.encoder import KPFCNN
    from d3feat_b200.variables import ParamStore, use_params
    cfg = synth.Config(**T.TRAINING_3DMATCH)
    n = 1500
    a = synth.room_fragment(0, n)
    R = np.array([[np.cos(0.3), -np.sin(0.3), 0], [np.sin(0.3), np.cos(0.3), 0], [0, 0, 1]])
    pts = np.concatenate([a, (a @ R.T + np.array([0.5, -0.2, 0.1])).astype(np.float32)])
    anc = np.random.default_rng(0).choice(n, 256).astype(np.int32)
    store = ParamStore(synth.make_params(cfg, seed=0), cuda)
    enc = KPFCNN(cfg, store, LIMITS, device=cuda)
    inputs = enc.build_inputs(pts, np.array([n, n], np.int32))
    params = T.trainable(store)
    opt = T.MomentumClip(params, cfg.learning_rate, cfg.momentum, cfg.grad_clip_norm)
    ag = torch.from_numpy(anc).to(cuda)
    v, acc = None, None
    for step in range(2):
        with use_params(store):
            desc, scores = T.forward(inputs, cfg)
            loss = T.d3feat_loss(desc, scores, ag, ag + n, inputs["points"][0], cfg)[0]
        opt.zero_grad()
        loss.backward()
        grads = [p.grad.cpu().numpy() for p in params]
        if v is None:
            v = [p.detach().cpu().numpy() for p in params]
            acc = [np.zeros_like(x) for x in v]
        opt.step()
        norms = [float(np.sqrt(oo.l2sum(g))) for g in grads]
        print("step %d: loss %.5f, gradient norms %.3g .. %.3g" % (step, float(loss.detach()), min(norms), max(norms)))
        for i in range(len(v)):
            v[i], acc[i] = oo.momentum_clip_update(v[i], acc[i], grads[i], cfg.learning_rate, cfg.momentum,
                                                   cfg.grad_clip_norm)
        for i, p in enumerate(params):
            assert np.array_equal(bits(p), bits(v[i])), i
            assert np.array_equal(bits(opt.state[i]), bits(acc[i])), i


def test_rank_mean_against_the_oracle(cuda):
    from d3feat_b200 import distributed as D
    rng = np.random.default_rng(7)
    for R, P in ((1, 5), (2, 1), (3, 2049), (8, 100003)):
        x = (rng.normal(size=(R, P)) * 10.0 ** rng.uniform(-20, 20, size=(R, P))).astype(np.float32)
        if P > 2:
            x[:, 0] = -0.0
            x[0, 1] = np.nan
        xg = torch.from_numpy(x).to(cuda)
        got = D.rank_mean(xg)
        assert same(got, oo.rank_mean(x)), (R, P)
        if R == 1:
            assert np.array_equal(bits(got), bits(x[0]))   # the input, NaN payload and -0.0 included
        out = xg[0]
        D.rank_mean(xg, out=out)                           # in place over rank 0's row
        assert np.array_equal(bits(out), bits(got)), (R, P)
