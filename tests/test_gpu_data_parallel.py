"""GPU: data-parallel training (distributed.reduce_gradients, reduce_moving_statistics, gather_step_stats with
training.MomentumClip). World size 1 over NCCL equals the single-GPU step bit for bit; world size 2, two processes on one
GPU over gloo, leaves both ranks with the same store, bit for bit equal to a single-process emulation that computes both
ranks' gradients and statistics in turn and applies d3f_rank_mean and the update."""
import datetime
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

pytestmark = pytest.mark.gpu

LIMITS = [34, 34, 34, 34, 34]
N_POINTS = 1200
STEPS = 3
WORLD = 2
INVALID = (1, 1)          # (step, rank) whose pair has too few correspondences: only the weight-decay gradient


def pair(seed, k=256):
    """An anchor / positive pair of one room fragment (rotated and shifted) and k keypoint correspondences."""
    from d3feat_b200 import synth
    a = synth.room_fragment(seed, N_POINTS)
    th = 0.2 + 0.1 * seed
    R = np.array([[np.cos(th), -np.sin(th), 0], [np.sin(th), np.cos(th), 0], [0, 0, 1]])
    b = (a @ R.T + np.array([0.5, -0.2, 0.1])).astype(np.float32)
    anc = np.random.default_rng(seed).choice(N_POINTS, k, replace=True).astype(np.int32)
    return np.concatenate([a, b]), np.array([N_POINTS, N_POINTS], np.int32), anc, anc + N_POINTS


def rank_pair(step, rank, world):
    """Each rank's pair: seed = step * world + rank; the INVALID one keeps 16 keypoints (< keypts_num / 2)."""
    pts, lens, anc, pos = pair(step * world + rank)
    if (step, rank) == INVALID:
        anc, pos = anc[:16], pos[:16]
    return pts, lens, anc, pos


class Trainer:
    """One replica: store, encoder and the reference's update."""

    def __init__(self, dev):
        from d3feat_b200 import synth, training as T
        from d3feat_b200.encoder import KPFCNN
        from d3feat_b200.variables import ParamStore
        self.dev = dev
        self.cfg = synth.Config(**T.TRAINING_3DMATCH)
        self.store = ParamStore(synth.make_params(self.cfg, seed=0), dev)
        self.enc = KPFCNN(self.cfg, self.store, LIMITS, device=dev)
        self.params = T.trainable(self.store)
        self.opt = T.MomentumClip(self.params, self.cfg.learning_rate, self.cfg.momentum, self.cfg.grad_clip_norm)

    def backward(self, pts, lens, anc, pos):
        """forward + d3feat_loss + backward on one pair (batch norm updates the moving statistics): the 6 stats."""
        from d3feat_b200 import training as T
        from d3feat_b200.variables import use_params
        inputs = self.enc.build_inputs(pts, lens)
        ag, pg = (torch.from_numpy(np.ascontiguousarray(x)).to(self.dev) for x in (anc, pos))
        with use_params(self.store):
            desc, scores = T.forward(inputs, self.cfg)
            out = T.d3feat_loss(desc, scores, ag, pg, inputs["points"][0], self.cfg)
        out[0].backward()
        return out

    def snapshot(self):
        return {n: t.detach().cpu().numpy().copy() for n, t in self.store.t.items()}, \
               [a.cpu().numpy().copy() for a in self.opt.state]


def dp_step(tr, step, rank, world, group=None):
    """The data-parallel step as a user writes it."""
    from d3feat_b200 import distributed as D
    tr.opt.zero_grad()
    stats = tr.backward(*rank_pair(step, rank, world))
    D.reduce_gradients(tr.params, group)
    tr.opt.step()
    D.reduce_moving_statistics(tr.store, group)
    return D.gather_step_stats(stats, group)


def bits_equal(a, b):
    return np.array_equal(np.asarray(a, np.float32).view(np.uint32), np.asarray(b, np.float32).view(np.uint32))


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


# ---------------------------------------------------------------------------------------------------- world size 1

def test_world_size_one_over_nccl_equals_the_single_gpu_step(cuda):
    single = Trainer(cuda)
    for step in range(STEPS):
        single.opt.zero_grad()
        single.backward(*rank_pair(step, 0, 1))
        single.opt.step()
    torch.cuda.synchronize()
    ref_store, ref_acc = single.snapshot()

    dist.init_process_group("nccl", init_method="tcp://127.0.0.1:%d" % _free_port(), rank=0, world_size=1,
                            timeout=datetime.timedelta(seconds=120))
    try:
        tr = Trainer(cuda)
        for step in range(STEPS):
            logged = dp_step(tr, step, 0, 1)
        torch.cuda.synchronize()
        assert tuple(logged.shape) == (1, 6)
    finally:
        dist.destroy_process_group()
    store, acc = tr.snapshot()
    assert set(store) == set(ref_store)
    for n in ref_store:
        assert bits_equal(store[n], ref_store[n]), n
    for a, b in zip(acc, ref_acc):
        assert bits_equal(a, b)


# ---------------------------------------------------------------------------------------------------- world size 2

def _stage_gloo_through_host():
    """gloo's all_gather on CUDA tensors, through host memory, if this torch build's gloo refuses CUDA tensors."""
    probe = torch.ones(3, device="cuda")
    outs = [torch.empty_like(probe) for _ in range(dist.get_world_size())]
    try:
        dist.all_gather(outs, probe)
        return False
    except RuntimeError:
        pass
    gather = dist.all_gather

    def staged(tensor_list, tensor, group=None, async_op=False):
        host = [torch.empty_like(t, device="cpu") for t in tensor_list]
        gather(host, tensor.cpu(), group=group)
        for t, h in zip(tensor_list, host):
            t.copy_(h)

    dist.all_gather = staged
    return True


def _worker(rank, world, port, out_dir):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    torch.cuda.set_device(0)
    dist.init_process_group("gloo", rank=rank, world_size=world, timeout=datetime.timedelta(seconds=300))
    try:
        staged = _stage_gloo_through_host()
        tr = Trainer(torch.device("cuda", 0))
        logged = [dp_step(tr, step, rank, world).cpu().numpy() for step in range(STEPS)]
        torch.cuda.synchronize()
        store, acc = tr.snapshot()
        np.savez(os.path.join(out_dir, "rank%d.npz" % rank), logged=np.stack(logged), staged=staged,
                 **{"store:" + n: v for n, v in store.items()}, **{"accum:%d" % i: a for i, a in enumerate(acc)})
    finally:
        dist.destroy_process_group()


def emulate(dev, world):
    """Both ranks in one process: each rank's gradients and statistics from the same starting state, in turn, then
    d3f_rank_mean over them and the update."""
    from d3feat_b200 import distributed as D
    tr = Trainer(dev)
    names = [n for n in sorted(tr.store.t) if n.rsplit("/", 1)[-1] in ("moving_mean", "moving_variance")]
    moving = [tr.store.t[n] for n in names]
    logged = []
    for step in range(STEPS):
        start = [t.clone() for t in moving]
        grads, stats, losses = [], [], []
        for rank in range(world):
            for t, s in zip(moving, start):
                t.copy_(s)
            for p in tr.params:
                p.grad = None
            out = tr.backward(*rank_pair(step, rank, world))
            g = [p.grad if p.grad is not None else torch.zeros_like(p) for p in tr.params]
            if step > 0:
                # the replicas zero their gradients in place after the first step: autograd then adds into +0
                g = [torch.zeros_like(x) + x for x in g]
            grads.append(torch.cat([x.reshape(-1) for x in g]))
            stats.append(torch.cat([t.reshape(-1) for t in moving]))
            losses.append(torch.stack([v.detach().reshape(()).float() for v in out]))
        gm = D.rank_mean(torch.stack(grads))
        o = 0
        for p in tr.params:
            p.grad = gm[o:o + p.numel()].view(p.shape).clone()
            o += p.numel()
        tr.opt.step()
        sm = D.rank_mean(torch.stack(stats))
        o = 0
        for t in moving:
            t.copy_(sm[o:o + t.numel()].view(t.shape))
            o += t.numel()
        logged.append(torch.stack(losses).cpu().numpy())
    torch.cuda.synchronize()
    return tr.snapshot(), np.stack(logged)


def test_world_size_two_over_gloo_equals_the_emulation(cuda, tmp_path):
    port = _free_port()
    ctx = mp.get_context("spawn")
    procs = [ctx.Process(target=_worker, args=(r, WORLD, port, str(tmp_path))) for r in range(WORLD)]
    try:
        for p in procs:
            p.start()
        for p in procs:
            p.join(timeout=900)
    finally:
        for p in procs:                          # joined on every path: no process outlives the test
            if p.is_alive():
                p.kill()
            p.join()
    assert [p.exitcode for p in procs] == [0] * WORLD
    ranks = [dict(np.load(tmp_path / ("rank%d.npz" % r))) for r in range(WORLD)]
    print("gloo all_gather %s" % ("staged through host memory" if bool(ranks[0]["staged"]) else "on CUDA tensors"))
    (store, acc), logged = emulate(cuda, WORLD)
    for r in ranks:
        for n, v in store.items():
            assert bits_equal(r["store:" + n], v), n
        for i, a in enumerate(acc):
            assert bits_equal(r["accum:%d" % i], a), i
        assert bits_equal(r["logged"], logged)
    inv_step, inv_rank = INVALID
    assert logged[inv_step, inv_rank, 3] == -1.0 and logged[inv_step, inv_rank, 1] == 0.0   # accuracy -1, no desc loss
    assert (logged[:, :, 3] >= 0).sum() == STEPS * WORLD - 1
    # the ranks trained on different pairs: their losses differ
    assert not np.array_equal(logged[0, 0], logged[0, 1])
