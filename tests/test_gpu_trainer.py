"""GPU: the training loop (trainer.Trainer) on small synthetic 3DMatch-style fragments and a small architecture with a
decoder, epoch_steps = 3, validation_size = 2. Two epochs equal a plain loop over the existing API bit for bit; a run
restored from its epoch-1 snapshot in a fresh process ends with the same bits as the uninterrupted one; validation
means equal the losses computed by hand on the inference path; the per-step bookkeeping never synchronises; data
parallel at world size 1 (NCCL) and 2 (gloo, two processes) leaves every rank with the same bits, and only rank 0
writes."""
import datetime
import os

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

pytestmark = pytest.mark.gpu

ARCH = ["simple", "resnetb", "resnetb_strided", "resnetb", "nearest_upsample", "unary", "last_unary"]
LIMITS = [34, 34]
N_POINTS = 1500
ANC_TO_POS = {0: [1, 2], 1: [0, 3], 2: [3, 0], 3: [0]}
SEED = 11


def make_config(**kw):
    from d3feat_b200 import synth, training as T
    base = dict(T.TRAINING_3DMATCH, architecture=list(ARCH), first_features_dim=32, epoch_steps=3, max_epoch=2,
                validation_size=2, snapshot_gap=1, lr_decays={0: 0.5})
    base.update(kw)
    return synth.Config(**base)


def clouds(dev):
    """Four overlapping subsets of one room in its frame, with 1 mm of noise (3DMatch fragments of a scene)."""
    from d3feat_b200 import synth
    room = synth.room_fragment(0, 2 * N_POINTS)
    rng = np.random.default_rng(0)
    parts = [room[np.sort(rng.choice(len(room), N_POINTS, replace=False))] for _ in range(4)]
    parts = [(p + rng.uniform(-1e-3, 1e-3, p.shape)).astype(np.float32) for p in parts]
    return torch.from_numpy(np.concatenate(parts)).to(dev), np.full(4, N_POINTS, np.int32)


def make_trainer(dev, saving_path=None, group=None, **kw):
    from d3feat_b200 import synth, trainer
    from d3feat_b200.variables import ParamStore
    cfg = make_config(**kw)
    pts, lens = clouds(dev)
    train = trainer.ThreeDMatchSchedule(pts, lens, ANC_TO_POS, seed=1)
    val = trainer.ThreeDMatchSchedule(pts, lens, ANC_TO_POS, seed=2)
    store = ParamStore(synth.make_params(cfg, seed=0), dev)
    return trainer.Trainer(cfg, store, LIMITS, train, lambda epoch, i: val(epoch, i), saving_path=saving_path,
                           group=group, seed=SEED)


def state(tr):
    return {n: t.detach().cpu().numpy().copy() for n, t in tr.store.t.items()}, \
           [a.cpu().numpy().copy() for a in tr.opt.state]


def bits_equal(a, b):
    return np.array_equal(np.asarray(a, np.float32).view(np.uint32), np.asarray(b, np.float32).view(np.uint32))


def assert_same_state(a, b):
    (sa, aa), (sb, ab) = a, b
    assert set(sa) == set(sb)
    for n in sa:
        assert bits_equal(sa[n], sb[n]), n
    assert len(aa) == len(ab)
    for i, (x, y) in enumerate(zip(aa, ab)):
        assert bits_equal(x, y), i


def same_means(a, b):
    return all((np.isnan(x) and np.isnan(y)) or bits_equal(x, y) for x, y in zip(a, b))


# ---------------------------------------------------------------------------------------------------- one process

def test_two_epochs_equal_a_plain_loop(cuda):
    from d3feat_b200 import synth, trainer, training as T, training_data as td
    from d3feat_b200.encoder import KPFCNN
    from d3feat_b200.variables import ParamStore, use_params
    tr = make_trainer(cuda)
    tr.train()
    torch.cuda.synchronize()
    # epoch 0: epoch_steps + 1 = 4 steps; epoch 1 would run epoch_steps + 2 = 5, but 4 anchors run out first
    assert [h["epoch_n"] for h in tr.history] == [4, 5] and tr.config.epoch_steps == 4 and tr.step == 9

    cfg = make_config()
    pts, lens = clouds(cuda)
    sched = trainer.ThreeDMatchSchedule(pts, lens, ANC_TO_POS, seed=1)
    store = ParamStore(synth.make_params(cfg, seed=0), cuda)
    enc = KPFCNN(cfg, store, LIMITS, device=cuda)
    params = T.trainable(store)
    opt = T.MomentumClip(params, cfg.learning_rate, cfg.momentum, cfg.grad_clip_norm)
    for epoch in range(2):
        opt.lr = T.learning_rate(cfg, epoch)
        for i in range(4):
            seed = trainer.draw(SEED, epoch, i, trainer.STEP_SEED)
            batch = td.training_pairs(*sched(epoch, i), cfg, "3dmatch", seed=seed)
            points, lengths, anc, pos, backup = batch.pair(0)
            inputs = enc.build_inputs(points, lengths)
            opt.zero_grad()
            with use_params(store):
                desc, scores = T.forward(inputs, cfg)
                loss = T.d3feat_loss(desc, scores, anc, pos, backup, cfg)[0]
            loss.backward()
            opt.step()
    torch.cuda.synchronize()
    assert opt.lr == float(np.float32(np.float32(0.1) * np.float32(0.5)))
    assert_same_state(state(tr), ({n: t.detach().cpu().numpy() for n, t in store.t.items()},
                                  [a.cpu().numpy() for a in opt.state]))


def _resume_worker(snap, out):
    torch.cuda.set_device(0)
    tr = make_trainer(torch.device("cuda", 0))
    tr.restore(snap)
    assert (tr.epoch, tr.step, tr.epoch_n, tr.config.epoch_steps) == (1, 4, 1, 4)
    tr.train()
    torch.cuda.synchronize()
    store, acc = state(tr)
    np.savez(out, **{"store:" + n: v for n, v in store.items()}, **{"accum:%d" % i: a for i, a in enumerate(acc)})


def test_resume_from_a_snapshot_in_a_fresh_process(cuda, tmp_path):
    from d3feat_b200 import io_utils, tf_checkpoint as ck
    run = str(tmp_path / "run")
    tr = make_trainer(cuda, saving_path=run)
    tr.train()
    torch.cuda.synchronize()
    full = state(tr)
    snaps = os.path.join(run, "snapshots")
    assert sorted(os.listdir(snaps)) == sorted("snap-%d%s.%s" % (n, side, ext) for n in (1, 2)
                                               for side in ("", ".trainer")
                                               for ext in ("index", "data-00000-of-00001"))
    # snap-2 is the final store, and a run directory loads as a released one does
    last = ck.load_params(os.path.join(snaps, "snap-2"))
    for n, v in full[0].items():
        assert bits_equal(last[n], v), n
    cfg = io_utils.load_config(run)
    assert cfg.architecture == ARCH and cfg.first_features_dim == 32 and cfg.dataset == "3DMatch"
    assert os.path.exists(os.path.join(run, "kernel_points", "epoch0", "layer_0_simple_0.ply"))
    assert os.path.exists(os.path.join(run, "kernel_points", "epoch1", "layer_0_simple_0.npy"))
    lines = open(os.path.join(run, "training.txt")).read().splitlines()
    assert len(lines) == 1 + 8 + 2 and lines[-1].startswith("3DMatch Epoch   2: desc_loss = ")

    out = str(tmp_path / "resumed.npz")
    p = mp.get_context("spawn").Process(target=_resume_worker, args=(os.path.join(snaps, "snap-1"), out))
    try:
        p.start()
        p.join(timeout=900)
    finally:
        if p.is_alive():
            p.kill()
        p.join()
    assert p.exitcode == 0
    z = np.load(out)
    resumed = ({n[len("store:"):]: z[n] for n in z.files if n.startswith("store:")},
               [z["accum:%d" % i] for i in range(len(full[1]))])
    assert_same_state(resumed, full)


def test_validation_means_equal_the_inference_path_by_hand(cuda):
    """Validation runs on the store the steps updated in place: the inference caches (folded batch norms, packed
    weights) filled before training must be refreshed, so a fresh store of the same values gives the same bits."""
    from d3feat_b200 import trainer, training as T, training_data as td
    from d3feat_b200.encoder import KPFCNN
    from d3feat_b200.variables import ParamStore, use_params
    tr = make_trainer(cuda, max_epoch=1)
    before = tr.validation()                           # fills the inference caches of the initial store
    tr.train()
    torch.cuda.synchronize()
    got = tr.history[0]["val"]
    assert not same_means(got, before)
    cfg = make_config()
    fresh = ParamStore({n: t.detach().cpu().numpy() for n, t in tr.store.t.items()}, cuda)
    enc = KPFCNN(cfg, fresh, LIMITS, device=cuda)
    pts, lens = clouds(cuda)
    val = trainer.ThreeDMatchSchedule(pts, lens, ANC_TO_POS, seed=2)
    rows = []
    with torch.no_grad():
        for i in range(2):
            batch = td.training_pairs(*val(1, i), cfg, "3dmatch", seed=trainer.draw(SEED, 1, i,
                                                                                    trainer.VALIDATION_SEED))
            points, lengths, anc, pos, backup = batch.pair(0)
            out = enc(points, lengths)
            with use_params(fresh):
                stats = T.d3feat_loss(out["descriptors"], out["scores"], anc, pos, backup, cfg)
            rows.append([float(s) for s in stats[1:]])
    want = trainer.epoch_means(np.array(rows, np.float32))
    assert same_means(got, want), (got, want)
    assert np.isfinite(want[0]) and want[2] > 0


def test_step_bookkeeping_never_synchronises(cuda):
    tr = make_trainer(cuda)
    src = tr.train_pairs(0, 0, 0, 1)
    stats = tr.train_step(src, tr.step_seed(0, 0))
    rows = torch.zeros((5, 5), dtype=torch.float32, device=cuda)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for i in range(4):
            tr.train_pairs(1, i, 0, 1)
            tr.val_pairs(1, i)
            tr.step_seed(1, i)
            tr.record(rows, i + 1, stats)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    host = rows.cpu().numpy()
    assert all(bits_equal(host[i + 1], [float(s.detach()) for s in stats[1:]]) for i in range(4))


# ---------------------------------------------------------------------------------------------------- data parallel

def _free_port():
    import socket
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def test_world_size_one_over_nccl_equals_one_process(cuda, tmp_path):
    single = make_trainer(cuda, max_epoch=1)
    single.train()
    torch.cuda.synchronize()
    dist.init_process_group("nccl", init_method="tcp://127.0.0.1:%d" % _free_port(), rank=0, world_size=1,
                            timeout=datetime.timedelta(seconds=120))
    try:
        tr = make_trainer(cuda, saving_path=str(tmp_path / "run"), group=dist.group.WORLD, max_epoch=1)
        tr.train()
        torch.cuda.synchronize()
    finally:
        dist.destroy_process_group()
    assert_same_state(state(tr), state(single))
    assert same_means(tr.history[0]["train"], single.history[0]["train"])
    assert os.path.exists(str(tmp_path / "run" / "snapshots" / "snap-1.index"))


def _dp_worker(rank, world, port, out_dir):
    from test_gpu_data_parallel import _stage_gloo_through_host
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    torch.cuda.set_device(0)
    dist.init_process_group("gloo", rank=rank, world_size=world, timeout=datetime.timedelta(seconds=300))
    try:
        _stage_gloo_through_host()
        tr = make_trainer(torch.device("cuda", 0), saving_path=os.path.join(out_dir, "run%d" % rank),
                          group=dist.group.WORLD)
        tr.train()
        torch.cuda.synchronize()
        store, acc = state(tr)
        np.savez(os.path.join(out_dir, "rank%d.npz" % rank), steps=tr.step,
                 **{"store:" + n: v for n, v in store.items()}, **{"accum:%d" % i: a for i, a in enumerate(acc)})
    finally:
        dist.destroy_process_group()


def test_world_size_two_over_gloo_same_bits_and_rank_zero_writes(cuda, tmp_path):
    world, port = 2, _free_port()
    ctx = mp.get_context("spawn")
    procs = [ctx.Process(target=_dp_worker, args=(r, world, port, str(tmp_path))) for r in range(world)]
    try:
        for p in procs:
            p.start()
        for p in procs:
            p.join(timeout=900)
    finally:
        for p in procs:
            if p.is_alive():
                p.kill()
            p.join()
    assert [p.exitcode for p in procs] == [0] * world
    r0, r1 = (dict(np.load(tmp_path / ("rank%d.npz" % r))) for r in range(world))
    assert set(r0) == set(r1)
    for n in r0:
        assert bits_equal(r0[n], r1[n]), n
    # 4 anchors over 2 ranks: 2 steps, then the third finds them used up, in both epochs
    assert int(r0["steps"]) == 6
    # the ranks trained together: the store moved away from the initial parameters
    from d3feat_b200 import synth
    init = synth.make_params(make_config(), seed=0)
    assert not bits_equal(r0["store:layer_0/simple_0/weights"], init["layer_0/simple_0/weights"])
    assert os.path.exists(str(tmp_path / "run0" / "snapshots" / "snap-2.index"))
    assert not os.path.exists(str(tmp_path / "run1"))
