"""The training loop's host logic (d3feat_b200/trainer.py), CPU only: the epoch accounting against a literal
transcription of utils/trainer.py:232-408, the reference's statistic exclusions and means, the 3DMatch and KITTI
schedules, snapshots against the released snap-54 index, the side file and parameters.txt."""
import math
import os
import types
import warnings

import numpy as np
import pytest
import torch

from d3feat_b200 import io_utils, synth, tf_checkpoint as ck, trainer as TR, training

from test_checkpoint_io import released_snapshot


class OutOfRange(Exception):
    pass


def reference_loop(config, values, gen_len):
    """utils/trainer.py:232-408 with the session replaced: values(step) -> (L_desc, L_det, acc, d_pos, d_neg) float32,
    the generator yields gen_len pairs per epoch. Returns per epoch (epoch_n at the end, snapshot or None, lr after
    the end, config.epoch_steps after the end, the five means)."""
    out = []
    training_step, training_epoch = 0, 0
    epoch_n, mean_epoch_n = 1, 0
    lr = np.float32(config.learning_rate)
    pulled = 0
    desc_loss_buf, det_loss_buf, accuracy_buf, ave_d_pos_buf, ave_d_neg_buf = [], [], [], [], []
    while training_epoch < config.max_epoch:
        try:
            if pulled == gen_len:
                raise OutOfRange
            pulled += 1
            L_desc, L_det, acc, ave_d_pos, ave_d_neg = values(training_step)
            if L_desc != 0:
                desc_loss_buf.append(L_desc)
            if acc > 0:
                accuracy_buf.append(acc)
            if L_det != 0:
                det_loss_buf.append(L_det)
            if ave_d_pos != 0:
                ave_d_pos_buf.append(ave_d_pos)
            if ave_d_neg != 0:
                ave_d_neg_buf.append(ave_d_neg)
            if epoch_n > config.epoch_steps:
                raise OutOfRange
        except OutOfRange:
            with warnings.catch_warnings():
                warnings.simplefilter("ignore", RuntimeWarning)                     # np.mean([]) is NaN
                means = (np.mean(desc_loss_buf), np.mean(det_loss_buf), np.mean(accuracy_buf), np.mean(ave_d_pos_buf),
                         np.mean(ave_d_neg_buf))
            desc_loss_buf, accuracy_buf, det_loss_buf, ave_d_pos_buf, ave_d_neg_buf = [], [], [], [], []
            end_n = epoch_n
            mean_epoch_n += (epoch_n - mean_epoch_n) / (training_epoch + 1)
            epoch_n = 0
            config.epoch_steps = int(np.floor(mean_epoch_n))
            snap = training_epoch + 1 if (training_epoch + 1) % config.snapshot_gap == 0 else None
            if training_epoch in config.lr_decays:
                lr = np.float32(lr * np.float32(config.lr_decays[training_epoch]))    # tf.multiply of a float32 var
            training_epoch += 1
            pulled = 0                                                                # train_init_op
            out.append((end_n, snap, float(lr), config.epoch_steps, means))
        training_step += 1
        epoch_n += 1
    return out


class StubTrainer(TR.Trainer):
    """The loop of trainer.Trainer with its step, validation and snapshot writers replaced: no network, no GPU."""

    def __init__(self, config, values, gen_len, saving_path):
        self.config, self.saving_path, self.group, self.rank, self.world, self.seed = config, saving_path, None, 0, 1, 0
        self.train_pairs = lambda epoch, i, rank, world: None if i >= gen_len else (epoch, i)
        self.dataset, self.history, self.values = "3dmatch", [], values
        self.store = types.SimpleNamespace(device=torch.device("cpu"), t={})
        self.opt = types.SimpleNamespace(lr=None)
        self.snaps, self.sides, self.kernel_epochs, self.lrs = [], [], [], []
        self._reset_counters()

    def train_step(self, source, seed):
        return (None,) + tuple(torch.tensor(v) for v in self.values(self.step))

    def validation(self):
        self.lrs.append(self.opt.lr)
        return (np.float32(0),) * 5

    def _snapshot(self, n):
        self.snaps.append(n)

    def _side_file(self, n):
        self.sides.append((n, self.epoch, self.step + 1, self.epoch_n + 1))

    def _kernel_points(self, epoch):
        self.kernel_epochs.append(epoch)


def step_values(step):
    """Per-step statistics with the cases the reference filters: zero losses, accuracy -1 / 0, NaN, negatives."""
    r = np.random.default_rng(step)
    v = r.uniform(0.01, 2.0, 5).astype(np.float32)
    k = step % 7
    if k == 1:
        v[:] = [0, 0, -1, 0, 0]                    # d3feat_loss below keypts_num / 2
    elif k == 3:
        v[2] = 0
    elif k == 4:
        v[0], v[3] = np.nan, np.nan
    elif k == 5:
        v[1] = -v[1]                               # the detection loss can be negative
    return tuple(np.float32(x) for x in v)


def cfg_for(epoch_steps, max_epoch, gap, decays):
    return synth.Config(**dict(training.TRAINING_3DMATCH, epoch_steps=epoch_steps, max_epoch=max_epoch,
                               snapshot_gap=gap, validation_size=0, lr_decays=decays))


def same(a, b):
    return all((math.isnan(x) and math.isnan(y)) or np.float32(x).view(np.uint32) == np.float32(y).view(np.uint32)
               for x, y in zip(a, b))


@pytest.mark.parametrize("epoch_steps,gen_len,max_epoch,gap", [(3, 100, 5, 1), (5, 100, 6, 2), (4, 5, 4, 1),
                                                               (6, 4, 3, 1), (1, 2, 5, 3), (10, 11, 4, 2)])
def test_epoch_accounting_matches_the_reference_loop(tmp_path, epoch_steps, gen_len, max_epoch, gap):
    decays = {0: 0.5, 2: 0.1 ** (1 / 80), 3: 0.9}
    ref = reference_loop(cfg_for(epoch_steps, max_epoch, gap, decays), step_values, gen_len)
    cfg = cfg_for(epoch_steps, max_epoch, gap, decays)
    tr = StubTrainer(cfg, step_values, gen_len, str(tmp_path))
    tr.train()
    assert len(tr.history) == len(ref) == max_epoch
    for e, (h, (end_n, snap, lr, steps, means)) in enumerate(zip(tr.history, ref)):
        assert h["epoch"] == e and h["epoch_n"] == end_n
        assert same(h["train"], means), (e, h["train"], means)
        assert tr.lrs[e] == lr == training.learning_rate(cfg, e + 1)
    assert tr.snaps == [s for _, s, _, _, _ in ref if s is not None]
    assert tr.kernel_epochs == [0] + [s - 1 for s in tr.snaps]
    assert cfg.epoch_steps == ref[-1][3]
    # the side file holds the counters of the step after the snapshot's epoch end
    assert [n for n, *_ in tr.sides] == tr.snaps and all(epoch == n and epoch_n == 1 for n, epoch, _, epoch_n in tr.sides)
    assert tr.step == sum(end_n for end_n, *_ in ref)
    # the first epoch runs epoch_steps + 1 steps, the later ones epoch_steps + 2 (given enough pairs)
    if gen_len > epoch_steps + 2:
        assert [h["epoch_n"] for h in tr.history] == [epoch_steps + 1] + [epoch_steps + 2] * (max_epoch - 1)
    lines = open(os.path.join(str(tmp_path), "training.txt")).read().splitlines()
    assert lines[0] == "Steps desc_loss det_loss train_accuracy d_pos d_neg time memory"
    rows = [ln for ln in lines[1:] if not ln.startswith("3DMatch Epoch")]
    assert len(rows) == sum(min(end_n, gen_len) for end_n, *_ in ref)
    first = rows[0].split()
    assert first[0] == "0" and first[1:6] == ["{:.3f}".format(step_values(0)[0]), "{:.3f}".format(step_values(0)[1]),
                                              "{:.2f}".format(step_values(0)[2]), "{:.2f}".format(step_values(0)[3]),
                                              "{:.2f}".format(step_values(0)[4])]
    assert io_utils.load_config(str(tmp_path)).architecture == cfg.architecture


def test_epoch_means_apply_the_reference_exclusions():
    rows = np.array([[0, 0, -1, 0, 0], [1.5, -0.25, 0.5, 0.7, 1.1], [np.nan, 0.1, np.nan, np.nan, 0],
                     [0.3, np.nan, 0, 0.2, np.nan], [2.0, 0.0, 1.0, -0.0, 0.9], [0.1, 1e-30, -0.5, 1e30, 1e-45]],
                    np.float32)
    bufs = [[], [], [], [], []]
    for r in rows:
        L_desc, L_det, acc, d_pos, d_neg = (np.float32(x) for x in r)
        if L_desc != 0:
            bufs[0].append(L_desc)
        if acc > 0:
            bufs[2].append(acc)
        if L_det != 0:
            bufs[1].append(L_det)
        if d_pos != 0:
            bufs[3].append(d_pos)
        if d_neg != 0:
            bufs[4].append(d_neg)
    got = TR.epoch_means(rows)
    want = tuple(np.mean(b) for b in bufs)
    assert same(got, want) and math.isnan(got[0]) and not math.isnan(got[2])
    assert all(isinstance(g, np.float32) for g in got)
    assert same(TR.epoch_means(rows[:1]), (np.nan, np.nan, np.nan, np.nan, np.nan))
    assert same(TR.epoch_means(np.zeros((0, 5), np.float32)), (np.nan,) * 5)
    # many values: np.mean's pairwise float32 sum over the same array as np.mean(list of float32 scalars)
    big = np.random.default_rng(0).uniform(0, 1, (5000, 5)).astype(np.float32)
    assert same(TR.epoch_means(big), tuple(np.mean([np.float32(x) for x in big[:, c]]) for c in range(5)))


def test_splitmix_matches_the_device_contract():
    # splitmix64 reference values (seed 0 stream: splitmix64(k * golden) for k = 1, 2, 3)
    assert [TR.splitmix64(k * TR.GOLDEN & TR.M64) for k in (1, 2, 3)] == [
        0xE220A8397B1DCDAF, 0x6E789E6AA1B965F4, 0x06C45D188009454F]
    idx = np.arange(1000, dtype=np.uint64)
    vec = TR.draw(123, 7, idx, TR.COIN)
    assert [int(v) for v in vec] == [TR.draw(123, 7, int(i), TR.COIN) for i in idx]
    assert TR.draw_index(TR.M64, 10) == 9 and TR.draw_index(0, 10) == 0


def _clouds(B, n=5):
    lens = np.full(B, n, np.int32)
    pts = torch.arange(B * n * 3, dtype=torch.float32).reshape(-1, 3)
    return pts, lens


def test_3dmatch_schedule():
    pts, lens = _clouds(12)
    anc_to_pos = {a: [(a + 1) % 12, (a + 3) % 12, (a + 7) % 12] for a in range(0, 12, 2)}
    anc_to_pos[1] = [4]
    s = TR.ThreeDMatchSchedule(pts, lens, anc_to_pos, seed=5)
    anchors = list(anc_to_pos)
    orders = []
    for epoch in range(6):
        ids = [s.pair_ids(epoch, j) for j in range(len(anchors))]
        assert sorted(a for a, _ in ids) == sorted(anchors)                     # every anchor once per epoch
        assert all(p in anc_to_pos[a] for a, p in ids)                          # positives only from anc_to_pos
        orders.append([a for a, _ in ids])
        again = TR.ThreeDMatchSchedule(pts, lens, anc_to_pos, seed=5)
        assert [again.pair_ids(epoch, j) for j in range(len(anchors))] == ids  # (seed, epoch) decides
    assert len({tuple(o) for o in orders}) > 1
    other = TR.ThreeDMatchSchedule(pts, lens, anc_to_pos, seed=6)
    assert [other.order(e) for e in range(6)] != orders
    # both positive rules occur: the first positive and a uniform one
    firsts = [s.pair_ids(e, j)[1] == anc_to_pos[s.order(e)[j]][0] for e in range(40) for j in range(len(anchors))]
    assert 0.3 < np.mean(firsts) < 0.95
    # a step's source: the pair's two clouds stacked, run out when a rank's pair is missing
    a, p = s.pair_ids(2, 3)
    pp, ll, pair, trans = s(2, 3)
    assert torch.equal(pp, torch.cat([pts[5 * a:5 * a + 5], pts[5 * p:5 * p + 5]])) and ll.tolist() == [5, 5]
    assert pair.tolist() == [[0, 1]] and torch.equal(trans[0], torch.eye(4, dtype=torch.float64))
    assert s(2, len(anchors) - 1) is not None and s(2, len(anchors)) is None
    assert s(0, 2, 1, 2)[0].shape == (10, 3) and s(0, 3, 0, 2) is None              # 7 anchors, world 2: 3 steps
    with pytest.raises(ValueError):
        TR.ThreeDMatchSchedule(pts, lens, {0: []})


def test_kitti_schedule():
    pts, lens = _clouds(4)
    pairs = [(0, 1), (1, 2), (3, 0)]
    trans = np.stack([np.eye(4) * (k + 1) for k in range(3)])
    s = TR.KittiSchedule(pts, lens, pairs, trans)
    for epoch in (0, 3):
        for i, (a, b) in enumerate(pairs):
            pp, _, _, t = s(epoch, i)
            assert torch.equal(pp, torch.cat([pts[5 * a:5 * a + 5], pts[5 * b:5 * b + 5]]))
            assert np.array_equal(t[0].numpy(), trans[i])
        assert s(epoch, 3) is None
    assert torch.equal(s(0, 0, 1, 2)[0], s(0, 1)[0]) and s(0, 1, 0, 2) is None


def test_snapshot_matches_the_released_index(tmp_path, golden):
    """The trainer's snapshot of a 3DMatch store holds exactly the names, shapes and dtype of the released snap-54,
    and load_params reads it back bit for bit."""
    z = golden("released_checkpoints.npz")
    released = {k: z[k] for k in z.files if k.startswith("contraloss54|")}
    prefix, entries = released_snapshot(released, "contraloss54", 54, tmp_path / "released")
    cfg = io_utils.load_config(os.path.dirname(prefix))
    from d3feat_b200.variables import ParamStore
    tr = object.__new__(TR.Trainer)
    tr.store, tr.saving_path = ParamStore(synth.make_params(cfg, seed=3), "cpu"), str(tmp_path / "run")
    tr._snapshot(54)
    mine = str(tmp_path / "run" / "snapshots" / "snap-54")
    _, got = ck.read_index(mine)
    assert len(entries) == len(got) == 196
    assert {n: (tuple(e["shape"]), e["dtype"]) for n, e in got.items()} == {
        n: (tuple(e["shape"]), e["dtype"]) for n, e in entries.items()}
    back = ck.load_params(mine)
    for n, t in tr.store.t.items():
        assert np.array_equal(back[n].view(np.uint32), t.numpy().view(np.uint32)), n


def test_side_file_and_parameters_round_trip(tmp_path):
    rng = np.random.default_rng(0)
    slots = {"layer_0/simple_0/weights": rng.normal(size=(15, 1, 64)).astype(np.float32),
             "uplayer_1/unary_0/batch_normalization/gamma": rng.normal(size=(32,)).astype(np.float32)}
    extra = {"trainer/epoch": np.int64(12), "trainer/learning_rate": np.float32(0.0123),
             "trainer/seed": np.uint64(TR.M64), "trainer/mean_epoch_n": np.float64(5001.5)}
    ck.write_slots(str(tmp_path / "snap-12.trainer"), slots, extra)
    got, state = ck.read_slots(str(tmp_path / "snap-12.trainer"))
    assert set(got) == set(slots) and set(state) == set(extra)
    for n in slots:
        assert np.array_equal(got[n], slots[n])
    for n in extra:
        assert state[n].dtype == np.asarray(extra[n]).dtype and state[n] == extra[n]
    _, entries = ck.read_index(str(tmp_path / "snap-12.trainer"))
    assert "KernelPointNetwork/layer_0/simple_0/weights/Momentum" in entries
    with pytest.raises(ck.CheckpointError):
        ck.write_slots(str(tmp_path / "bad"), {}, {"KernelPointNetwork/x": np.zeros(1)})

    cfg = synth.Config(**dict(training.TRAINING_3DMATCH, epoch_steps=2918, max_epoch=200, validation_size=500,
                              snapshot_gap=1, dataset="3DMatch", in_points_dim=3, batch_num=1))
    io_utils.save_config(cfg, str(tmp_path))
    back = io_utils.load_config(str(tmp_path))
    for k in ("architecture", "num_layers", "first_features_dim", "in_features_dim", "in_points_dim", "use_batch_norm",
              "batch_norm_momentum", "first_subsampling_dl", "num_kernel_points", "density_parameter",
              "fixed_kernel_points", "KP_extent", "KP_influence", "convolution_mode", "modulated", "dataset",
              "batch_num"):
        assert getattr(back, k) == getattr(cfg, k), k
    text = open(str(tmp_path / "parameters.txt")).read()
    assert "epoch_steps = 2918\n" in text and "lr_decay_epochs = 1:0.971628 2:0.971628" in text
    assert "learning_rate = 0.100000\n" in text and "use_batch_norm = 1\n" in text


def test_fast_crc_equals_the_byte_serial_crc():
    rng = np.random.default_rng(1)
    tab = ck._CRC_TABLE
    for n in (1 << 16, (1 << 16) + 1, 3 * 4096 * 7 + 13):
        data = rng.integers(0, 256, n, dtype=np.uint8).tobytes()
        for crc in (0, 0xDEADBEEF):
            c = (~crc) & 0xFFFFFFFF
            for b in data:
                c = int(tab[(c ^ b) & 0xFF]) ^ (c >> 8)
            assert ck.crc32c(data, crc) == (~c) & 0xFFFFFFFF
