"""The reference's training loop (utils/trainer.py:200-485) around the existing step: epochs, per-epoch statistics,
validation, the learning-rate schedule and snapshots the reference can read, plus an exact resume.

    tr = trainer.Trainer(config, store, neighborhood_limits, train_pairs, val_pairs, saving_path=run_dir, group=None)
    tr.train()                                        # until config.max_epoch
    tr.restore(run_dir + "/snapshots/snap-12")        # then tr.train() continues bit for bit

A step is the one of README "Training on several GPUs": training_data.training_pairs of the source's pair,
enc.build_inputs, training.forward, training.d3feat_loss, backward, distributed.reduce_gradients (with a group),
MomentumClip.step, distributed.reduce_moving_statistics (with a group). Rank r of a world of W takes pair i * W + r of
the epoch at its step i. Only rank 0 reads statistics back, validates and writes files.

Sources. train_pairs(epoch, i, rank, world) and val_pairs(epoch, i) return what training_data.training_pairs takes for
one pair, (points [n,3] float32, lengths [2] int32, pairs [1,2] int32, trans [1,4,4] float64, all on the device), or
None when the epoch's generator has run out (the reference's OutOfRangeError). train_pairs.dataset names the
training_pairs mode ("3dmatch" or "kitti"). ThreeDMatchSchedule and KittiSchedule are two such sources over clouds
held in memory. Pair validity is not checked (that would read the device back): a source should hand out pairs with
enough correspondences, as the reference's generators do.

Epoch accounting, transcribed from :232-408. epoch_n starts at 1 and mean_epoch_n at 0. A step runs, and its
statistics count, then the epoch ends when epoch_n > config.epoch_steps, or before the step when the source returns
None. At the end: the epoch means; mean_epoch_n += (epoch_n - mean_epoch_n) / (epoch + 1), epoch_n = 0 and
config.epoch_steps = floor(mean_epoch_n); snap-{epoch+1} every config.snapshot_gap epochs, with the kernel points and
weights under kernel_points/epoch{epoch}; the learning-rate decay when epoch is in config.lr_decays
(training.learning_rate(config, epoch + 1)); epoch += 1; validation. Then the step counter and epoch_n increment, as
after every step. So the first epoch runs config.epoch_steps + 1 steps and, since epoch_steps then becomes that count,
every later epoch config.epoch_steps + 2 (of the configured value); an epoch cut short by its source still counts the
attempt that found it empty in epoch_n and in the step counter.

Statistics. Each step copies its (desc_loss, det_loss, accuracy, d_pos, d_neg) into row epoch_n of a device buffer
[epoch_steps + 2, 5], an on-stream copy with no synchronisation, and the buffer is read once at the epoch end. The
means apply the reference's exclusions (desc != 0, det != 0, accuracy > 0, d_pos != 0, d_neg != 0) and np.mean to
the float32 values (epoch_means), so they are the reference's means bit for bit given the same per-step values.
training.txt gets the reference's header, a row per step in its format and one validation line per epoch, all written
at the epoch end. Deviations: the time column is the host time at which the step was enqueued (not when it completed)
since train() was called, and the memory column is the peak resident set size in MB (resource.getrusage), not the
current one.

Validation (:417-485) runs the inference KPFCNN on the current store under torch.no_grad(): the reference feeds
dropout_prob = 1.0, which switches its batch norm to the moving statistics. It takes config.validation_size pairs of
val_pairs, d3feat_loss on each, the same buffer, exclusions and means, one read.

Snapshots. snapshots/snap-{n} is a TF bundle of exactly the model variables under KernelPointNetwork/, as the
reference's Saver writes it (no optimizer slots; the released snap-54 holds 196 entries). snapshots/snap-{n}.trainer is
a second bundle with the momentum accumulators (under TF's slot names, tf_checkpoint.write_slots) and the loop's state
at the next step: epoch, step, epoch_n, mean_epoch_n, epoch_steps, learning rate and seed. parameters.txt is written
at the start and at every epoch end (io_utils.save_config), so a run directory loads as a released one does.

Random draws are counter-based splitmix64 (csrc/rng.cuh's function, restated on the host) of (seed, epoch, index,
purpose): the schedules' permutations and positive choices and the training_pairs seeds. Python's random and numpy's
streams are not reproduced, so the pairs differ from the reference's; but a run is bitwise deterministic, and a run
stopped at a snapshot and restored gives the same bits as one that was never stopped.
"""
import os
import resource
import time
import warnings

import numpy as np
import torch

from . import distributed, io_utils, tf_checkpoint, training, training_data
from .encoder import KPFCNN
from .variables import use_params

M64 = (1 << 64) - 1
GOLDEN = 0x9E3779B97F4A7C15           # csrc/rng.cuh kGolden

# the purpose of a draw: the low 3 bits of its counter
PERMUTATION, COIN, CHOICE, STEP_SEED, VALIDATION_SEED = range(5)

STATS = ("desc_loss", "det_loss", "accuracy", "d_pos", "d_neg")
FINE_TUNE_EXCLUDE = ("softmax", "head_unary_conv", "/fc/", "offset")      # utils/trainer.py:98
DATASET_NAMES = {"3dmatch": "3DMatch", "kitti": "KITTI"}                   # config.dataset of training_*.py


# ----------------------------------------------------------------------------------------------------
#  counter-based draws
# ----------------------------------------------------------------------------------------------------

def splitmix64(z):
    """csrc/rng.cuh splitmix64 of uint64 z (a Python int or a numpy uint64 array)."""
    if isinstance(z, np.ndarray):
        z = z.astype(np.uint64)
        with np.errstate(over="ignore"):
            z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
            z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        return z ^ (z >> np.uint64(31))
    z &= M64
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & M64
    return z ^ (z >> 31)


def draw(seed, epoch, index, purpose):
    """splitmix64(seed + counter * golden), counter = ((epoch << 32) | index) * 8 + purpose. index may be a numpy
    integer array (the draws of every index at once)."""
    if isinstance(index, np.ndarray):
        c = ((np.uint64(epoch) << np.uint64(32)) | index.astype(np.uint64)) * np.uint64(8) + np.uint64(purpose)
        with np.errstate(over="ignore"):
            return splitmix64(np.uint64(seed & M64) + c * np.uint64(GOLDEN))
    c = (((int(epoch) << 32) | int(index)) * 8 + purpose) & M64
    return splitmix64(int(seed) + c * GOLDEN)


def draw_index(z, n):
    """csrc/rng.cuh draw_index: an index in [0, n) from draw z, ((z >> 32) * n) >> 32."""
    return ((int(z) >> 32) * int(n)) >> 32


def draw_unit(z):
    """A float64 in [0, 1) from draw z: its top 53 bits (random.random()'s resolution)."""
    return (int(z) >> 11) * 2.0 ** -53


# ----------------------------------------------------------------------------------------------------
#  schedules
# ----------------------------------------------------------------------------------------------------

class _Clouds:
    """Stacked device clouds: the pair of clouds (a, b) as one training_pairs input without a synchronisation."""

    def __init__(self, points, lengths, who):
        lens = np.asarray(lengths.cpu() if torch.is_tensor(lengths) else lengths, np.int64).reshape(-1)
        if not torch.is_tensor(points) or points.dtype != torch.float32 or points.dim() != 2 or points.shape[1] != 3:
            raise ValueError("%s: points must be a float32 [N,3] tensor (on the GPU for training_pairs)" % who)
        if (lens < 0).any() or int(lens.sum()) != int(points.shape[0]):
            raise ValueError("%s: lengths must be non-negative and sum to the %d points" % (who, points.shape[0]))
        self.points, self.n = points, len(lens)
        self.start = np.concatenate([[0], np.cumsum(lens)])
        self.lengths = torch.as_tensor(lens.astype(np.int32)).to(points.device)
        self.pair = torch.tensor([[0, 1]], dtype=torch.int32).to(points.device)

    def get(self, a, b):
        pts = torch.cat([self.points[self.start[a]:self.start[a + 1]], self.points[self.start[b]:self.start[b + 1]]])
        return pts, torch.stack((self.lengths[a], self.lengths[b])), self.pair


class ThreeDMatchSchedule:
    """datasets/ThreeDMatch.py:148-200 over clouds in memory. points [N,3] float32 CUDA, lengths [B] (host or device,
    read once): the fragments, already in a common frame (trans is the identity). anc_to_pos {anchor: [positives]}
    of cloud indices. Epoch e visits the anchors in a permutation (the stable order of their draws), and pair j takes
    the first positive when its coin is above 1/2, otherwise a uniform one (the reference's random.random() > 0.5 /
    random.choice). The generator is restarted at every epoch; step i of rank r takes pair i * world + r, and the
    epoch runs out (None) at the first step whose pairs do not all exist."""
    dataset = "3dmatch"

    def __init__(self, points, lengths, anc_to_pos, seed=0):
        self.clouds = _Clouds(points, lengths, "ThreeDMatchSchedule")
        self.anchors = [int(a) for a in anc_to_pos]
        self.positives = {int(a): [int(p) for p in anc_to_pos[a]] for a in anc_to_pos}
        for a, ps in self.positives.items():
            if not ps or not all(0 <= c < self.clouds.n for c in [a] + ps):
                raise ValueError("ThreeDMatchSchedule: anchor %d: positives %s must be non-empty cloud indices" % (
                    a, ps))
        self.seed = int(seed)
        self.trans = torch.eye(4, dtype=torch.float64).reshape(1, 4, 4).to(points.device)
        self._perm = (None, None)

    def order(self, epoch):
        """The anchors of epoch `epoch` in the order the generator visits them."""
        if self._perm[0] != epoch:
            keys = draw(self.seed, epoch, np.arange(len(self.anchors), dtype=np.uint64), PERMUTATION)
            self._perm = (epoch, [self.anchors[k] for k in np.argsort(keys, kind="stable")])
        return self._perm[1]

    def pair_ids(self, epoch, j):
        """(anchor, positive) cloud indices of pair j of epoch `epoch`."""
        a = self.order(epoch)[j]
        ps = self.positives[a]
        if draw_unit(draw(self.seed, epoch, j, COIN)) > 0.5:
            return a, ps[0]
        return a, ps[draw_index(draw(self.seed, epoch, j, CHOICE), len(ps))]

    def __call__(self, epoch, i, rank=0, world=1):
        if (i + 1) * world > len(self.anchors):
            return None
        pts, lens, pair = self.clouds.get(*self.pair_ids(epoch, i * world + rank))
        return pts, lens, pair, self.trans


class KittiSchedule:
    """KITTI pairs over scans in memory: points [N,3] float32 CUDA, lengths [B], pairs [(anchor, positive)] of cloud
    indices, trans [P,4,4] float64 (anchor onto positive; numpy or device). Every epoch takes the pair list in order
    (the reference permutes it with numpy's stream: order the list yourself to shuffle it). Step i of rank r takes
    pair i * world + r; the epoch runs out (None) at the first step whose pairs do not all exist."""
    dataset = "kitti"

    def __init__(self, points, lengths, pairs, trans):
        self.clouds = _Clouds(points, lengths, "KittiSchedule")
        self.pairs = [(int(a), int(b)) for a, b in pairs]
        if not all(0 <= c < self.clouds.n for p in self.pairs for c in p):
            raise ValueError("KittiSchedule: pairs must name clouds in [0, %d)" % self.clouds.n)
        trans = torch.as_tensor(trans, dtype=torch.float64)
        if tuple(trans.shape) != (len(self.pairs), 4, 4):
            raise ValueError("KittiSchedule: trans must be [%d,4,4]" % len(self.pairs))
        self.trans = trans.to(points.device).contiguous()

    def __call__(self, epoch, i, rank=0, world=1):
        if (i + 1) * world > len(self.pairs):
            return None
        j = i * world + rank
        pts, lens, pair = self.clouds.get(*self.pairs[j])
        return pts, lens, pair, self.trans[j:j + 1]


# ----------------------------------------------------------------------------------------------------
#  statistics
# ----------------------------------------------------------------------------------------------------

def epoch_means(rows):
    """rows float32 [n, 5] of (desc_loss, det_loss, accuracy, d_pos, d_neg) -> the five means of utils/trainer.py:
    284-293 / 339-343: np.mean of the float32 values that pass desc != 0, det != 0, accuracy > 0, d_pos != 0,
    d_neg != 0 (NaN passes != 0 and fails > 0, as there). An empty selection gives NaN, as np.mean([]) does."""
    rows = np.asarray(rows, np.float32).reshape(-1, 5)
    keep = (rows[:, 0] != 0, rows[:, 1] != 0, rows[:, 2] > 0, rows[:, 3] != 0, rows[:, 4] != 0)
    out = []
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", RuntimeWarning)
        for c, k in enumerate(keep):
            out.append(np.mean(rows[k, c]))
    return tuple(out)


def _peak_rss_mb():
    return resource.getrusage(resource.RUSAGE_SELF).ru_maxrss * 1e-3


# ----------------------------------------------------------------------------------------------------
#  the loop
# ----------------------------------------------------------------------------------------------------

class Trainer:
    """The reference's trainer (module docstring) over a ParamStore. config needs, besides the network's and the
    step's attributes (training.TRAINING_3DMATCH / TRAINING_KITTI), max_epoch, epoch_steps, validation_size and
    snapshot_gap; lr_decays is optional. config.epoch_steps is updated at every epoch end, as the reference does.
    store: the ParamStore trained in place (training.trainable marks its parameters). saving_path: the run directory,
    or None to write nothing. group: a torch.distributed process group for data-parallel training, or None for one
    process. seed: the seed of the training_pairs draws.

    After train(): history holds one dict per epoch run (epoch, epoch_n at its end, and on rank 0 the train and val
    means) and opt.state the accumulators, in the order of param_names."""

    def __init__(self, config, store, neighborhood_limits, train_pairs, val_pairs, saving_path=None, group=None,
                 seed=0):
        for key in ("max_epoch", "epoch_steps", "validation_size", "snapshot_gap"):
            v = getattr(config, key, None)
            if isinstance(v, bool) or not isinstance(v, (int, np.integer)) or v < (0 if key == "validation_size"
                                                                                  else 1):
                raise ValueError("Trainer: config.%s=%r must be a positive integer" % (key, v))
        dataset = getattr(train_pairs, "dataset", None)
        if dataset not in training_data.DATASETS:
            raise ValueError("Trainer: train_pairs.dataset=%r must be one of %s" % (dataset, training_data.DATASETS))
        self.config, self.store, self.dataset = config, store, dataset
        self.train_pairs, self.val_pairs = train_pairs, val_pairs
        self.saving_path, self.group, self.seed = saving_path, group, int(seed)
        if group is None:
            self.rank, self.world = 0, 1
        else:
            self.rank, self.world = torch.distributed.get_rank(group), torch.distributed.get_world_size(group)
        self.enc = KPFCNN(config, store, neighborhood_limits, device=store.device)
        self.params = training.trainable(store)
        self.param_names = [n for n in sorted(store.t) if n.rsplit("/", 1)[-1] in training.TRAINABLE]
        self.opt = training.MomentumClip(self.params, config.learning_rate, config.momentum, config.grad_clip_norm)
        self.history = []
        self._reset_counters()

    # -------------------------------------------------------------------------------------------- state

    def _reset_counters(self):
        self.epoch, self.step, self.epoch_n, self.mean_epoch_n = 0, 0, 1, 0
        self.opt.lr = training.learning_rate(self.config, 0)

    def _writes(self):
        return self.saving_path is not None and self.rank == 0

    def restore(self, prefix, model_only=False):
        """Load snapshot `prefix` (snapshots/snap-N) into the store. model_only=False: also its side file (the
        accumulators and the loop's counters, learning rate, epoch_steps and seed), so that train() continues as the
        run that wrote it would have. model_only=True: a fresh start from a reference snapshot, with the reference's
        fine-tuning exclusions (variables whose name holds softmax, head_unary_conv, /fc/ or offset keep their
        values), zero accumulators and fresh counters. The store's tensors are written in place."""
        params = tf_checkpoint.load_params(prefix)
        names = sorted(self.store.t)
        if model_only:
            names = [n for n in names if not any(x in tf_checkpoint.MODEL_SCOPE + n for x in FINE_TUNE_EXCLUDE)]
        elif set(params) != set(names):
            raise tf_checkpoint.CheckpointError("%s: variables differ from the store's: %s" % (
                prefix, sorted(set(params) ^ set(names))[:8]))
        for n in names:
            if n not in params:
                raise tf_checkpoint.CheckpointError("%s: no variable %s" % (prefix, n))
            if tuple(params[n].shape) != tuple(self.store.t[n].shape):
                raise tf_checkpoint.CheckpointError("%s: %s has shape %s, the store %s" % (
                    prefix, n, params[n].shape, tuple(self.store.t[n].shape)))
        with torch.no_grad():
            for n in names:
                self.store.t[n].copy_(torch.from_numpy(np.ascontiguousarray(params[n], np.float32)))
            if model_only:
                for a in self.opt.state:
                    a.zero_()
        if model_only:
            self._reset_counters()
            return
        slots, state = tf_checkpoint.read_slots(prefix + ".trainer")
        if set(slots) != set(self.param_names):
            raise tf_checkpoint.CheckpointError("%s.trainer: slots differ from the trainable variables" % prefix)
        with torch.no_grad():
            for a, n in zip(self.opt.state, self.param_names):
                a.copy_(torch.from_numpy(slots[n]))
        self.epoch, self.step, self.epoch_n = (int(state["trainer/" + k]) for k in ("epoch", "step", "epoch_n"))
        self.mean_epoch_n = float(state["trainer/mean_epoch_n"])
        self.config.epoch_steps = int(state["trainer/epoch_steps"])
        self.opt.lr = float(state["trainer/learning_rate"])
        self.seed = int(state["trainer/seed"])

    def _snapshot(self, n):
        d = os.path.join(self.saving_path, "snapshots")
        tf_checkpoint.write_checkpoint(os.path.join(d, "snap-%d" % n), {
            tf_checkpoint.MODEL_SCOPE + k: t.detach().cpu().numpy() for k, t in self.store.t.items()})

    def _side_file(self, n):
        """The loop's state at the step after the epoch end of snap-{n}."""
        state = {"trainer/epoch": np.int64(self.epoch), "trainer/step": np.int64(self.step + 1),
                 "trainer/epoch_n": np.int64(self.epoch_n + 1), "trainer/mean_epoch_n": np.float64(self.mean_epoch_n),
                 "trainer/epoch_steps": np.int64(self.config.epoch_steps),
                 "trainer/learning_rate": np.float32(self.opt.lr), "trainer/seed": np.uint64(self.seed)}
        tf_checkpoint.write_slots(os.path.join(self.saving_path, "snapshots", "snap-%d.trainer" % n),
                                  {k: a.cpu().numpy() for k, a in zip(self.param_names, self.opt.state)}, state)

    def _kernel_points(self, epoch):
        """utils/trainer.py:503-557: every kernel_points variable as a PLY and every weights variable as .npy under
        kernel_points/epoch{epoch}, named by the variable's scopes joined with '_'."""
        d = os.path.join(self.saving_path, "kernel_points", "epoch%d" % epoch)
        os.makedirs(d, exist_ok=True)
        for n, t in sorted(self.store.t.items()):
            base = "_".join(n.split("/")[:-1])
            if "kernel_points" in n:
                kp = t.detach().cpu().numpy()
                io_utils.write_ply_points(os.path.join(d, base + ".ply"), kp[:, 0, :] if kp.ndim > 2 else kp)
            elif "weights" in n:
                np.save(os.path.join(d, base + ".npy"), t.detach().cpu().numpy())

    # -------------------------------------------------------------------------------------------- step

    def step_seed(self, epoch, i, rank=0, world=1):
        """The training_pairs seed of step i of rank `rank` in epoch `epoch`."""
        return draw(self.seed, epoch, i * world + rank, STEP_SEED)

    def train_step(self, source, seed):
        """One step on the source's pair: the six values of d3feat_loss (device tensors)."""
        batch = training_data.training_pairs(*source, self.config, self.dataset, seed=seed)
        points, lengths, anc, pos, backup = batch.pair(0)
        inputs = self.enc.build_inputs(points, lengths)
        self.opt.zero_grad()
        with use_params(self.store):
            desc, scores = training.forward(inputs, self.config)
            stats = training.d3feat_loss(desc, scores, anc, pos, backup, self.config)
        stats[0].backward()
        if self.group is not None:
            distributed.reduce_gradients(self.params, self.group)
        self.opt.step()
        if self.group is not None:
            distributed.reduce_moving_statistics(self.store, self.group)
        return stats

    def record(self, rows, row, stats):
        """Copy the five logged values of d3feat_loss's result into rows[row] on the stream (no synchronisation)."""
        rows[row].copy_(torch.stack([s.detach().reshape(()) for s in stats[1:6]]))

    def validation(self):
        """:417-485: the five means over config.validation_size pairs of val_pairs on the inference path."""
        n = int(self.config.validation_size)
        rows = torch.zeros((max(n, 1), 5), dtype=torch.float32, device=self.store.device)
        done = 0
        with torch.no_grad():
            for i in range(n):
                source = self.val_pairs(self.epoch, i)
                if source is None:
                    break
                batch = training_data.training_pairs(*source, self.config, self.dataset,
                                                     seed=draw(self.seed, self.epoch, i, VALIDATION_SEED))
                points, lengths, anc, pos, backup = batch.pair(0)
                out = self.enc(points, lengths, decoder=True)
                with use_params(self.store):
                    stats = training.d3feat_loss(out["descriptors"], out["scores"], anc, pos, backup, self.config)
                self.record(rows, i, stats)
                done += 1
        return epoch_means(rows[:done].cpu().numpy())

    # -------------------------------------------------------------------------------------------- loop

    def train(self):
        """Run epochs until config.max_epoch (module docstring); from where restore() left the counters."""
        cfg, writes = self.config, self._writes()
        log = os.path.join(self.saving_path, "training.txt") if writes else None
        if writes:
            os.makedirs(self.saving_path, exist_ok=True)
            io_utils.save_config(cfg, self.saving_path, DATASET_NAMES[self.dataset])
            if self.epoch == 0 and self.step == 0:
                self._kernel_points(0)
            if not os.path.exists(log):
                with open(log, "w") as fh:
                    fh.write("Steps desc_loss det_loss train_accuracy d_pos d_neg time memory\n")
        t0 = time.time()
        rows, steps = None, []
        while self.epoch < cfg.max_epoch:
            if rows is None:
                rows = torch.zeros((cfg.epoch_steps + 2, 5), dtype=torch.float32, device=self.store.device)
            source = self.train_pairs(self.epoch, self.epoch_n - 1, self.rank, self.world)
            if source is not None:
                stats = self.train_step(source, self.step_seed(self.epoch, self.epoch_n - 1, self.rank, self.world))
                if self.rank == 0:
                    self.record(rows, self.epoch_n, stats)
                    steps.append((self.step, self.epoch_n, time.time() - t0, _peak_rss_mb()))
            if source is None or self.epoch_n > cfg.epoch_steps:
                self._epoch_end(rows, steps, log)
                rows, steps = None, []
            self.step += 1
            self.epoch_n += 1

    def _epoch_end(self, rows, steps, log):
        cfg = self.config
        entry = dict(epoch=self.epoch, epoch_n=self.epoch_n)
        if self.rank == 0:
            host = rows.cpu().numpy()                                    # the epoch's one read
            entry["train"] = epoch_means(host[[r for _, r, _, _ in steps]])
            if log is not None:
                with open(log, "a") as fh:
                    for s, r, t, mem in steps:
                        fh.write("{:d} {:.3f} {:.3f} {:.2f} {:.2f} {:.2f} {:.3f} {:.1f}\n".format(
                            s, *(float(v) for v in host[r]), t, mem))
        self.mean_epoch_n += (self.epoch_n - self.mean_epoch_n) / (self.epoch + 1)
        self.epoch_n = 0
        cfg.epoch_steps = int(np.floor(self.mean_epoch_n))
        writes = self._writes()
        if writes:
            io_utils.save_config(cfg, self.saving_path, DATASET_NAMES[self.dataset])
        snap = (self.epoch + 1) % cfg.snapshot_gap == 0
        if snap and writes:
            self._snapshot(self.epoch + 1)
            self._kernel_points(self.epoch)
        decays = getattr(cfg, "lr_decays", None) or {}
        if self.epoch in decays:
            self.opt.lr = training.learning_rate(cfg, self.epoch + 1)
        self.epoch += 1
        if snap and writes:
            self._side_file(self.epoch)
        if self.rank == 0:
            entry["val"] = self.validation()
            if log is not None:
                with open(log, "a") as fh:
                    fh.write("{:s} Epoch {:3d}: desc_loss = {:.3f} det_loss = {:.3f} accuracy = {:.2f}% d_pos = {:.3f} "
                             "d_neg = {:.3f}\n".format(DATASET_NAMES[self.dataset], self.epoch, entry["val"][0],
                                                       entry["val"][1], entry["val"][2] * 100, entry["val"][3],
                                                       entry["val"][4]))
        self.history.append(entry)
