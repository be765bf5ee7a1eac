"""User-facing driver of the hot path: stacked point-cloud fragments in, per-level encoder features (and,
optionally, the 32-d descriptors of the D3Feat decoder) out.

Mirrors how the reference is driven at test time (utils/tester.py:177-233: one sess.run per batch that
executes the tf.data pyramid on the CPU and the network on the device); here both halves run on the GPU:

    enc = KPFCNN(config, params, neighborhood_limits)
    out = enc(points_host_or_cuda, lengths)           # pyramid + encoder (+ decoder)
"""
from collections import namedtuple

import numpy as np
import torch

from . import network_blocks as nb
from . import pyramid
from .evaluation import OPTIONS as EVALUATE_OPTIONS, GroundTruth, check_evaluate_options, check_truth, evaluate_pairs
from .keypoints import sample_keypoints, select_keypoints
from .matching import host_pairs, match_keypoints
from .registration import ICP_OPTIONS, OPTIONS as REGISTER_OPTIONS, check_icp_options, check_options, icp_pairs, \
    register_pairs
from .variables import ParamStore, use_params
from .voxel import VoxelStage, voxel_down_sample

# GraphPipeline(..., keypoints=k) result: descriptors [cap0,32], scores [cap0,1], keypoints (KeypointSet, k per cloud)
Detections = namedtuple("Detections", "descriptors scores keypoints")
# GraphPipeline(..., keypoints=k, match_pairs=pairs) result: the same plus matches (matching.Matches of every pair)
MatchedDetections = namedtuple("MatchedDetections", "descriptors scores keypoints matches")
# GraphPipeline(..., match_pairs=pairs, register={...}) result: the same plus registration (registration.Registration)
RegisteredDetections = namedtuple("RegisteredDetections", "descriptors scores keypoints matches registration")
# GraphPipeline(..., register={...}, icp={...}) result: the same plus refinement (registration.Refinement)
RefinedDetections = namedtuple("RefinedDetections", "descriptors scores keypoints matches registration refinement")
# GraphPipeline(..., match_pairs=pairs, evaluate={...}) result: the same plus evaluation (evaluation.Evaluation);
# registration / refinement are None when the pipeline does not run them
EvaluatedDetections = namedtuple("EvaluatedDetections",
                                 "descriptors scores keypoints matches registration refinement evaluation")
# GraphPipeline(..., match_pairs=pairs, sweep={...}) result: the fields above (None for the stages the pipeline does not
# run) plus sweep, a dict (arm, count) -> SweepEntry in the order of sweep_arms x sweep_counts
SweptDetections = namedtuple("SweptDetections",
                             "descriptors scores keypoints matches registration refinement evaluation sweep")
SweepEntry = namedtuple("SweepEntry", "keypoints matches registration refinement evaluation")
SWEEP_ARMS = ("score", "random")
SWEEP_OPTIONS = ("counts", "arms", "seed")


def check_sweep(sweep, keypoints, who="GraphPipeline"):
    """(counts, arms, seed) of a sweep={...} option, or ValueError: counts strictly descending within [1, keypoints],
    arms a non-empty subset of SWEEP_ARMS without repeats (default both), seed an integer in [0, 2^64) (default 0)."""
    if not isinstance(sweep, dict) or set(sweep) - set(SWEEP_OPTIONS) or "counts" not in sweep:
        raise ValueError("%s: sweep must be a dict of %s with counts, got %r" % (who, SWEEP_OPTIONS, sweep))

    def is_int(x):
        return not isinstance(x, bool) and isinstance(x, (int, np.integer))
    try:
        counts = tuple(sweep["counts"])
    except TypeError:
        counts = None
    if not counts or not all(is_int(c) for c in counts):
        raise ValueError("%s: sweep counts=%r must be a non-empty sequence of integers" % (who, sweep["counts"]))
    counts = tuple(int(c) for c in counts)
    if any(b >= a for a, b in zip(counts, counts[1:])) or not 1 <= counts[-1] or counts[0] > keypoints:
        raise ValueError("%s: sweep counts=%r must descend strictly within [1, keypoints=%d]" % (who, counts,
                                                                                                 keypoints))
    arms = sweep.get("arms", SWEEP_ARMS)
    arms = (arms,) if isinstance(arms, str) else arms
    try:
        arms = tuple(arms)
    except TypeError:
        arms = ()
    if not arms or any(a not in SWEEP_ARMS for a in arms) or len(set(arms)) != len(arms):
        raise ValueError("%s: sweep arms=%r must be a non-empty subset of %s" % (who, sweep.get("arms"), SWEEP_ARMS))
    seed = sweep.get("seed", 0)
    if not is_int(seed) or not 0 <= int(seed) < 2 ** 64:
        raise ValueError("%s: sweep seed=%r must be an integer in [0, 2^64)" % (who, seed))
    return counts, arms, int(seed)


class KPFCNN:
    def __init__(self, config, params, neighborhood_limits, device="cuda"):
        self.config = config
        self.device = torch.device(device)
        self.store = params if isinstance(params, ParamStore) else ParamStore(params, self.device)
        self.limits = [int(x) for x in neighborhood_limits]
        self.has_decoder = any("upsample" in b for b in config.architecture)

    def build_inputs_static(self, buffers):
        """Sync-free pyramid over the batch already sitting in buffers.points0 / lengths0 / n0 (see
        pyramid.descriptor_input, static form). Every tensor is a whole capacity-sized buffer."""
        inputs = pyramid.descriptor_input(self.config, buffers.points0, buffers.lengths0, self.limits, buffers=buffers,
                                          static=True)
        inputs["features"] = buffers.features0
        return inputs

    def build_inputs(self, stacked_points, stacked_lengths, features=None, bbox=None, buffers=None):
        pts = stacked_points
        if not torch.is_tensor(pts):
            pts = torch.as_tensor(np.ascontiguousarray(pts, np.float32))
        pts = pts.to(self.device, non_blocking=True)
        lens = stacked_lengths
        if not torch.is_tensor(lens):
            lens = torch.as_tensor(np.ascontiguousarray(lens, np.int32))
        lens = lens.to(self.device, non_blocking=True)
        inputs = pyramid.descriptor_input(self.config, pts, lens, self.limits, bbox=bbox, buffers=buffers)
        if features is None:
            # the 3DMatch generator feeds a constant-one feature (datasets/ThreeDMatch.py:316)
            features = torch.ones((pts.shape[0], self.config.in_features_dim), dtype=torch.float32, device=self.device)
        elif not torch.is_tensor(features):
            features = torch.as_tensor(np.ascontiguousarray(features, np.float32)).to(self.device)
        inputs["features"] = features
        return inputs

    def encode(self, inputs):
        """assemble_CNN_blocks on prepared inputs -> list F of per-level features."""
        with use_params(self.store):
            return nb.assemble_CNN_blocks(inputs, self.config, 1.0)

    def describe(self, inputs, F, with_scores=False):
        """Decoder -> descriptors [N,32]; with_scores=True -> (descriptors, detection scores [N,1]) -- the two arrays
        tester.generate_descriptor dumps per fragment (utils/tester.py)."""
        with use_params(self.store):
            return nb.assemble_FCNN_decoder(inputs, self.config, F, 1.0, with_scores=with_scores)

    def __call__(self, stacked_points, stacked_lengths, features=None, bbox=None, decoder=None, num_keypoints=None):
        """num_keypoints=k (decoder runs): the result also holds "keypoints", the KeypointSet of the k highest-scoring
        level-0 points of every cloud (keypoints.select_keypoints)."""
        inputs = self.build_inputs(stacked_points, stacked_lengths, features, bbox)
        F = self.encode(inputs)
        use_dec = self.has_decoder if decoder is None else decoder
        if num_keypoints is not None and not use_dec:
            raise ValueError("KPFCNN: num_keypoints needs the decoder (its detection scores)")
        desc, scores = self.describe(inputs, F, with_scores=True) if use_dec else (None, None)
        out = dict(inputs=inputs, F=F, descriptors=desc, scores=scores)
        if num_keypoints is not None:
            out["keypoints"] = select_keypoints(scores, inputs["lengths"][0], num_keypoints,
                                                points=inputs["points"][0], descriptors=desc)
        return out


class BatchPipeline:
    """Throughput mode: the input pyramid of batch i+1 is built on a second CUDA stream while the encoder of batch i
    runs -- the overlap the reference gets from tf.data prefetch (its CPU pyramid runs ahead of the GPU model,
    datasets/common.py:744-763). Usage:

        pipe = BatchPipeline(enc)
        pipe.prime(points0, lengths0, bbox0)            # pyramid of the first batch
        for i in range(K):
            out = pipe.step(points_next, lengths_next, bbox_next)   # encoder(i) || pyramid(i+1); returns F of batch i
        pipe.drain()
    """

    def __init__(self, enc, decoder=False, post=None):
        self.enc = enc
        self.decoder = decoder
        self.post = post                      # optional callable(inputs, F) run on the encoder stream (e.g. all-gather)
        dev = enc.device
        self.s_pyr = torch.cuda.Stream(device=dev)
        self.s_enc = torch.cuda.Stream(device=dev)
        self.ready = torch.cuda.Event()
        self.pending = None
        self.keep = []                        # keeps the previous batch's tensors alive until its kernels are done
        # Ring of pre-allocated pyramid slots: slot (i mod DEPTH) is rewritten by pyramid(i + DEPTH) only after the
        # host has waited for encoder(i) (self.done), so at most DEPTH - 1 encoders are ever queued behind the host
        # and steady-state batches allocate nothing for the pyramid.
        self.slots = [None] * self.DEPTH
        self.done = [None] * self.DEPTH
        self.n_built = 0

    DEPTH = 3

    def _slot(self, n_points, n_clouds):
        k = self.n_built % self.DEPTH
        self.n_built += 1
        if self.done[k] is not None:
            self.done[k].synchronize()        # the encoder that read this slot DEPTH batches ago has finished
        buf = self.slots[k]
        if buf is None or not buf.fits(n_points, n_clouds, self.enc.limits):
            buf = pyramid.PyramidBuffers(self.enc.config, self.enc.limits, int(n_points * 1.05) + 64, n_clouds,
                                         self.enc.device)
            self.slots[k] = buf
        return k, buf

    def _build(self, points, lengths, bbox, inputs_ready):
        k, buf = self._slot(int(points.shape[0]), int(lengths.shape[0]))
        self.s_pyr.wait_event(inputs_ready)   # caller-produced CUDA inputs are complete before the pyramid reads them
        with torch.cuda.stream(self.s_pyr):
            inputs = self.enc.build_inputs(points, lengths, bbox=bbox, buffers=buf)
            self.ready.record(self.s_pyr)
        for t in (points, lengths):           # caller tensors are read on the pyramid stream
            if torch.is_tensor(t) and t.is_cuda:
                t.record_stream(self.s_pyr)
        inputs["_slot"] = k
        for v in inputs.values():             # the pyramid's tensors are consumed on the encoder stream
            for t in (v if isinstance(v, (list, tuple)) else [v]):
                if torch.is_tensor(t) and t.is_cuda:
                    t.record_stream(self.s_enc)
        return inputs

    def _mark_inputs(self):
        """Event on the caller's current stream: everything the caller enqueued so far (the next batch's CUDA inputs)."""
        ev = torch.cuda.Event()
        ev.record(torch.cuda.current_stream(self.enc.device))
        return ev

    def prime(self, points, lengths, bbox=None):
        self.pending = self._build(points, lengths, bbox, self._mark_inputs())

    def step(self, next_points=None, next_lengths=None, next_bbox=None, pre=None):
        """Enqueue encoder(current batch) on the encoder stream, then build the pyramid of the next batch on the
        pyramid stream (the host blocks only in that stream's size read-backs). Returns the current batch's result.

        Stream contract: the result is produced on the private encoder stream; before returning, the CALLER's
        current stream is made to wait for it (an event, no host sync) and the result's memory is tied to that
        stream, so `res.cpu()` or a kernel launched on the caller's stream reads finished data."""
        inputs = self.pending
        cur = torch.cuda.current_stream(self.enc.device)
        # taken BEFORE `cur` is made to wait for this batch's encoder: the next pyramid then depends on the caller's
        # inputs only, not on encoder(i) -- the pyramid(i+1) || encoder(i) overlap is preserved
        inputs_ready = self._mark_inputs() if next_points is not None else None
        with torch.cuda.stream(self.s_enc):
            self.s_enc.wait_event(self.ready)
            if pre is not None:
                pre()
            F = self.enc.encode(inputs)
            res = self.enc.describe(inputs, F) if self.decoder else F[-1]
            if self.post is not None:
                res = self.post(inputs, res)
            ev = torch.cuda.Event()
            ev.record(self.s_enc)
            self.done[inputs["_slot"]] = ev
        cur.wait_event(ev)
        for t in (res if isinstance(res, (list, tuple)) else [res]):
            if torch.is_tensor(t) and t.is_cuda:
                t.record_stream(cur)
        self.result_event = ev
        self.keep = [inputs, F]
        self.pending = (self._build(next_points, next_lengths, next_bbox, inputs_ready)
                        if next_points is not None else None)
        return res

    def drain(self):
        self.s_pyr.synchronize()
        self.s_enc.synchronize()
        self.keep = []


class GraphPipeline:
    """Throughput / latency mode without the host in the loop: the whole step is two CUDA graph launches.

    The pyramid is built in its static form (capacity-sized launches, level sizes stay in device memory, no
    device->host read), the encoder's kernels take their row counts from the same device counters, so the launch
    sequence of a step depends only on the shape BUCKET (number of clouds, per-level capacities, scene bounds), not on
    the batch. Per ring slot the pyramid and the encoder are captured once and then replayed:

        pipe = GraphPipeline.for_batch(enc, points0, lengths0)     # one exact (synchronising) pass sizes the bucket
        pipe.prime(points, lengths)                                # H2D / D2D copy into the slot + pyramid graph
        for ...:
            res, counts = pipe.step(next_points, next_lengths)     # encoder graph (i) || pyramid graph (i+1)
        pipe.drain(); pipe.check()                                 # status bits: capacity overflow / points out of bounds

    `res` is the slot's static output buffer [capacity of the last level, C] and `counts` the device int32 level sizes
    (counts[l] for level l < L; rows of `res` beyond counts[L - 1] are undefined); both stay valid until the slot is
    reused DEPTH steps later. Mirrors the overlap the reference gets from tf.data prefetch (datasets/common.py:744-763).

    keypoints=k (needs decoder=True): the encoder graph also runs the detection scores and the per-cloud top-k
    selection, and `res` is a Detections(descriptors [cap0,32], scores [cap0,1], keypoints) whose KeypointSet holds
    the k highest-scoring level-0 points of every cloud -- slot buffers too, valid for the same DEPTH steps.

    match_pairs=[(src, tgt), ...] (needs keypoints): the encoder graph then also matches the keypoint descriptors of
    every pair (matching.match_keypoints), and `res` is a MatchedDetections(descriptors, scores, keypoints, matches).
    The pairs are fixed for the pipeline: KITTI's tester is [(0, 1)], a 3DMatch scene batch every i < j.

    register={...} (needs match_pairs): the keyword arguments of registration.register_pairs ({} for the 3DMatch
    evaluation's defaults). The encoder graph then also estimates every pair's pose by RANSAC over its matches, and
    `res` is a RegisteredDetections(descriptors, scores, keypoints, matches, registration).

    icp=dict(distance=...) (needs register): the keyword arguments of registration.icp_pairs (distance,
    max_iterations, relative_fitness, relative_rmse). The encoder graph then also refines every pair's RANSAC pose by
    point-to-point ICP over the level-0 clouds of the batch (its points, lengths and device row count, within the
    pipeline's bbox), and `res` is a RefinedDetections(descriptors, scores, keypoints, matches, registration,
    refinement).

    evaluate={...} (needs match_pairs): the keyword arguments of evaluation.evaluate_pairs ({} for the 3DMatch
    evaluation's defaults). Every batch then comes with its evaluation.GroundTruth of the match pairs, loaded into the
    slot with its points: prime(points, lengths, truth=...), step(next_points, next_lengths, next_truth=...). The
    encoder graph also scores the keypoints, the matches and, with register (and icp), the RANSAC (and ICP) poses
    against it, and `res` is an EvaluatedDetections(descriptors, scores, keypoints, matches, registration, refinement,
    evaluation) with that step's per-pair metrics and totals. step() adds the step's totals into a running fp64 vector
    on the caller's stream, in step order; evaluation_totals() reads it (one device->host read, for
    evaluation.summary(totals, pipe.evaluate_levels, pipe.evaluate_pose_sets)) and reset_evaluation() zeroes it.

    voxel_size=v (with raw_capacity, the raw rows a slot holds): batches are raw scans. prime / step take the raw
    points and lengths, and the pyramid graph starts with voxel.voxel_down_sample's static form, which writes the slot's
    level 0 (points, lengths, row count) on the device: raw scans in, the reference's voxel_down_sample(v) input stage
    inside the graph, no host step. Capacities and bbox are those of the voxelised level 0 (for_batch sizes them from
    one voxelised batch); more voxels than capacities[0] set status bit 1, a cloud wider than the bbox allows bit 0.
    Keypoints, ICP and the evaluation see the voxelised level 0.

    sweep=dict(counts=(5000, 2500, 1000, 500, 250), arms=("score", "random"), seed=0) (needs match_pairs): D3Feat's
    keypoint-count experiment, the testers' `-pred` and `-rand` arms. counts descend strictly and are at most
    keypoints; arms is a non-empty subset of ("score", "random"). The encoder graph then also runs, for every (arm,
    count), the pipeline's matching, registration, ICP and evaluation on that arm's keypoint set, and `res` is a
    SweptDetections: the fields of the pipeline's regular result plus sweep, a dict (arm, count) -> SweepEntry(keypoints,
    matches, registration, refinement, evaluation). The score arm at count c is select_keypoints(k=c), exactly the
    keypoints of a pipeline built with keypoints=c. The random arm draws counts[0] uniform slots per cloud, with
    replacement (keypoints.sample_keypoints with the sweep's seed, one draw per step and cloud, shared by every pair of
    the cloud); count c is its first c slots, which sample_keypoints(k=c) gathers directly (each slot is its own draw).
    With evaluate, the repeatability levels are checked against the smallest count, and every stage, the regular result
    included, uses them; evaluation_totals() is then [len(arms), len(counts), n_tot], for evaluation.sweep_summary(totals,
    pipe.sweep_arms, pipe.sweep_counts, pipe.evaluate_levels, pipe.evaluate_pose_sets)."""

    DEPTH = 4

    def __init__(self, enc, capacities, n_clouds, bbox, decoder=False, post=None, encoder_streams=2, keypoints=None,
                 match_pairs=None, register=None, icp=None, evaluate=None, voxel_size=None, raw_capacity=None,
                 sweep=None):
        if keypoints is not None and not decoder:
            raise ValueError("GraphPipeline: keypoints=%r needs decoder=True (the detection scores)" % (keypoints,))
        if keypoints is not None and int(keypoints) < 1:
            raise ValueError("GraphPipeline: keypoints=%r must be >= 1" % (keypoints,))
        if match_pairs is not None and keypoints is None:
            raise ValueError("GraphPipeline: match_pairs needs keypoints=k (the descriptors it matches)")
        self.sweep_counts = self.sweep_arms = self.sweep_seed = None
        if sweep is not None:
            if match_pairs is None:
                raise ValueError("GraphPipeline: sweep needs match_pairs (the pairs every keypoint count is matched on)")
            self.sweep_counts, self.sweep_arms, self.sweep_seed = check_sweep(sweep, int(keypoints))
        if voxel_size is not None and raw_capacity is None:
            raise ValueError("GraphPipeline: voxel_size needs raw_capacity (the raw rows a slot holds)")
        if register is not None:
            if match_pairs is None:
                raise ValueError("GraphPipeline: register needs match_pairs (the matches it registers)")
            if not isinstance(register, dict) or set(register) - set(REGISTER_OPTIONS):
                raise ValueError("GraphPipeline: register must be a dict of register_pairs options %s, got %r" % (
                    REGISTER_OPTIONS, register))
            check_options(**register, who="GraphPipeline")
        if icp is not None:
            if register is None:
                raise ValueError("GraphPipeline: icp needs register (the RANSAC poses it refines)")
            if not isinstance(icp, dict) or set(icp) - set(ICP_OPTIONS) or "distance" not in icp:
                raise ValueError("GraphPipeline: icp must be a dict of icp_pairs options %s with a distance, got %r" % (
                    ICP_OPTIONS, icp))
            check_icp_options(**icp, who="GraphPipeline")
        if evaluate is not None:
            if match_pairs is None:
                raise ValueError("GraphPipeline: evaluate needs match_pairs (the pairs it scores)")
            if not isinstance(evaluate, dict) or set(evaluate) - set(EVALUATE_OPTIONS):
                raise ValueError("GraphPipeline: evaluate must be a dict of evaluate_pairs options %s, got %r" % (
                    EVALUATE_OPTIONS, evaluate))
            k_min = int(keypoints) if sweep is None else self.sweep_counts[-1]
            self.evaluate_levels = check_evaluate_options(k_min, **evaluate, who="GraphPipeline")[0]
            self.evaluate_pose_sets = ("ransac",) * (register is not None) + ("icp",) * (icp is not None)
        self.evaluate = None if evaluate is None else dict(evaluate)
        if sweep is not None and evaluate is not None:
            self.evaluate["repeat_levels"] = self.evaluate_levels     # one set of levels for every count
        self.icp = None if icp is None else dict(icp)
        pairs = None if match_pairs is None else host_pairs(match_pairs, int(n_clouds), "GraphPipeline")
        self.register = None if register is None else dict(register)
        self.keypoints = None if keypoints is None else int(keypoints)
        self.enc, self.decoder, self.post = enc, decoder, post
        dev = enc.device
        self.match_pairs = None if pairs is None else torch.from_numpy(pairs).to(dev)
        self.caps = [int(c) for c in capacities]
        self.n_clouds = int(n_clouds)
        self.bbox = np.ascontiguousarray(bbox, np.float32)
        self.s_pyr = torch.cuda.Stream(device=dev)
        # Encoders of consecutive batches alternate between `encoder_streams` streams: the deep pyramid levels (a few
        # thousand rows) cannot fill 132 SMs on their own, so the tail of encoder(i) runs under the level-0 kernels of
        # encoder(i + 1). Results still come back in batch order (each step waits for its own batch's event).
        self.s_encs = [torch.cuda.Stream(device=dev) for _ in range(max(1, int(encoder_streams)))]
        self.s_enc = self.s_encs[0]
        self.n_stepped = 0
        self.DEPTH = len(self.s_encs) + 2     # encoders in flight + the pyramid being built + one slot of slack
        self.slots = [pyramid.PyramidBuffers(enc.config, enc.limits, self.caps, self.n_clouds, dev, bbox=self.bbox)
                      for _ in range(self.DEPTH)]
        # per slot: the raw batch and the voxel stage that writes the slot's level 0
        self.voxel = (None if voxel_size is None else
                      [VoxelStage(raw_capacity, self.n_clouds, voxel_size, self.bbox, dev) for _ in range(self.DEPTH)])
        self.g_pyr = [None] * self.DEPTH
        self.g_enc = [None] * self.DEPTH
        self.out = [None] * self.DEPTH          # (inputs, F, res) captured per slot
        self.ready = [torch.cuda.Event() for _ in range(self.DEPTH)]
        self.done = [None] * self.DEPTH
        self.kernels_per_step = 0
        self.n_loaded = 0
        self.pending = None
        if self.evaluate is not None:
            P = int(self.match_pairs.shape[0])
            f64 = torch.float64
            # per slot: the batch's truth, loaded with its points (info always present; bit 1 cleared without one)
            self.truth = [GroundTruth(torch.zeros((P, 4, 4), dtype=f64, device=dev),
                                      torch.zeros((P, 6, 6), dtype=f64, device=dev),
                                      torch.zeros((P,), dtype=torch.int32, device=dev)) for _ in range(self.DEPTH)]
            n_tot = 4 + len(self.evaluate_levels) + 7 * len(self.evaluate_pose_sets)
            shape = (n_tot,) if sweep is None else (len(self.sweep_arms), len(self.sweep_counts), n_tot)
            self.eval_running = torch.zeros(shape, dtype=f64, device=dev)
            self.sweep_totals = [None] * self.DEPTH     # per slot: the step's sweep totals, stacked in the graph

    @classmethod
    def for_batch(cls, enc, points, lengths, slack=1.125, margin=0.05, **kw):
        """Bucket from a representative batch: one exact pass gives the level sizes (capacities = sizes x slack) and
        the scene bounds (its bbox inflated by `margin` of the extent on every side). With voxel_size=v the batch is
        raw: it is voxelised once (voxel.voxel_down_sample) and sizes the bucket as above, and the raw capacity is its
        row count x slack rounded up to 256."""
        if kw.get("voxel_size") is not None:
            dev = enc.device
            points = (points if torch.is_tensor(points) else
                      torch.as_tensor(np.ascontiguousarray(points, np.float32))).to(dev)
            lengths = (lengths if torch.is_tensor(lengths) else
                       torch.as_tensor(np.ascontiguousarray(lengths, np.int32))).to(dev)
            kw.setdefault("raw_capacity", max(-(-int(int(points.shape[0]) * slack) // 256) * 256, 256))
            points, lengths = voxel_down_sample(points, lengths, kw["voxel_size"])
        inputs = enc.build_inputs(points, lengths)
        sizes = [int(p.shape[0]) for p in inputs["points"]]
        pts = inputs["points"][0]
        bb = pyramid.ops.host_bbox(pts)
        ext = np.maximum(bb[3:] - bb[:3], 1e-3)
        bb = np.concatenate([bb[:3] - margin * ext, bb[3:] + margin * ext]).astype(np.float32)
        return cls(enc, pyramid.bucket_capacities(sizes, slack), int(lengths.shape[0]), bb, **kw)

    # ---- one slot -----------------------------------------------------------------------------------------
    def _run_pyramid(self, k):
        if self.voxel is not None:
            buf = self.slots[k]
            self.voxel[k].run(buf.points0, buf.lengths0, buf.n0, buf.status)
        return self.enc.build_inputs_static(self.slots[k])

    def _run_encoder(self, inputs, k):
        F = self.enc.encode(inputs)
        if self.keypoints is not None:
            desc, scores = self.enc.describe(inputs, F, with_scores=True)
            kp = select_keypoints(scores, inputs["lengths"][0], self.keypoints, points=inputs["points"][0],
                                  descriptors=desc, rows=inputs["rows"][0])
            if self.match_pairs is not None:
                m, reg, ref, ev = self._run_pairs(inputs, k, kp)
                if self.sweep_counts is not None:
                    return F, self._run_sweep(inputs, k, desc, scores, SweepEntry(kp, m, reg, ref, ev))
                if ev is not None:
                    return F, EvaluatedDetections(desc, scores, kp, m, reg, ref, ev)
                if ref is not None:
                    return F, RefinedDetections(desc, scores, kp, m, reg, ref)
                if reg is not None:
                    return F, RegisteredDetections(desc, scores, kp, m, reg)
                return F, MatchedDetections(desc, scores, kp, m)
            return F, Detections(desc, scores, kp)
        res = self.enc.describe(inputs, F) if self.decoder else F[-1]
        return F, res

    def _run_pairs(self, inputs, k, kp):
        """(matches, registration, refinement, evaluation) of the match pairs on the keypoint set kp, None for the
        stages the pipeline does not run."""
        m = match_keypoints(kp, self.match_pairs)
        reg = ref = ev = None
        if self.register is not None:
            reg = register_pairs(kp, m, self.match_pairs, **self.register)
            if self.icp is not None:
                ref = icp_pairs(inputs["points"][0], inputs["lengths"][0], self.match_pairs, reg.pose,
                                rows=inputs["rows"][0], bbox=self.bbox, **self.icp)
        if self.evaluate is not None:
            ev = evaluate_pairs(kp, m, self.match_pairs, self.truth[k], reg, ref, **self.evaluate)
        return m, reg, ref, ev

    def _run_sweep(self, inputs, k, desc, scores, main):
        """Every (arm, count) of the sweep on slot k, after the regular result `main` (a SweepEntry). The score arm at
        count == keypoints is `main` itself; the random arm's count c is the first c slots of the counts[0] draw, drawn
        directly with k=c."""
        pts, lens, rows = inputs["points"][0], inputs["lengths"][0], inputs["rows"][0]
        entries = {}
        for arm in self.sweep_arms:
            for c in self.sweep_counts:
                if arm == "score" and c == self.keypoints:
                    entries[(arm, c)] = main
                    continue
                if arm == "score":
                    kp = select_keypoints(scores, lens, c, points=pts, descriptors=desc, rows=rows)
                else:
                    kp = sample_keypoints(lens, c, self.sweep_seed, points=pts, descriptors=desc, scores=scores,
                                          rows=rows)
                entries[(arm, c)] = SweepEntry(kp, *self._run_pairs(inputs, k, kp))
        if self.evaluate is not None:
            self.sweep_totals[k] = torch.stack([e.evaluation.totals for e in entries.values()]).view(
                self.eval_running.shape)
        return SweptDetections(desc, scores, *main, entries)

    def _capture(self, k):
        """Eager warm-up of both halves on slot k (lazy one-time work: weight packing, BN folding, kernel attributes,
        the library's auxiliary stream), then the two captures."""
        from . import _lib
        for _ in range(2):
            with torch.cuda.stream(self.s_pyr):
                inputs = self._run_pyramid(k)
            self.s_enc.wait_stream(self.s_pyr)
            with torch.cuda.stream(self.s_enc):
                self._run_encoder(inputs, k)
            self.s_pyr.wait_stream(self.s_enc)
        torch.cuda.synchronize(self.enc.device)
        n0 = _lib.launch_count()
        gp = torch.cuda.CUDAGraph()
        with torch.cuda.graph(gp, stream=self.s_pyr):
            inputs = self._run_pyramid(k)
        ge = torch.cuda.CUDAGraph()
        with torch.cuda.graph(ge, stream=self.s_enc):
            F, res = self._run_encoder(inputs, k)
        self.kernels_per_step = _lib.launch_count() - n0
        self.g_pyr[k], self.g_enc[k], self.out[k] = gp, ge, (inputs, F, res)

    def _check_batch(self, points, lengths, truth):
        """ValueError unless the batch fits the slots (raw or level-0 rows, number of clouds) and comes with the truth
        the pipeline needs. Changes nothing: a rejected batch leaves the pipeline as it was."""
        if self.evaluate is not None and truth is None:
            raise ValueError("GraphPipeline: evaluate needs the truth of every batch (prime(..., truth=...), "
                             "step(..., next_truth=...))")
        if self.evaluate is None and truth is not None:
            raise ValueError("GraphPipeline: truth given to a pipeline built without evaluate")
        if truth is not None:
            check_truth(truth, int(self.match_pairs.shape[0]), "GraphPipeline")
        n0 = int(points.shape[0])
        cap = int(self.slots[0].points0.shape[0]) if self.voxel is None else self.voxel[0].capacity
        if n0 > cap or int(lengths.shape[0]) != self.n_clouds:
            raise ValueError("GraphPipeline: batch (%d points, %d clouds) does not fit the bucket (%d, %d)" % (
                n0, int(lengths.shape[0]), cap, self.n_clouds))

    def _load(self, points, lengths, inputs_ready, truth=None):
        """Copy a batch that passed _check_batch into the next slot and replay its pyramid graph."""
        k = self.n_loaded % self.DEPTH
        self.n_loaded += 1
        if self.done[k] is not None:
            self.done[k].synchronize()        # bounds the host's run-ahead to DEPTH steps (normally long complete)
        buf = self.slots[k]
        # the batch goes into the slot's level 0, or with voxel_size into its raw buffers
        dst = (buf.points0, buf.lengths0, buf.n0) if self.voxel is None else \
            (self.voxel[k].points, self.voxel[k].lengths, self.voxel[k].n)
        n0 = int(points.shape[0])
        if self.g_pyr[k] is None:             # first use of the slot: fill it, then capture its two graphs
            dst[0][:n0].copy_(torch.as_tensor(points), non_blocking=True)
            dst[1].copy_(torch.as_tensor(lengths), non_blocking=True)
            dst[2].fill_(n0)
            torch.cuda.synchronize(self.enc.device)
            self._capture(k)
        self.s_pyr.wait_event(inputs_ready)
        with torch.cuda.stream(self.s_pyr):
            dst[0][:n0].copy_(torch.as_tensor(points), non_blocking=True)
            dst[1].copy_(torch.as_tensor(lengths), non_blocking=True)
            dst[2].fill_(n0)
            if truth is not None:
                self._load_truth(k, truth)
            self.g_pyr[k].replay()
            self.ready[k].record(self.s_pyr)
        for t in [points, lengths] + ([] if truth is None else [x for x in truth if x is not None]):
            if torch.is_tensor(t) and t.is_cuda:
                t.record_stream(self.s_pyr)
        return k

    def _load_truth(self, k, truth):
        """Copy a batch's truth into slot k (on the current stream); without info, flags bit 1 is cleared."""
        dst = self.truth[k]
        for d, x in ((dst.pose, truth.pose), (dst.flags, truth.flags)):
            d.copy_(x if torch.is_tensor(x) else torch.from_numpy(np.ascontiguousarray(x)), non_blocking=True)
        if truth.info is None:
            dst.flags.bitwise_and_(1)
        else:
            x = truth.info
            dst.info.copy_(x if torch.is_tensor(x) else torch.from_numpy(np.ascontiguousarray(x)), non_blocking=True)

    def _mark_inputs(self):
        ev = torch.cuda.Event()
        ev.record(torch.cuda.current_stream(self.enc.device))
        return ev

    def prime(self, points, lengths, truth=None):
        self._check_batch(points, lengths, truth)
        self.pending = self._load(points, lengths, self._mark_inputs(), truth)

    def step(self, next_points=None, next_lengths=None, pre=None, next_truth=None):
        """Replay encoder(current batch), then load + replay the pyramid of the next batch on the other stream.
        Returns (result buffer, device level counts) of the current batch, ordered on the caller's stream.

        A next batch that does not fit (too many rows, another number of clouds, missing or malformed truth) raises
        ValueError before anything runs: the current batch stays pending, and the next step() returns it once.

        A batch that outgrows the bucket on the device is not refused: its step runs on a defined truncation and sets
        the slot's status word (see check()). counts[0] is then at most capacities[0] (with voxel_size, the first
        capacities[0] voxels in (cloud, iz, iy, ix) order are kept). When subsampling level l - 1 fails, counts[l] is
        -1 (a cloud wider than the bbox allows, status bit 0) or -2 (more cells than capacities[l], status bit 1), and
        every deeper count is <= 0: those levels have no rows, their pool and upsample rows name no support, and every
        output of the step stays finite."""
        if next_points is not None:
            self._check_batch(next_points, next_lengths, next_truth)
        k = self.pending
        cur = torch.cuda.current_stream(self.enc.device)
        inputs_ready = self._mark_inputs() if next_points is not None else None
        inputs, F, res = self.out[k]
        s_enc = self.s_encs[self.n_stepped % len(self.s_encs)]
        self.n_stepped += 1
        self.s_enc = s_enc                    # the stream this step's result is produced on
        with torch.cuda.stream(s_enc):
            s_enc.wait_event(self.ready[k])
            if pre is not None:
                pre()
            self.g_enc[k].replay()
            if self.post is not None:
                res = self.post(inputs, res)
            ev = torch.cuda.Event()
            ev.record(s_enc)
            self.done[k] = ev
        cur.wait_event(ev)
        if self.evaluate is not None:
            # on the caller's stream, after this step's encoder: consecutive encoders may overlap on their two
            # streams, so the running totals are never written inside a graph
            self.eval_running.add_(self.out[k][2].evaluation.totals if self.sweep_counts is None else
                                   self.sweep_totals[k])
        self.pending = (self._load(next_points, next_lengths, inputs_ready, next_truth)
                        if next_points is not None else None)
        return res, self.slots[k].counts

    def evaluation_totals(self):
        """The running totals of every step since construction or reset_evaluation(), as float64 numpy (one
        device->host read on the caller's stream, after the pyramid of the pending batch): see evaluation.summary.
        Raises RuntimeError, as check() does, once any batch loaded so far has overflowed the bucket: its totals
        were computed on truncated clouds. With sweep the totals are [len(sweep_arms), len(sweep_counts), n_tot]."""
        cur = torch.cuda.current_stream(self.enc.device)
        cur.wait_stream(self.s_pyr)
        status = torch.cat([buf.status for buf in self.slots]).to(torch.float64)
        n = self.eval_running.numel()
        got = torch.cat([self.eval_running.reshape(-1), status]).cpu().numpy()
        self._raise_on_status(got[n:].astype(np.int64))
        return got[:n].reshape(self.eval_running.shape)

    def reset_evaluation(self):
        """Zero the running totals. The status words stay set: see check()."""
        self.eval_running.zero_()

    def drain(self):
        self.s_pyr.synchronize()
        for s in self.s_encs:
            s.synchronize()

    def check(self):
        """Raise if any batch loaded so far overflowed the bucket (synchronises). The status words are sticky: they
        are never cleared, so once one is set check() and evaluation_totals() raise for the rest of the pipeline's
        life; a bucket that has overflowed has to be rebuilt larger."""
        self.drain()
        self._raise_on_status([int(buf.status.item()) for buf in self.slots])

    @staticmethod
    def _raise_on_status(status):
        for k, st in enumerate(status):
            if st:
                raise RuntimeError("GraphPipeline: slot %d status %d (%s)" % (
                    k, st, "a cloud wider than the scene bounds" if st & 1 else "a level exceeded its capacity"))
