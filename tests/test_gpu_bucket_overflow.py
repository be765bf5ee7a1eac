"""GraphPipeline on batches that outgrow the bucket it was sized for: the step that overflows, and every step after it.

One small bucket (17 clouds, capacities CAPS, a 2 m scene box) runs every stage: the voxel stage (voxel_size, or
without it for the level overflows), the pyramid, the encoder and decoder, 64 keypoints, matching, RANSAC, ICP and the
evaluation. Its regular batches are the B17 serving batches of tests/test_gpu_many_clouds_serving.py; each is checked
once against the oracles (check_chain on its static form) and once through a fresh pipeline, the reference.

The overflowing batches are made from data only, and the CPU tests at the end show with the oracles that each one hits
its condition and nothing else:
* more voxels than capacities[0]: status bit 1, level 0 = the C port's voxelisation cut to its first capacities[0]
  voxels, and everything downstream equal to check_chain on that level 0;
* more cells at level l than capacities[l], l = 1 .. 4 on its own: status bit 1, counts[l] = -2, every deeper count
  <= 0, the levels above and the kept cells of level l equal to the oracle pyramid, the upsample rows into level l all
  padding, no index row written past its count, every float output finite and two replays bit-identical;
* one cloud wider than the scene box (bit 0, counts[1] = -1), and that together with the voxel overflow (bits 0 and 1);
* one cloud moved 5 and 50 box extents away, width unchanged: no bit, the whole chain exact, ICP included.
After every overflow the following steps, through the overflowed slot and the others, equal the reference bit for bit.
The status word is sticky: check() and evaluation_totals() raise to the end, reset_evaluation() does not clear it.
A next batch refused with ValueError (too many raw rows, wrong cloud count, bad or missing truth) changes nothing: the
pending batch comes back once and the running totals equal those of a pipeline that never saw it."""
import functools

import numpy as np
import pytest
import torch

from oracle.voxel_native import port_voxel_down_sample

from test_gpu_many_clouds import LIMITS, SENTINEL, bits, clip_lengths, expected_pyramid, oracle_pyramid
from test_gpu_many_clouds_serving import ICP, K, REGISTER, check_chain, fields, pairs_for, serving_batch, static_run, t
from test_gpu_voxel_serving import same_bits, snapshot

V = 0.025                                    # voxel size of the raw batches (finer than the scene's 3 cm spacing)
CAPS = [1536, 1024, 768, 512, 256]           # the bucket: >= 1.25 x every regular batch's level size + 64
RAW_CAP = 2048                               # raw rows a slot holds
B = 17
EVALUATE = dict(repeat_levels=[4, 16, 64])
STATUS_WIDE, STATUS_CAPACITY = 1, 2


# ---- batches ----------------------------------------------------------------------------------------------------------

def config():
    from d3feat_b200 import synth
    return synth.Config(architecture=synth.ARCH_3DMATCH)


def level_dl(l):
    """The grid size of the subsampling that makes level l (1 .. 4)."""
    from d3feat_b200 import pyramid as pyr
    return pyr._level_radii(config())[l - 1]["dl"]


@functools.lru_cache(maxsize=None)
def good():
    """The regular batches: B17 serving batches 0 .. 4 (level-0 clouds, or raw scans for the voxel stage)."""
    return [serving_batch("B17", v) for v in range(5)]


PAIRS = pairs_for(good()[0][1])


def truth():
    from d3feat_b200.evaluation import GroundTruth
    P = len(PAIRS)
    return GroundTruth(np.tile(np.eye(4), (P, 1, 1)), None, np.ones(P, np.int32))


@functools.lru_cache(maxsize=None)
def bbox():
    """A 2 m cube around every regular batch."""
    P = np.concatenate([p for p, _ in good()], 0)
    c = (P.min(0) + P.max(0)) / 2
    return np.concatenate([c - 1.0, c + 1.0]).astype(np.float32)


def clouds_of(P, L):
    assert int(np.sum(L)) == len(P)
    start = np.concatenate([[0], np.cumsum(L)])
    return [P[start[b]:start[b + 1]] for b in range(len(L))]


def stack(clouds):
    return (np.ascontiguousarray(np.concatenate(clouds, 0), np.float32),
            np.array([len(c) for c in clouds], np.int32))


def lattice(n, spacing, centre):
    """The first n points of a cubic lattice around centre. spacing > the grid size puts every point in a cell of its
    own, whatever the grid's origin."""
    side = int(np.ceil(n ** (1 / 3) - 1e-9))
    ijk = np.stack(np.meshgrid(*[np.arange(side)] * 3, indexing="ij"), -1).reshape(-1, 3)[:n]
    return (centre + (ijk - (side - 1) / 2) * spacing).astype(np.float32)


def fill_empty(P, L, n, spacing, which=None):
    """The batch with n lattice points spread over its empty clouds (or the clouds `which`)."""
    clouds = clouds_of(P, L)
    empty = [b for b in range(len(L)) if L[b] == 0] if which is None else list(which)
    centre = (bbox()[:3] + bbox()[3:]) / 2
    per = -(-n // len(empty))
    for b in empty:
        m = min(per, n)
        clouds[b] = lattice(m, spacing, centre)
        n -= m
    return stack(clouds)


BIG = 13                                     # the 450-point cloud of batch 0
WIDE = 3                                     # a 31-point random subset of the whole room in batch 0


def reshaped(P, L, how):
    """Cloud WIDE scaled 60 times about its mean ("wide": its voxel stage can merge at most 31 voxels), or cloud BIG
    moved by f box extents ("moved<f>")."""
    clouds = clouds_of(P, L)
    if how == "wide":
        c = clouds[WIDE]
        m = c.mean(0)
        clouds[WIDE] = m + (c - m) * np.float32(60.0)
    else:
        clouds[BIG] = clouds[BIG] + float(how[5:]) * (bbox()[3:] - bbox()[:3])
    return stack(clouds)


@functools.lru_cache(maxsize=None)
def voxel_overflow():
    """Batch 0 with three lattice clouds appended (clouds 14-16, one point per voxel): 96 voxels more than CAPS[0]."""
    P, L = good()[0]
    M = len(port_voxel_down_sample(P, L, V)[0])
    return fill_empty(P, L, CAPS[0] - M + 96, 1.7 * V, which=(14, 15, 16))


@functools.lru_cache(maxsize=None)
def level_overflow(l):
    """Batch 4 (one cloud of 300 points) with lattice clouds in its 16 empty clouds, one point per level-l cell: 32
    cells more than CAPS[l] at level l, within every capacity above it."""
    P, L = good()[4]
    sizes = [p.shape[0] for p in oracle_pyramid(config(), P, L)["points"]]
    return fill_empty(P, L, CAPS[l] - sizes[l] + 32, 1.7 * level_dl(l))


@functools.lru_cache(maxsize=None)
def case_batch(case):
    if case == "voxel":
        return voxel_overflow()
    if case == "wide":
        return reshaped(*good()[0], "wide")
    if case == "both":
        return reshaped(*voxel_overflow(), "wide")
    if case.startswith("moved"):
        return reshaped(*good()[0], case)
    return level_overflow(int(case[5:]))


def truncated_voxels(P, L):
    """The C port's voxelisation cut to its first CAPS[0] voxels (cloud, iz, iy, ix order), lengths to match."""
    vp, vl = port_voxel_down_sample(P, L, V)
    return vp[:CAPS[0]], clip_lengths(vl, CAPS[0])


# ---- pipelines --------------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def model(cuda):
    from d3feat_b200 import synth
    from d3feat_b200.encoder import KPFCNN
    cfg = config()
    return KPFCNN(cfg, synth.make_params(cfg, 0), LIMITS, device=cuda)


def make_pipe(model, voxel):
    from d3feat_b200.encoder import GraphPipeline
    return GraphPipeline(model, CAPS, B, bbox(), decoder=True, keypoints=K, match_pairs=PAIRS, register=REGISTER,
                         icp=ICP, evaluate=EVALUATE, voxel_size=V if voxel else None,
                         raw_capacity=RAW_CAP if voxel else None)


@pytest.fixture
def voxel_pipe(model):
    """A fresh bucket with every stage on, raw scans in."""
    return make_pipe(model, True)


@pytest.fixture
def plain_pipe(model):
    """The same bucket without voxel_size: level-0 clouds in."""
    return make_pipe(model, False)


def run(pipe, feed, before=None, after=None):
    """prime + one step per batch of feed; returns the snapshot of every step. before(i, pipe) runs before the step that
    loads feed[i], after(i, k, res, counts) once step i has returned (synchronised; k: the slot of feed[i])."""
    cuda = pipe.enc.device
    pipe.prime(t(feed[0][0], cuda), t(feed[0][1], cuda), truth=truth())
    snaps = []
    for i in range(len(feed)):
        if before is not None and i + 1 < len(feed):
            before(i + 1, pipe)
        k = pipe.pending
        nxt = feed[i + 1] if i + 1 < len(feed) else None
        res, counts = (pipe.step(t(nxt[0], cuda), t(nxt[1], cuda), next_truth=truth()) if nxt else pipe.step())
        torch.cuda.synchronize()
        snaps.append(snapshot(res, counts))
        if after is not None:
            after(i, k, res, counts)
    pipe.drain()
    return snaps


def level0(P, L, voxel):
    return port_voxel_down_sample(P, L, V) if voxel else (P, L)


def eager_chain(model, pipe, P, L, what, seed):
    """check_chain on the static form of level-0 clouds (P, L); returns (level counts, fields of the chain)."""
    tr, inputs, res = static_run(model, pipe, P, L)
    check_chain(tr, P, L, len(P), *res, PAIRS, what, seed=seed)
    return inputs["counts"][:5].cpu().tolist(), fields(res, len(P))


def assert_step_equals_chain(snap, chain, what):
    counts, want = chain
    assert snap["counts"][:5].tolist() == counts, (what, snap["counts"], counts)
    for name, a in want.items():
        assert same_bits(snap[name], a.cpu().numpy()), (what, name)


def reference(model, voxel):
    """The regular batches through a fresh pipeline, each step equal to check_chain on its level 0."""
    pipe = make_pipe(model, voxel)
    snaps = run(pipe, good())
    pipe.check()
    for i, (P, L) in enumerate(good()):
        chain = eager_chain(model, pipe, *level0(P, L, voxel), "reference %d" % i, i)
        assert_step_equals_chain(snaps[i], chain, "reference %d" % i)
    return snaps, pipe.evaluation_totals()


@pytest.fixture(scope="module")
def voxel_reference(model):
    return reference(model, True)


@pytest.fixture(scope="module")
def plain_reference(model):
    return reference(model, False)


def assert_same_steps(got, want, what):
    assert set(got) == set(want)
    bad = [k for k in got if not same_bits(got[k], want[k])]
    assert bad == [], (what, bad)


# Regular batches 0 .. 3 fill (and capture) the four slots; the overflowing batch then lands in slot 0 and the regular
# batches after it pass through every slot, slot 0 again included.
BEFORE = [0, 1, 2, 3]
AFTER = [4, 0, 1, 2]


def statuses(pipe):
    pipe.drain()
    return [int(buf.status.item()) for buf in pipe.slots]


def assert_sticky(pipe):
    """check() and evaluation_totals() raise, and keep raising after reset_evaluation()."""
    for _ in range(2):
        with pytest.raises(RuntimeError, match="status"):
            pipe.check()
        with pytest.raises(RuntimeError, match="status"):
            pipe.evaluation_totals()
        pipe.reset_evaluation()


def assert_finite(snap, what):
    for name in ("descriptors", "scores", "keypoints.points", "keypoints.descriptors", "keypoints.scores",
                 "matches.sim_st", "matches.sim_ts", "registration.pose", "refinement.pose"):
        assert np.isfinite(snap[name]).all(), (what, name)


def assert_later_steps(snaps, n_bad, ref, what):
    for j, g in enumerate(BEFORE):
        assert_same_steps(snaps[j], ref[g], "%s: step %d before" % (what, j))
    for j, g in enumerate(AFTER):
        i = len(BEFORE) + n_bad + j
        assert_same_steps(snaps[i], ref[g], "%s: step %d after" % (what, i))


# ---- more voxels than capacities[0] -----------------------------------------------------------------------------------

@pytest.mark.gpu
def test_voxel_overflow_is_a_defined_truncation(model, voxel_pipe, voxel_reference):
    ref, _ = voxel_reference
    bad = case_batch("voxel")
    feed = [good()[g] for g in BEFORE] + [bad] + [good()[g] for g in AFTER]
    seen = {}

    def after(i, k, res, counts):
        if i == len(BEFORE):
            buf = voxel_pipe.slots[k]
            seen["slot"] = k
            seen["points0"] = buf.points0.cpu().numpy()
            seen["lengths0"] = buf.lengths0.cpu().numpy()
            seen["n0"] = int(buf.n0.item())

    snaps = run(voxel_pipe, feed, after=after)
    st = statuses(voxel_pipe)
    print("voxel overflow: status %s, counts %s" % (st, snaps[len(BEFORE)]["counts"][:5].tolist()))
    assert st == [STATUS_CAPACITY if k == seen["slot"] else 0 for k in range(len(st))]
    vp, vl = truncated_voxels(*bad)
    assert seen["n0"] == CAPS[0] == len(vp)
    assert np.array_equal(bits(seen["points0"][:CAPS[0]]), bits(vp))
    assert np.array_equal(seen["lengths0"], vl)
    assert 0 < vl[-1] < port_voxel_down_sample(*bad, V)[1][-1]         # the cut falls inside the last cloud
    chain = eager_chain(model, voxel_pipe, vp, vl, "voxel overflow", 7)
    assert_step_equals_chain(snaps[len(BEFORE)], chain, "voxel overflow")
    assert_later_steps(snaps, 1, ref, "voxel overflow")
    assert_sticky(voxel_pipe)


# ---- more cells at level l than capacities[l] -------------------------------------------------------------------------

def guard(pipe, k):
    """Slot k's index matrices and deeper levels filled with SENTINEL; its captured encoder outputs (the per-level
    features the decoder reads, the descriptors and scores) with NaN."""
    torch.cuda.synchronize()
    buf = pipe.slots[k]
    for x in buf.pts[1:] + buf.len[1:] + buf.nb + buf.pool + buf.up:
        if x is not None:
            x.view(torch.int32).fill_(int(SENTINEL))
    _, F, res = pipe.out[k]
    for x in list(F) + [res.descriptors, res.scores]:
        x.fill_(float("nan"))
    torch.cuda.synchronize()


def check_overflowed_slot(pipe, k, P, L, l, counts):
    """Slot k after a step whose level l overflowed: levels above l equal the oracle, level l holds the oracle's first
    CAPS[l] cells, the upsample rows into level l are all padding (the device count, -2), and no matrix row at or past
    what its count allows was written. The per-level features are finite up to their counts."""
    ref = oracle_pyramid(config(), P, L)
    exp = expected_pyramid(ref, len(P))
    buf = pipe.slots[k]
    c = counts[:5]
    assert c[:l] == exp["sizes"][:l] and exp["sizes"][l] > CAPS[l], (c, exp["sizes"])
    assert c[l] == -2 and all(x <= 0 for x in c[l + 1:]), c
    for m in range(l):
        n = c[m]
        if m > 0:
            assert np.array_equal(bits(buf.pts[m][:n].cpu().numpy()), bits(exp["points"][m])), m
            assert np.array_equal(buf.len[m].cpu().numpy(), exp["lengths"][m]), m
        assert np.array_equal(buf.nb[m][:n].cpu().numpy(), exp["neighbors"][m]), m
        if m + 1 < l:
            assert np.array_equal(buf.pool[m][:c[m + 1]].cpu().numpy(), exp["pools"][m]), m
            assert np.array_equal(buf.up[m][:n].cpu().numpy(), exp["upsamples"][m]), m
    assert (buf.up[l - 1][:c[l - 1]].cpu().numpy() == -2).all()
    assert np.array_equal(bits(buf.pts[l].cpu().numpy()), bits(ref["points"][l][:CAPS[l]]))
    assert np.array_equal(buf.len[l].cpu().numpy(), clip_lengths(ref["lengths"][l], CAPS[l]))
    rows = [max(x, 0) for x in c]
    for m in range(5):
        tails = [("neighbors", buf.nb[m], rows[m])]
        if m > 0:
            tails.append(("points", buf.pts[m], CAPS[l] if m == l else rows[m]))
        if m < 4:
            tails += [("pools", buf.pool[m], rows[m + 1]), ("upsamples", buf.up[m], rows[m])]
        for what, x, n in tails:
            tail = x[n:].contiguous().view(torch.int32).cpu().numpy()
            assert (tail == SENTINEL).all(), "%s level %d: %d rows past %d written" % (
                what, m, int((tail != SENTINEL).any(-1).sum()), n)
    _, F, _ = pipe.out[k]
    for m, x in enumerate(F):
        assert torch.isfinite(x[:rows[m]]).all(), m


@pytest.mark.gpu
@pytest.mark.parametrize("l", [1, 2, 3, 4])
def test_level_overflow(model, plain_pipe, plain_reference, l):
    """The overflowing batch twice (slots 0 and 1, slot 0 guarded), then the regular batches through every slot."""
    ref, _ = plain_reference
    bad = case_batch("level%d" % l)
    feed = [good()[g] for g in BEFORE] + [bad, bad] + [good()[g] for g in AFTER]
    slots = []

    def before(i, pipe):
        if i == len(BEFORE):
            guard(pipe, pipe.n_loaded % pipe.DEPTH)

    def after(i, k, res, counts):
        if i in (len(BEFORE), len(BEFORE) + 1):
            slots.append(k)
        if i == len(BEFORE):
            check_overflowed_slot(plain_pipe, k, *bad, l, counts[:5].cpu().tolist())

    snaps = run(plain_pipe, feed, before=before, after=after)
    st = statuses(plain_pipe)
    first, second = snaps[len(BEFORE)], snaps[len(BEFORE) + 1]
    print("level %d overflow: status %s, counts %s" % (l, st, first["counts"][:5].tolist()))
    assert st == [STATUS_CAPACITY if k in slots else 0 for k in range(len(st))] and len(set(slots)) == 2
    assert_same_steps(first, second, "level %d: two replays" % l)
    assert_finite(first, "level %d" % l)
    assert_later_steps(snaps, 2, ref, "level %d" % l)
    assert_sticky(plain_pipe)


# ---- scene bounds -----------------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("case", ["wide", "both"])
def test_cloud_wider_than_the_bbox(model, voxel_pipe, voxel_reference, case):
    """Bit 0 (and, with the voxel overflow, bit 1): the pyramid stops at level 1 (counts[1] = -1); the step stays
    finite and the next steps are exact."""
    ref, _ = voxel_reference
    feed = [good()[g] for g in BEFORE] + [case_batch(case)] + [good()[g] for g in AFTER]
    slot = []
    snaps = run(voxel_pipe, feed, after=lambda i, k, res, counts: slot.append(k) if i == len(BEFORE) else None)
    st = statuses(voxel_pipe)
    c = snaps[len(BEFORE)]["counts"][:5].tolist()
    print("%s: status %s, counts %s" % (case, st, c))
    want = STATUS_WIDE | (STATUS_CAPACITY if case == "both" else 0)
    assert st == [want if k == slot[0] else 0 for k in range(len(st))]
    assert c[1] == -1 and all(x <= 0 for x in c[2:]), c
    if case == "both":
        assert c[0] == CAPS[0]
    assert_finite(snaps[len(BEFORE)], case)
    assert_later_steps(snaps, 1, ref, case)
    assert_sticky(voxel_pipe)


@pytest.mark.gpu
def test_cloud_moved_outside_the_bbox_stays_exact(model, voxel_pipe, voxel_reference):
    """Cloud 13 moved 5 and then 50 box extents away: no status bit, and both steps, ICP over the moved cloud included,
    equal check_chain on the C port's voxelisation."""
    ref, _ = voxel_reference
    moved = [case_batch("moved5"), case_batch("moved50")]
    feed = [good()[g] for g in BEFORE] + moved + [good()[g] for g in AFTER]
    snaps = run(voxel_pipe, feed)
    print("moved: status %s, counts %s" % (statuses(voxel_pipe), [snaps[len(BEFORE) + j]["counts"][:5].tolist()
                                                                   for j in range(2)]))
    voxel_pipe.check()
    for j, batch in enumerate(moved):
        chain = eager_chain(model, voxel_pipe, *port_voxel_down_sample(*batch, V), "moved %d" % j, 20 + j)
        assert_step_equals_chain(snaps[len(BEFORE) + j], chain, "moved %d" % j)
    assert_later_steps(snaps, 2, ref, "moved")


# ---- a next batch refused on the host ---------------------------------------------------------------------------------

def rejected(cuda):
    """(points, lengths, truth) of next batches that step() refuses."""
    from d3feat_b200.evaluation import GroundTruth
    P, L = good()[1]
    T = truth()
    too_many = np.concatenate([P] * (RAW_CAP // len(P) + 1), 0)
    return [(t(too_many, cuda), t(L, cuda), T),
            (t(P, cuda), t(L[:-1], cuda), T),
            (t(P, cuda), t(L, cuda), GroundTruth(T.pose[:-1], None, T.flags[:-1])),
            (t(P, cuda), t(L, cuda), None)]


@pytest.mark.gpu
def test_rejected_next_batch_changes_nothing(cuda, voxel_pipe, voxel_reference):
    """Every refused next batch raises ValueError with the pending batch untouched: the next step returns it once, and
    the running totals equal the reference's, which never saw a refused batch."""
    ref, ref_totals = voxel_reference
    feed = good()
    pipe = voxel_pipe
    pipe.prime(t(feed[0][0], cuda), t(feed[0][1], cuda), truth=truth())
    snaps = []
    for i in range(len(feed)):
        if i == 1:
            for P, L, T in rejected(cuda):
                pending, loaded = pipe.pending, pipe.n_loaded
                with pytest.raises(ValueError, match="GraphPipeline"):
                    pipe.step(P, L, next_truth=T)
                assert (pipe.pending, pipe.n_loaded) == (pending, loaded)
        nxt = feed[i + 1] if i + 1 < len(feed) else None
        res, counts = pipe.step(t(nxt[0], cuda), t(nxt[1], cuda), next_truth=truth()) if nxt else pipe.step()
        torch.cuda.synchronize()
        snaps.append(snapshot(res, counts))
    pipe.check()
    for i, (got, want) in enumerate(zip(snaps, ref)):
        assert_same_steps(got, want, "step %d" % i)
    assert same_bits(pipe.evaluation_totals(), ref_totals)


# ---- CPU: every batch hits its condition and nothing else ------------------------------------------------------------

def level_sizes(P, L):
    return [p.shape[0] for p in oracle_pyramid(config(), P, L)["points"]]


def widest(P, L):
    return max((np.ptp(c, 0) for c in clouds_of(P, L) if len(c)), key=lambda e: e.max())


def test_regular_batches_fit_the_bucket():
    ext = bbox()[3:] - bbox()[:3]
    for P, L in good():
        assert len(P) <= RAW_CAP and (widest(P, L) <= ext).all()
        for voxel in (True, False):
            sizes = level_sizes(*level0(P, L, voxel))
            assert all(1.25 * n + 64 <= c for n, c in zip(sizes, CAPS)), (sizes, CAPS)
    assert all(CAPS[l] > CAPS[l + 1] for l in range(4))


def test_voxel_overflow_batch():
    P, L = case_batch("voxel")
    M = len(port_voxel_down_sample(P, L, V)[0])
    assert len(P) <= RAW_CAP and CAPS[0] < M and (widest(P, L) <= bbox()[3:] - bbox()[:3]).all()
    sizes = level_sizes(*truncated_voxels(P, L))
    assert sizes[0] == CAPS[0] and all(n <= c for n, c in zip(sizes, CAPS)), sizes


@pytest.mark.parametrize("l", [1, 2, 3, 4])
def test_level_overflow_batch(l):
    P, L = case_batch("level%d" % l)
    sizes = level_sizes(P, L)
    assert all(sizes[m] <= CAPS[m] for m in range(l)) and sizes[l] > CAPS[l], (l, sizes)
    assert (widest(P, L) <= bbox()[3:] - bbox()[:3]).all()


@pytest.mark.parametrize("case", ["wide", "both", "moved5", "moved50"])
def test_scene_bounds_batches(case):
    P, L = case_batch(case)
    ext = bbox()[3:] - bbox()[:3]
    vp, vl = port_voxel_down_sample(P, L, V)
    if case.startswith("moved"):
        assert (clouds_of(P, L)[BIG].min(0) > bbox()[3:]).all()           # wholly outside the box
        assert (widest(P, L) <= ext).all()
        assert all(n <= c for n, c in zip(level_sizes(vp, vl), CAPS))
    else:
        # every axis 3 times the box: more cells than the box's sort key holds, and past the voxel key on every axis
        assert (np.ptp(clouds_of(P, L)[WIDE], 0) > 3 * ext).all()
        assert L[WIDE] == 31
        assert (len(vp) > CAPS[0] + L[WIDE]) == (case == "both")
