"""Multi-GPU: whole point-cloud fragments shard across ranks (one process per GPU); the only exchange step is
ONE all-gather of the per-fragment descriptors at the end (NCCL over NVLink/NVSwitch between H100s, gloo in
the CPU tests). The reference is single-process (SURVEY.md 8e): fragments are independent units, so there is no
data-path collective inside the pyramid or the encoder.

Data-parallel training: each rank runs training.forward / d3feat_loss / backward on its own pair, then
reduce_gradients, the update (training.MomentumClip) and reduce_moving_statistics. Both reductions all-gather the
ranks' values and take their mean in rank order in fp64 (d3f_rank_mean): an all-gather only copies, so, unlike
all_reduce, whose summation order depends on NCCL's algorithm and the topology, the result is the same bits on every
rank, run to run and for any topology.
"""
import torch
import torch.distributed as dist

from . import _lib


def shard_fragments(n_fragments, rank, world_size):
    """Fragment f -> rank f mod world_size (round robin keeps per-rank point counts balanced for
    similarly sized fragments). Returns the list of fragment ids owned by `rank`."""
    return [f for f in range(n_fragments) if f % world_size == rank]


def _world(group):
    if not dist.is_available() or not dist.is_initialized():
        return 1
    return dist.get_world_size(group)


def all_gather_descriptors_padded(local_desc, rows_per_fragment, capacity, group=None, max_fragments=None,
                                  rows_dev=None):
    """Sync-free gather used on the hot path.

    local_desc: float32[R, D] stacked descriptors of this rank's fragments (R is the tensor's shape, host-known);
    rows_per_fragment: int tensor [F] ON THE DEVICE (the last pyramid level's stack lengths) -- it is never read
    on the host here; capacity: rows reserved per rank (>= R on every rank); max_fragments: fragments reserved per
    rank (>= F on every rank; default F, which then must be the same on all ranks -- with round-robin sharding that
    only holds when n_fragments % world == 0).
    rows_dev (optional): int device scalar with the ACTUAL number of valid rows when local_desc is a capacity-sized
    buffer whose row count only the device knows (the graph-replayed pipeline); it replaces R in the meta row.
    Returns (gathered [world, capacity, D], meta [world, 2 + max_fragments] int64 = [R, F, rows per fragment...,
    zero padding]), both on the device; no host synchronisation, two collectives (one of them a few bytes).
    """
    R, D = local_desc.shape
    if R > capacity:
        raise ValueError("all_gather_descriptors_padded: %d rows exceed the per-rank capacity %d" % (R, capacity))
    F = int(rows_per_fragment.shape[0])
    Fmax = F if max_fragments is None else int(max_fragments)
    if F > Fmax:
        raise ValueError("all_gather_descriptors_padded: %d fragments exceed max_fragments %d" % (F, Fmax))
    dev = local_desc.device
    world = _world(group)
    # R and F enter the device as fill-kernel arguments: torch.tensor([R], device=...) would be a pageable host->device
    # copy, which synchronises the stream first (the host would wait for the whole encoder queued before this call
    # and the pyramid(i+1) || encoder(i) overlap would be lost on every rank)
    meta = torch.zeros((2 + Fmax,), dtype=torch.int64, device=dev)
    if rows_dev is not None:
        meta[0:1] = rows_dev.reshape(1).to(torch.int64)
    else:
        meta[0:1].fill_(R)
    meta[1:2].fill_(F)
    meta[2:2 + F] = rows_per_fragment.to(torch.int64)
    if R == capacity and local_desc.is_contiguous():
        padded = local_desc                     # already a capacity-sized buffer: no staging copy
    else:
        padded = torch.zeros((capacity, D), dtype=local_desc.dtype, device=dev)
        padded[:R] = local_desc
    if world == 1:
        return padded.unsqueeze(0), meta.unsqueeze(0)
    metas = torch.empty((world, meta.numel()), dtype=torch.int64, device=dev)
    gathered = torch.empty((world, capacity, D), dtype=local_desc.dtype, device=dev)
    if dev.type == "cuda":
        dist.all_gather_into_tensor(metas.view(-1), meta, group=group)
        dist.all_gather_into_tensor(gathered.view(-1, D), padded, group=group)
    else:
        dist.all_gather(list(metas.unbind(0)), meta, group=group)
        dist.all_gather(list(gathered.unbind(0)), padded, group=group)
    return gathered, metas


def unpack_gathered(gathered, metas):
    """Host-side compaction of the padded gather: (desc_all [sum R, D], rows_all list[int], owner list[int]);
    rank 0's fragments first, then rank 1's, ... (each rank's own order preserved; fragments with zero rows keep
    their slot). Synchronises."""
    m = metas.cpu()
    world = m.shape[0]
    rows = [int(m[r, 0]) for r in range(world)]
    desc_all = torch.cat([gathered[r, :rows[r]] for r in range(world)], 0)
    rows_all, owner = [], []
    for r in range(world):
        nf = int(m[r, 1])                                 # explicit fragment count: zero-row fragments are not padding
        rows_all += [int(x) for x in m[r, 2:2 + nf]]
        owner += [r] * nf
    return desc_all, rows_all, owner


def all_gather_descriptors(local_desc, local_rows_per_fragment, group=None):
    """Convenience form with exact shapes (reads sizes on the host): returns
    (desc_all [R_total, D], rows_all list[int], owner list[int]). Ranks may own different numbers of fragments."""
    if _world(group) == 1:
        return local_desc, list(local_rows_per_fragment), [0] * len(local_rows_per_fragment)
    dev = local_desc.device
    world = _world(group)
    n_local = len(local_rows_per_fragment)
    sizes = torch.tensor([local_desc.shape[0], n_local], dtype=torch.int64, device=dev)
    all_sizes = [torch.zeros_like(sizes) for _ in range(world)]
    dist.all_gather(all_sizes, sizes, group=group)
    cap = max(int(s[0]) for s in all_sizes)
    fmax = max(int(s[1]) for s in all_sizes)
    rows_t = torch.tensor(list(local_rows_per_fragment), dtype=torch.int64, device=dev).reshape(-1)
    gathered, metas = all_gather_descriptors_padded(local_desc, rows_t, max(cap, 1), group, max_fragments=max(fmax, 1))
    return unpack_gathered(gathered, metas)


# ----------------------------------------------------------------------------------------------------
#  data-parallel training
# ----------------------------------------------------------------------------------------------------

def rank_mean(x, out=None):
    """x float32 [R, P] (CUDA) -> out [P] = fl32((x[0] + ... + x[R-1]) / R), summed in fp64 in rank order
    (d3f_rank_mean; oracle/optim_np.rank_mean). R = 1 returns x[0]'s bits. out may be x[0]."""
    op = "rank_mean"
    x = _lib.tensor_arg(x, op + ": x", torch.float32, (None, None))
    R, P = x.shape
    if R < 1:
        raise ValueError("%s: x has no ranks" % op)
    if out is None:
        out = torch.empty((P,), dtype=torch.float32, device=x.device)
    elif not (torch.is_tensor(out) and out.is_contiguous()):
        raise ValueError("%s: out must be a contiguous tensor (it is written in place)" % op)
    out = _lib.tensor_arg(out, op + ": out", torch.float32, (P,), x.device)
    _lib.check(_lib.lib().d3f_rank_mean(_lib.ptr(x), R, P, _lib.ptr(out), _lib.stream()), "d3f_rank_mean")
    return out


def _gather_rows(flat, group):
    """[R, P]: every rank's flat float32 buffer, in rank order. Without a process group: flat as [1, P]."""
    if not dist.is_available() or not dist.is_initialized():
        return flat.view(1, -1)
    out = torch.empty((dist.get_world_size(group), flat.numel()), dtype=flat.dtype, device=flat.device)
    if dist.get_backend(group) == "nccl":
        dist.all_gather_into_tensor(out.view(-1), flat, group=group)
    else:
        dist.all_gather(list(out.unbind(0)), flat, group=group)
    return out


def _mean_over_ranks(tensors, group):
    """Replace every tensor's values by their mean over the ranks (rank order, fp64), in place."""
    if not tensors:
        return
    flat = torch.cat([t.detach().reshape(-1) for t in tensors])
    mean = rank_mean(_gather_rows(flat, group), out=flat)
    views = [m.view(t.shape) for m, t in zip(mean.split([t.numel() for t in tensors]), tensors)]
    with torch.no_grad():
        torch._foreach_copy_(tensors, views)        # one launch for all tensors, not one per tensor


def reduce_gradients(params, group=None):
    """Data-parallel gradient: every parameter's .grad becomes the mean of the ranks' gradients, taken in rank order
    in fp64 (rank_mean) over one all-gather of all gradients, so every rank holds the same bits. With one pair per
    rank this is the gradient of the mean of the ranks' losses. A parameter without a gradient counts as zero (its
    .grad is created), so a rank whose pair was skipped still takes part. Every rank must pass the same parameters in
    the same order. No host synchronisation (the collective is enqueued on the current stream)."""
    params = list(params)
    for i, p in enumerate(params):
        _lib.tensor_arg(p, "reduce_gradients: params[%d]" % i, torch.float32)
        if p.grad is None:
            p.grad = torch.zeros_like(p, memory_format=torch.contiguous_format)
        else:
            _lib.tensor_arg(p.grad, "reduce_gradients: params[%d].grad" % i, torch.float32, tuple(p.shape), p.device)
    _mean_over_ranks([p.grad for p in params], group)


def reduce_moving_statistics(store, group=None):
    """Replace every moving_mean / moving_variance of the ParamStore by its mean over the ranks (rank_mean, in
    place), so that every replica holds the same store and writes the same snapshot. Call it after each step: each
    rank's batch norm updated its own statistics from its own pair."""
    names = [n for n in sorted(store.t) if n.rsplit("/", 1)[-1] in ("moving_mean", "moving_variance")]
    for n in names:
        _lib.tensor_arg(store.t[n], "reduce_moving_statistics: " + n, torch.float32)
    _mean_over_ranks([store.t[n] for n in names], group)


STEP_STATS = ("loss", "desc_loss", "det_loss", "accuracy", "d_pos", "d_neg")


def gather_step_stats(stats, group=None):
    """[R, 6] float32 on the device: every rank's (loss, desc_loss, det_loss, accuracy, d_pos, d_neg), the values
    training.d3feat_loss returns, in rank order (for logging; no host synchronisation)."""
    stats = list(stats)
    if len(stats) != len(STEP_STATS):
        raise ValueError("gather_step_stats: %d values, expected the %d of d3feat_loss %s" % (
            len(stats), len(STEP_STATS), STEP_STATS))
    flat = torch.stack([v.detach().reshape(()).to(torch.float32) for v in stats])
    return _gather_rows(flat, group).clone()
