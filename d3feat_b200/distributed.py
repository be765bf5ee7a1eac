"""Multi-GPU: whole point-cloud fragments shard across ranks (one process per GPU); the only exchange step is
ONE all-gather of the per-fragment descriptors at the end (NCCL over NVLink/NVSwitch between H100s, gloo in
the CPU tests). The reference is single-process (SURVEY.md 8e): fragments are independent units, so there is no
data-path collective inside the pyramid or the encoder.
"""
import torch
import torch.distributed as dist


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
