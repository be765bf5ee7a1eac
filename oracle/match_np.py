"""numpy restatement of descriptor matching between keypoint sets (d3f_match_descriptors).

similarity() is the contract's sequential-channel fp32 sum: every product and every sum rounded to float32 on its own,
channels in ascending order, so it reproduces the kernel bit for bit. The nearest neighbours are np.argmax (NaN above
everything, -0.0 equal to +0.0, ties to the smallest index); the mutual rule is the 3DMatch evaluation's
build_correspondence (geometric_registration/evaluate.py:11-27): keep (i, nn_st[i]) when nn_ts[nn_st[i]] == i, in
ascending i. reference_correspondence() restates that function's own formulation, argmin of sqrt(2 - 2 a.b)."""
import numpy as np

CANONICAL_NAN = np.array([0x7fc00000], np.uint32).view(np.float32)[0]


def similarity(a, b):
    """s[i, j] = sum_c a[i, c] * b[j, c] in float32, c ascending, no fused multiply-add."""
    a = np.asarray(a, np.float32)
    b = np.asarray(b, np.float32)
    s = np.zeros((a.shape[0], b.shape[0]), np.float32)
    with np.errstate(invalid="ignore", over="ignore"):
        for c in range(a.shape[1]):
            s = s + np.multiply.outer(a[:, c], b[:, c])
    return s


def nearest(s):
    """(nn_st, sim_st, nn_ts, sim_ts) of a non-empty similarity matrix: np.argmax along each axis and the value there."""
    n, m = s.shape
    nn_st = np.argmax(s, axis=1).astype(np.int32)
    nn_ts = np.argmax(s, axis=0).astype(np.int32)
    return nn_st, s[np.arange(n), nn_st], nn_ts, s[nn_ts, np.arange(m)]


def mutual(nn_st, nn_ts):
    """[(i, nn_st[i])] for every i with nn_ts[nn_st[i]] == i, ascending i, as int32 [m, 2]."""
    i = np.arange(len(nn_st))
    keep = nn_ts[nn_st] == i
    return np.stack([i[keep], nn_st[keep]], 1).astype(np.int32).reshape(-1, 2)


def match(desc, count, pairs):
    """Matches of every pair as numpy arrays: dict(nn_st, sim_st, nn_ts, sim_ts [P,k], matches [P,k,2], n_matches [P]).
    Slots past the count get -1 / 0; a pair naming a cloud outside [0, B), or an empty cloud, matches nothing. NaN
    similarities are the canonical quiet NaN, as the kernel reports them."""
    desc = np.asarray(desc, np.float32)
    B, k, _ = desc.shape
    n = np.clip(np.asarray(count, np.int64), 0, k)
    pairs = np.asarray(pairs, np.int64).reshape(-1, 2)
    P = pairs.shape[0]
    out = dict(nn_st=np.full((P, k), -1, np.int32), sim_st=np.zeros((P, k), np.float32),
               nn_ts=np.full((P, k), -1, np.int32), sim_ts=np.zeros((P, k), np.float32),
               matches=np.full((P, k, 2), -1, np.int32), n_matches=np.zeros(P, np.int32))
    for p, (src, tgt) in enumerate(pairs):
        if not (0 <= src < B and 0 <= tgt < B):
            continue
        ns, nt = int(n[src]), int(n[tgt])
        if ns == 0 or nt == 0:
            continue
        s = similarity(desc[src, :ns], desc[tgt, :nt])
        nn_st, sim_st, nn_ts, sim_ts = nearest(s)
        m = mutual(nn_st, nn_ts)
        out["nn_st"][p, :ns], out["sim_st"][p, :ns] = nn_st, sim_st
        out["nn_ts"][p, :nt], out["sim_ts"][p, :nt] = nn_ts, sim_ts
        out["matches"][p, :len(m)] = m
        out["n_matches"][p] = len(m)
    for key in ("sim_st", "sim_ts"):
        out[key][np.isnan(out[key])] = CANONICAL_NAN
    return out


def reference_correspondence(a, b):
    """build_correspondence's own formulation: distances sqrt(2 - 2 a.b), argmin both ways, mutual pairs in ascending
    source order. Returns (nn_st, nn_ts, matches [m, 2])."""
    with np.errstate(invalid="ignore"):
        dist = np.sqrt(2 - 2 * (np.asarray(a, np.float32) @ np.asarray(b, np.float32).T))
    nn_st = np.argmin(dist, axis=1).astype(np.int32)
    nn_ts = np.argmin(dist, axis=0).astype(np.int32)
    return nn_st, nn_ts, mutual(nn_st, nn_ts)
