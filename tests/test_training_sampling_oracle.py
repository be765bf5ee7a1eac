"""CPU: the cases of tests/test_gpu_training_sampling.py tell a right sampler from a wrong one.

emulate() restates what the GPU does, not what the oracle does: sample_keys_kernel's key per row, a stable sort of the
keys over sort_bits(P) bits, and sample_pick_kernel's reads of the sorted candidates. It equals oracle/pairs_np.sample
on every case, and each emulated bug changes the oracle's answer on a named case:
  * keys truncated to sort_bits(P) - 1 bits: the three sort-width cases;
  * tied draws in reverse candidate order (an unstable sort): the tie case;
  * positions read at offset[p] + m instead of (offset[p] - offset[0]) + m: the slice case, and no other, since every
    other table starts at 0;
  * rows of no pair sorted first instead of last: every case that has such rows.
"""
import functools

import numpy as np
import pytest

from oracle import pairs_np as op
from test_gpu_training_sampling import CASES, TIES_N, TIES_SEED, case, sort_bits, sort_passes, tied_draws

BUGS = ("truncated_key", "unstable_ties", "absolute_position", "no_pair_first")


def emulate(offset, rows, anchor, k, replace, min_count, seed, bug=None):
    """(anc, pos, valid) as csrc/correspond.cu computes them, with one of BUGS if asked."""
    assert bug is None or bug in BUGS
    offset = np.asarray(offset, np.int64)
    rows = np.asarray(rows, np.int64).reshape(-1, 2)
    M, P = len(rows), len(offset) - 1
    lo = np.clip(offset[:P], 0, M)                              # candidates(): [lo, hi) clamped into [0, M)
    hi = np.minimum(np.maximum(offset[1:], lo), M)
    n = hi - lo
    valid = (n >= max(min_count, 1)) & (replace or (n >= k))
    m = np.arange(k)
    if replace:
        c = op.draw_index(op.draw(seed, np.arange(P)[:, None], m[None, :], op.SLOT_DRAW), n[:, None]).astype(np.int64)
    else:
        i = np.arange(M)
        p = np.maximum(np.searchsorted(lo, i, side="right") - 1, 0)   # the last pair starting at or before row i
        ours = (i >= lo[p]) & (i < hi[p])
        cand = np.where(ours, i - lo[p], 0)
        key = np.full(M, (P << 32) | 0xFFFFFFFF, np.uint64)
        key[ours] = (p[ours].astype(np.uint64) << np.uint64(32)) | (
            op.draw(seed, p[ours], cand[ours], op.SLOT_KEY) >> np.uint64(32))
        bits = sort_bits(P) - (bug == "truncated_key")
        key &= np.uint64((1 << bits) - 1)
        if bug == "unstable_ties":
            order = np.lexsort((-i, key))
        else:
            order = np.argsort(key, kind="stable")
        if bug == "no_pair_first":
            order = np.concatenate([order[~ours[order]], order[ours[order]]])
        base = lo if bug == "absolute_position" else lo - lo[0]
        at = np.where(valid[:, None], base[:, None] + m[None, :], 0)
        c = cand[order][at] if M else np.zeros((P, k), np.int64)
    ok = valid[:, None] & (c < n[:, None])
    r = np.where(ok, lo[:, None] + c, 0)
    anc = np.where(ok, rows[r, 0] if M else 0, -1).astype(np.int32)
    pos = np.where(ok, (rows[r, 1] if M else 0) + np.asarray(anchor, np.int64)[:, None], -1).astype(np.int32)
    return anc, pos, valid


@functools.lru_cache(maxsize=None)
def _oracle(name, j):
    c = case(name)
    return op.sample(c.offset, c.rows, c.anchor, *c.calls[j])


def _same(got, want):
    return all(np.array_equal(g, w) for g, w in zip(got, want))


def _caught(name, bug):
    """Whether the bug changes the result of any call of the case."""
    c = case(name)
    return any(not _same(emulate(c.offset, c.rows, c.anchor, *call, bug=bug), _oracle(name, j))
               for j, call in enumerate(c.calls))


@pytest.mark.parametrize("name", CASES)
def test_emulation_equals_the_oracle(name):
    c = case(name)
    for j, call in enumerate(c.calls):
        got = emulate(c.offset, c.rows, c.anchor, *call)
        for what, g, w in zip(("anc", "pos", "valid"), got, _oracle(name, j)):
            np.testing.assert_array_equal(g, w, err_msg="%s %s %s" % (name, call, what))


def test_sort_bits_and_passes():
    assert [sort_bits(P) for P in (1, 2, 120, 255, 256, 65535, 65536, 1 << 24)] == [33, 34, 39, 40, 41, 48, 49, 57]
    assert [sort_passes(P) for P in (255, 256, 65535, 65536, 1 << 24)] == [5, 6, 6, 7, 8]


@pytest.mark.parametrize("name", ["P255", "P256", "P65536"])
def test_a_key_one_bit_short_is_caught(name):
    """At P = 255 pairs 128 .. 254 sort among pairs 0 .. 126; at 256 and 65536 the rows of no pair (pair P) sort among
    pair 0's candidates and push every later pair's run back."""
    assert _caught(name, "truncated_key")


def test_an_unstable_order_of_tied_draws_is_caught():
    assert tied_draws(TIES_SEED, 0, TIES_N) > 0
    assert _caught("ties", "unstable_ties")


def test_positions_from_offset_not_offset0_are_caught_only_by_the_slice():
    assert _caught("slice", "absolute_position")
    for name in CASES:
        if name != "slice":
            assert int(case(name).offset[0]) == 0 and not _caught(name, "absolute_position"), name


@pytest.mark.parametrize("name", ["P255", "P256", "P65536", "slice", "tail"])
def test_rows_of_no_pair_sorted_first_are_caught(name):
    c = case(name)
    assert int(c.offset[0]) > 0 or int(c.offset[-1]) < len(c.rows)
    assert _caught(name, "no_pair_first")


def test_the_slice_samples_each_pair_from_its_own_rows():
    """rows[:, 0] is the row's own index, so every anchor the oracle samples for pair q of the slice lies in
    [offset[q], offset[q+1]) of the full rows."""
    c = case("slice")
    for j in range(len(c.calls)):
        anc, _, valid = _oracle("slice", j)
        assert valid.any()
        assert ((anc >= c.offset[:-1, None]) & (anc < c.offset[1:, None]))[valid].all()
