"""The numpy ranking model (tests/rank_model.py) against a brute-force sort with a comparator written from the order's
plain words: a higher pctr first, equal pctr bits by smaller index, +0 before -0, NaN of either sign after every
number."""
import functools
import math
import struct

import numpy as np
import pytest

from rank_model import PAD_INDEX, PAD_PCTR_BITS, rank_keys, rank_model


def _f(bits):
    return struct.unpack("<f", struct.pack("<I", bits))[0]


def _bits(x):
    return struct.unpack("<I", struct.pack("<f", x))[0]


def _cmp(a, b):
    """a, b = (index, float32 value as a Python float); negative when a ranks first."""
    (ia, pa), (ib, pb) = a, b
    na, nb = math.isnan(pa), math.isnan(pb)
    if na or nb:
        if na and nb:
            return ia - ib
        return 1 if na else -1
    if _bits(pa) == _bits(pb):
        return ia - ib
    if pa == pb:  # +0 and -0
        return -1 if _bits(pa) == 0 else 1
    return -1 if pa > pb else 1


def _brute(pctr, cand_ptr, k):
    R = len(cand_ptr) - 1
    index = np.full((R, k), 0xFFFFFFFF, np.uint32)
    bits = np.full((R, k), 0x7FC00000, np.uint32)
    for q in range(R):
        p = pctr[cand_ptr[q]:cand_ptr[q + 1]]
        order = sorted(((i, float(p[i])) for i in range(p.size)), key=functools.cmp_to_key(_cmp))[:k]
        for j, (i, _) in enumerate(order):
            index[q, j] = i
            bits[q, j] = p.view(np.uint32)[i]
    return index, bits


def _same(pctr, cand_ptr, k):
    pctr = np.asarray(pctr, np.float32)
    idx, top = rank_model(pctr, cand_ptr, k)
    want_idx, want_bits = _brute(pctr, cand_ptr, k)
    assert idx.shape == top.shape == (len(cand_ptr) - 1, k)
    assert np.array_equal(idx, want_idx)
    assert np.array_equal(top.view(np.uint32), want_bits)
    return idx, top


SPECIAL = [_f(0x7FC00000), _f(0xFFC00000), _f(0x7F800001), _f(0xFFFFFFFF), 0.0, -0.0, math.inf, -math.inf, 1.0, 1e-6,
           0.5, -1.0, _f(0x00000001), _f(0x80000001)]


def test_keys_order_specials():
    p = np.array(SPECIAL, np.float32)
    keys = rank_keys(p)
    assert len(set(keys.tolist())) == p.size
    assert all(keys[i] >> np.uint64(32) == 0 for i in range(4))  # NaN of either sign and any payload
    assert keys[6] > keys[8] > keys[10] > keys[9] > keys[12] > keys[4] > keys[5] > keys[13] > keys[11] > keys[7] > 0


@pytest.mark.parametrize("k", [1, 2, 5, 14, 20])
def test_specials_every_k(k):
    rng = np.random.default_rng(k)
    p = np.array(SPECIAL * 3, np.float32)[rng.permutation(3 * len(SPECIAL))]
    idx, top = _same(p, [0, p.size], k)
    m = min(k, p.size)
    # NaN last, in index order
    nan = np.isnan(top[0, :m])
    if nan.any():
        first = int(np.argmax(nan))
        assert nan[first:].all() and np.all(np.diff(idx[0, first:m].astype(np.int64)) > 0)


def test_ties_across_k():
    # a tie group of 7 equal scores that straddles position k = 5: two above it, three of the group taken by index
    p = np.array([0.3, 0.9, 0.3, 0.3, 0.95, 0.3, 0.1, 0.3, 0.3, 0.3], np.float32)
    idx, _ = _same(p, [0, p.size], 5)
    assert idx[0].tolist() == [4, 1, 0, 2, 3]
    # the clamped ends of the sigmoid
    p = np.array([1.0, 1e-6, 1.0, 1e-6, 1.0, 0.5, 1.0], np.float32)
    idx, _ = _same(p, [0, p.size], 6)
    assert idx[0].tolist() == [0, 2, 4, 6, 5, 1]


def test_padding_and_empty():
    p = np.array([0.2, _f(0x7FC00000), 0.7], np.float32)
    cand_ptr = [0, 0, 2, 2, 3]  # requests of 0, 2, 0 and 1 candidates
    idx, top = _same(p, cand_ptr, 4)
    assert idx.tolist() == [[PAD_INDEX] * 4, [0, 1] + [PAD_INDEX] * 2, [PAD_INDEX] * 4, [0] + [PAD_INDEX] * 3]
    assert (top.view(np.uint32)[0] == PAD_PCTR_BITS).all()
    assert top.view(np.uint32)[1].tolist() == [_bits(np.float32(0.2)), 0x7FC00000, 0x7FC00000, 0x7FC00000]
    # R > 0 without candidates, and R = 0
    idx, top = _same(np.zeros(0, np.float32), [0, 0, 0], 3)
    assert (idx == PAD_INDEX).all() and (top.view(np.uint32) == PAD_PCTR_BITS).all()
    idx, top = _same(np.zeros(0, np.float32), [0], 7)
    assert idx.shape == (0, 7)


@pytest.mark.parametrize("seed", range(6))
def test_random_batches(seed):
    rng = np.random.default_rng(seed)
    counts = rng.integers(0, 40, 12)
    cand_ptr = np.concatenate([[0], np.cumsum(counts)])
    # few distinct values, so that ties are frequent, with specials sprinkled in
    p = rng.choice(np.array([0.1, 0.2, 0.2, 0.5, 1.0, 1e-6] + SPECIAL, np.float32), int(cand_ptr[-1]))
    for k in (1, 3, 16, 50):
        _same(p, cand_ptr, k)
