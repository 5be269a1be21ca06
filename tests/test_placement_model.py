"""The key builders of placement_model.py against its restatement of the device's probe sequence and bucket rule
(CPU only; the GPU suite's probe-overflow tests check the restatement itself against the device)."""
import numpy as np
import pytest

import placement_model as P

CAPS = [10, 12, 16, 20, 31]
STRIDES = [(0, True, False), (4, False, False), (8, True, False), (16, True, False), (8, False, True)]


def test_multiplier_inverse():
    assert (P.A * P.A_INV) & P.M64 == 1
    rng = np.random.default_rng(0)
    for k in [0, 1, P.M64, *(int(x) for x in rng.integers(0, 2 ** 63, 50, dtype=np.uint64))]:
        assert P.key_of(P.m_of(k)) == k and P.m_of(P.key_of(k)) == k


def test_row_stride_and_bucket_rule():
    assert P.row_stride(0, True) == 32
    assert P.row_stride(4, False) == 64       # acc 48, + 16
    assert P.row_stride(16, True) == 256      # acc 96, + 16 + 128
    assert P.row_stride(8, False, canon=True) == 128   # acc 64, + 16 + 32 = 112
    assert P.bucket_log2(32, 20) == 2         # LR: 4 rows per 128-byte line
    assert P.bucket_log2(64, 20) == 1
    assert P.bucket_log2(256, 20) == 0
    assert P.bucket_log2(32, 5) == 0          # fewer than 16 buckets: linear probing
    assert P.bucket_log2(32, 20, "0") == 0 and P.bucket_log2(32, 20, "4") == 4 and P.bucket_log2(32, 20, "9") == 4
    assert P.bucket_log2(256, 20, "3") == 3 and P.bucket_log2(32, 20, "-2") == 0 and P.bucket_log2(32, 20, "") == 2
    assert P.bucket_log2(32, 7, "4") == 0


def _bshifts(log2cap):
    out = set()
    for K, ftrl, canon in STRIDES:
        stride = P.row_stride(K, ftrl, canon)
        for env in (None, "0", "3", "4"):
            out.add(P.bucket_log2(stride, log2cap, env))
    return sorted(out)


@pytest.mark.parametrize("log2cap", [6, 10, 12])
def test_probe_sequence_is_a_permutation(log2cap):
    """The first 2^log2cap probes of any key visit every slot once (so a chain of n keys fills n distinct slots)."""
    for bs in _bshifts(log2cap):
        for key in (P.tail(1, (3,))[0], P.head(1)[0], np.uint64(12345)):
            seq = [P.probe_slot(key, i, log2cap, bs) for i in range(1 << log2cap)]
            assert sorted(seq) == list(range(1 << log2cap))


@pytest.mark.parametrize("log2cap", CAPS)
def test_tail_keys_home_in_last_bucket_and_wrap(log2cap):
    keys = P.tail(64, j0s=(0, 1, 2, 3, 15))
    for bs in _bshifts(log2cap):
        nb = 1 << (log2cap - bs)
        for key in keys:
            j0 = (P.m_of(key) >> 9) & ((1 << bs) - 1)
            home = P.home_slot(key, log2cap, bs)
            assert home >> bs == nb - 1 and home & ((1 << bs) - 1) == j0
            # the walk leaves the last bucket for slot 0, then goes on slot by slot
            wrap = 1 << bs
            assert [P.probe_slot(key, wrap + i, log2cap, bs) for i in range(3)] == [0, 1, 2]
            assert {P.probe_slot(key, i, log2cap, bs) for i in range(wrap)} == set(range((nb - 1) << bs, nb << bs))


@pytest.mark.parametrize("log2cap", CAPS)
def test_head_keys_home_in_bucket_zero(log2cap):
    for bs in _bshifts(log2cap):
        for key in P.head(32):
            assert P.home_slot(key, log2cap, bs) >> bs == 0
            assert P.probe_slot(key, 1 << bs, log2cap, bs) == 1 << bs


@pytest.mark.parametrize("log2cap", CAPS)
def test_one_chain_shares_its_probe_sequence(log2cap):
    keys = P.one_chain(200)
    for bs in _bshifts(log2cap):
        ref = [P.probe_slot(keys[0], i, log2cap, bs) for i in range(40)]
        for key in keys[1:]:
            assert [P.probe_slot(key, i, log2cap, bs) for i in range(40)] == ref


@pytest.mark.parametrize("log2cap", CAPS)
def test_twin_of_empty_shares_the_reserved_keys_sequence(log2cap):
    twin = P.twin_of_empty()
    assert int(twin) != P.EMPTY_KEY
    for bs in _bshifts(log2cap):
        assert [P.probe_slot(twin, i, log2cap, bs) for i in range(40)] == \
               [P.probe_slot(P.EMPTY_KEY, i, log2cap, bs) for i in range(40)]


def test_builders_give_distinct_keys_never_the_reserved_one():
    parts = [P.tail(3000), P.tail(500, (1,), start=3000), P.head(2000), P.one_chain(8193, start=4000),
             P.tail(100, start=(1 << P.FREE_BITS) - 100)]
    allk = np.concatenate(parts)
    assert np.unique(allk).size == allk.size
    assert not (allk == np.uint64(P.EMPTY_KEY)).any()
    with pytest.raises(AssertionError):
        P.tail(2, start=(1 << P.FREE_BITS) - 1)
