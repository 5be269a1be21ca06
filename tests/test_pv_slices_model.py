"""CPU checks of the sliced progressive validation model (tests/pv_slices_model.py): a row counts once per slice its
keys name, in every slice they name, in none when they name none, and a partition of the rows sums to the whole."""
import numpy as np
import pytest

import pv_slices_model as S
import validation_model as V

INTS = ("rows", "positives", "negatives", "nan_rows", "overflow_rows")


def _stream(seed, rows):
    rng = np.random.default_rng(seed)
    p = rng.random(rows).astype(np.float32)
    p[rng.random(rows) < 0.05] = np.nan
    y = (rng.random(rows) < 0.3).astype(np.uint8)
    w = rng.choice(np.array([0.0, 0.5, 1.0, 3.0, -1.0], np.float32), rows, p=[0.1, 0.2, 0.5, 0.15, 0.05])
    return p, y, w


def test_repeated_keys_count_once():
    # row 0 names slice 0 by three tokens (two keys), row 1 by one
    rp = np.array([0, 4, 6], np.uint32)
    keys = np.array([10, 11, 10, 99, 98, 10], np.uint64)
    smap = {10: 0, 11: 0}
    assert [m.tolist() for m in S.slice_rows(rp, keys, smap, 1)] == [[0, 1]]
    p = np.array([0.25, 0.75], np.float32)
    y = np.array([0, 1], np.uint8)
    got = S.slice_reports(p, y, None, rp, keys, smap, 1, 8)[0]
    assert got == V.Pv(8).add(p, y).report()
    assert got["rows"] == 2 and got["auc"] == 1.0


def test_a_row_counts_in_two_slices_and_rows_without_slice_keys_in_none():
    rp = np.array([0, 2, 3, 5, 6], np.uint32)
    keys = np.array([1, 2, 1, 7, 8, 9], np.uint64)
    smap = {1: 0, 2: 1, 7: 1}
    rows = S.slice_rows(rp, keys, smap, 3)
    assert [m.tolist() for m in rows] == [[0, 1], [0, 2], []]  # row 3 (key 9) is in no slice, slice 2 is empty
    p, y, w = np.array([0.1, 0.2, 0.3, 0.4], np.float32), np.array([1, 0, 1, 0], np.uint8), None
    reps = S.slice_reports(p, y, w, rp, keys, smap, 3, 4)
    assert [r["rows"] for r in reps] == [2, 2, 0]
    assert np.isnan(reps[2]["logloss"]) and np.isnan(reps[2]["auc"])


@pytest.mark.parametrize("ms", [4, 8, 16])
def test_a_partition_sums_to_the_global_counts(ms):
    rng = np.random.default_rng(ms)
    rows, k = 800, 5
    p, y, w = _stream(ms, rows)
    lens = rng.integers(1, 70, rows)  # rows across several 32-token chunks
    rp = np.concatenate([[0], np.cumsum(lens)]).astype(np.uint32)
    keys = rng.integers(1000, 5000, int(rp[-1])).astype(np.uint64)
    # every row gets exactly one of the slice keys 0 .. 2k-1 (two keys per slice), at a random position
    skeys = rng.integers(0, 2 * k, rows).astype(np.uint64)
    keys[rp[:-1] + rng.integers(0, lens)] = skeys
    smap = {j: j // 2 for j in range(2 * k)}
    members = S.slice_rows(rp, keys, smap, k)
    assert sorted(np.concatenate(members).tolist()) == list(range(rows))
    reps = S.slice_reports(p, y, w, rp, keys, smap, k, ms)
    whole = V.Pv(ms).add(p, y, w).report()
    for f in INTS:
        assert sum(r[f] for r in reps) == whole[f], f
    assert whole["nan_rows"] > 0 and whole["overflow_rows"] > 0
