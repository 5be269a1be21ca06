"""Hand cases for the numpy statement of the serving model (serving_model.py)."""
import struct

import numpy as np
import pytest

import serving_model as M


def test_fm_sums_follow_the_kernels_association():
    # 1 + 2^-24 rounds back to 1 in float32: summed in k order the small terms vanish one by one; pairwise they would not
    v = np.array([1.0, 2.0 ** -24, 2.0 ** -24, 2.0 ** -24], np.float32)
    st, qt = M.fm_sums(v)
    assert st[0] == np.float32(1.0) and float(np.sum(v.astype(np.float64))) > 1.0
    assert qt[0] == np.float32(1.0)
    # v^2 is rounded to float32 before it is added: 3 * fl(0.1f^2), not fl(3 * 0.1^2)
    v = np.full(3, 0.1, np.float32)
    sq = np.float32(v[0] * v[0])
    _, qt = M.fm_sums(v)
    assert qt[0] == np.float32(np.float32(sq + sq) + sq)


@pytest.mark.parametrize("K", [8, 10, 16])
def test_fm_sums_against_a_scalar_loop(K):
    rng = np.random.default_rng(K)
    v = (rng.standard_normal((50, K)) * 1e-2).astype(np.float32)
    st, qt = M.fm_sums(v)
    for i in range(v.shape[0]):
        s, q = np.float32(0), np.float32(0)
        for k in range(K):
            s = np.float32(s + v[i, k])
            q = np.float32(q + np.float32(v[i, k] * v[i, k]))
        assert st[i] == s and qt[i] == q
    assert st.dtype == np.float32 and qt.dtype == np.float32


def test_prune_rule():
    w = np.array([0.0, -0.0, 1e-30, -2.0], np.float32)
    assert M.pruned(w, False, M.ABSENT_DEFAULT).tolist() == [True, True, False, False]
    assert M.pruned(w, False, M.ABSENT_ZERO).tolist() == [True, True, False, False]
    # FM, absent keys read as default rows: only rows whose latent block was never materialised can go
    ready = np.array([False, True, False, False])
    assert M.pruned(w, True, M.ABSENT_DEFAULT, v_ready=ready).tolist() == [True, False, False, False]
    # FM, absent keys read as nothing: w, st and qt must all be zero, whatever the latent block's state
    st = np.array([0.0, 0.0, 0.0, 0.0], np.float32)
    qt = np.array([0.0, 1e-8, 0.0, 0.0], np.float32)
    assert M.pruned(w, True, M.ABSENT_ZERO, st=st, qt=qt).tolist() == [True, False, False, False]
    st[0] = -0.0
    assert M.pruned(w, True, M.ABSENT_ZERO, st=st, qt=qt)[0]


def test_capacity_keeps_the_load_at_half():
    assert [M.capacity_for(n) for n in (0, 1, 512, 513, 1024, 1025)] == [1024, 1024, 1024, 2048, 2048, 4096]


def test_checksum_is_the_splitmix_sum():
    assert int(M.splitmix64(0)) == 0xE220A8397B1DCDAF  # the published first output of splitmix64 seeded with 0
    a = struct.pack("<QQ", 5, 7)
    assert M.section_sum(a) == (int(M.splitmix64(5 ^ 0)) + int(M.splitmix64(7 ^ 8))) % (1 << 64)
    assert M.section_sum(a, 1 << 40) != M.section_sum(a)


@pytest.mark.parametrize("fm", [False, True])
def test_file_round_trip_and_layout(fm):
    keys = np.array([9, 3, 2 ** 63 + 1, 4], np.uint64)
    w = np.array([0.5, -1.0, 0.25, 2.0], np.float32)
    st = np.array([1, 2, 3, 4], np.float32) if fm else None
    qt = np.array([5, 6, 7, 8], np.float32) if fm else None
    rows = M.rows_array(keys, w, st, qt)
    assert rows["key"].tolist() == sorted(keys.tolist())
    data = M.build_file(rows, 8 if fm else 0, 0, M.ABSENT_ZERO, 1, 0.0, 11, 10)
    assert len(data) == 104 + 32 + 4 * (32 if fm else 16)
    assert struct.unpack_from("<Q", data, M.OFFSETS["keys"])[0] == 4
    assert struct.unpack_from("<Q", data, M.OFFSETS["capacity"])[0] == 1024
    assert struct.unpack_from("<I", data, M.OFFSETS["row_bytes"])[0] == (32 if fm else 16)
    assert struct.unpack_from("<i", data, M.OFFSETS["absent"])[0] == M.ABSENT_ZERO
    assert struct.unpack_from("<Q", data, M.OFFSETS["pruned_keys"])[0] == 6
    # the first row follows the header and the chunk head: key 3, w -1
    assert struct.unpack_from("<Qf", data, 104 + 32) == (3, -1.0)
    if fm:
        assert struct.unpack_from("<ff", data, 104 + 32 + 12) == (2.0, 6.0)
    h, back = M.parse_file(data)
    assert h["source_keys"] == 10 and h["seed"] == 11 and back.tobytes() == rows.tobytes()
    # any flipped byte and any truncation is noticed
    for pos in (5, 20, 100, 104 + 8, 104 + 40, len(data) - 1):
        bad = bytearray(data)
        bad[pos] ^= 0x10
        with pytest.raises(ValueError):
            M.parse_file(bytes(bad))
    for cut in (0, 50, 104, 120, len(data) - 1):
        with pytest.raises(ValueError):
            M.parse_file(data[:cut])
    # a dirty padding byte is refused even when the checksums are right
    dirty = rows.copy()
    dirty["pad"][2] = 1 if dirty["pad"].ndim == 1 else [0, 1, 0]
    with pytest.raises(ValueError, match="padding"):
        M.parse_file(M.build_file(dirty, 8 if fm else 0, 0, M.ABSENT_ZERO, 1, 0.0, 11, 10))


def test_empty_model_file():
    data = M.build_file(M.rows_array([], []), 0, 1, M.ABSENT_DEFAULT, 0, 0.001, 0, 3)
    assert len(data) == 104
    h, rows = M.parse_file(data)
    assert h["keys"] == 0 and h["pruned_keys"] == 3 and rows.size == 0
