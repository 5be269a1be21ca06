"""Hand cases for the numpy statement of canonical serving models (canonical_serving_model.py)."""
import struct

import numpy as np
import pytest

import canonical_serving_model as CM
import delta_model as DM
import serving_model as SM


def test_row_bytes_round_16_plus_4k_up_to_a_sector():
    assert [CM.row_bytes(K) for K in CM.LATENT_DIMS] == [32, 64, 96, 160, 288, 544]
    for K in CM.LATENT_DIMS:
        assert CM.row_bytes(K) % 32 == 0 and CM.row_dtype(K).fields["v"][1] == 16


def test_row_packing_by_hand():
    rows = CM.rows_array([7, 3], [0.5, -2.0], [[1, 2, 3, 4, 5, 6, 7, 8], [9, 10, 11, 12, 13, 14, 15, 16]])
    raw = rows.tobytes()
    assert len(raw) == 2 * 64
    # sorted by key: key 3 first, then w, a zero word, v, and 16 bytes of zero padding
    assert struct.unpack_from("<QfI8f", raw, 0) == (3, -2.0, 0, 9, 10, 11, 12, 13, 14, 15, 16)
    assert raw[48:64] == bytes(16)
    assert struct.unpack_from("<Qf", raw, 64) == (7, 0.5)
    # piece c of v (coordinates 4c .. 4c+3) is the 16 bytes at 16 + 16c
    assert struct.unpack_from("<4f", raw, 64 + 16 + 16) == (5, 6, 7, 8)
    assert CM.padding_zero(rows).all()
    dirty = rows.copy()
    dirty["zero"][1] = 1
    assert CM.padding_zero(dirty).tolist() == [True, False]
    dirty = rows.copy()
    dirty["pad"][0, 15] = 1
    assert CM.padding_zero(dirty).tolist() == [False, True]
    # K = 4: no padding after v
    assert CM.row_dtype(4).names == ("key", "w", "zero", "v")


def test_prune_rules():
    w = np.array([0.0, -0.0, 0.0, 1e-30], np.float32)
    ready = np.array([False, True, True, False])
    v = np.array([[0.1, 0, 0, 0], [0, -0.0, 0, 0], [0, 0, 0, 1e-40], [0, 0, 0, 0]], np.float32)
    # DEFAULT: an absent key reads as its initial latent values, so only a block never materialised can go
    assert CM.pruned(w, SM.ABSENT_DEFAULT, ready, v).tolist() == [True, False, False, False]
    # ZERO: an absent key reads as nothing, so w and every v_k must be zero (either sign), whatever the block's state
    assert CM.pruned(w, SM.ABSENT_ZERO, ready, v).tolist() == [False, True, False, False]


def test_fingerprint_chains_every_word_of_a_row():
    rows = CM.rows_array([5], [1.0], [[2.0, 3.0, 4.0, 5.0]])
    words = np.frombuffer(rows.tobytes(), "<u8")
    assert words.size == 4
    h = np.uint64(0)
    for x in words:
        h = SM.splitmix64(h ^ x)
    assert CM.fingerprint(rows) == int(h)
    # K = 16: 12 words, and a change in the last coordinate changes it
    rows = CM.rows_array([1, 2], [0.0, 1.0], np.arange(32, dtype=np.float32).reshape(2, 16))
    other = rows.copy()
    other["v"][1, 15] = 0.0
    assert CM.fingerprint(rows) != CM.fingerprint(other) and CM.fingerprint(rows[:0]) == 0
    # order-free
    assert CM.fingerprint(rows) == CM.fingerprint(rows[::-1].copy())


@pytest.mark.parametrize("K", [4, 16, 128])
def test_model_file_layout_and_round_trip(K):
    rng = np.random.default_rng(K)
    keys = rng.choice(1 << 40, 5, replace=False).astype(np.uint64)
    rows = CM.rows_array(keys, rng.standard_normal(5), rng.standard_normal((5, K)))
    data = CM.model_file(rows, K, 0, SM.ABSENT_DEFAULT, 1, 0.0, 3, 9)
    assert len(data) == 104 + 32 + 5 * CM.row_bytes(K)
    assert struct.unpack_from("<i", data, SM.OFFSETS["fm"])[0] == 2
    assert struct.unpack_from("<i", data, SM.OFFSETS["latent_dim"])[0] == K
    assert struct.unpack_from("<I", data, SM.OFFSETS["row_bytes"])[0] == CM.row_bytes(K)
    assert struct.unpack_from("<Q", data, SM.OFFSETS["chunk_rows"])[0] == (64 << 20) // CM.row_bytes(K)
    assert struct.unpack_from("<Q", data, SM.OFFSETS["pruned_keys"])[0] == 4
    h, back = CM.parse_model_file(data)
    assert back.tobytes() == rows.tobytes() and h["keys"] == 5
    for pos in (36, 40, 104 + 8, len(data) - 1):
        bad = bytearray(data)
        bad[pos] ^= 0x10
        with pytest.raises(ValueError):
            CM.parse_model_file(bytes(bad))
    # dirty padding with checksums that pass is refused too
    dirty = rows.copy()
    dirty["zero"][2] = 7
    with pytest.raises(ValueError):
        CM.parse_model_file(CM.model_file(dirty, K, 0, SM.ABSENT_DEFAULT, 1, 0.0, 3, 9))


def test_delta_file_header_and_apply():
    K = 8
    a = CM.rows_array([1, 2, 3], [0.0, 1.0, 2.0], np.ones((3, K)))
    b = CM.rows_array([2, 3, 4], [1.0, 2.5, 3.0], np.ones((3, K)))
    up, de = DM.diff(a, b)
    assert up["key"].tolist() == [3, 4] and de.tolist() == [1]
    assert DM.apply(a, up, de).tobytes() == b.tobytes()
    data = CM.delta_file(a, b, 5, K, 0, SM.ABSENT_ZERO, 1, 0.0, 3)
    h = dict(zip(DM.FIELDS, DM.HEADER.unpack(data[:DM.HEADER.size])))
    assert h["fm"] == 2 and h["latent_dim"] == K and h["row_bytes"] == 64
    assert h["chunk_rows"] == (64 << 20) // 64 and h["upserts"] == 2 and h["deletes"] == 1
    assert h["base_fingerprint"] == CM.fingerprint(a) and h["result_fingerprint"] == CM.fingerprint(b)
    assert h["pruned_keys"] == 2 and h["header_checksum"] == SM.section_sum(data[:136])
    assert len(data) == 144 + 32 + 2 * 64 + 32 + 8
