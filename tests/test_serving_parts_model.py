"""Hand cases for the numpy statement of model parts and their merge (serving_parts_model.py)."""
import struct

import numpy as np
import pytest

import serving_model as M
import serving_parts_model as P

ARGS = dict(optimizer=0, absent=M.ABSENT_DEFAULT, v_init=1, v_const=0.0, seed=11)


def _split(keys, w, S, st=None, qt=None, extra_source=0):
    """part files of the rows (keys, w[, st, qt]) split S ways, each shard's source keys = its rows + extra_source"""
    s = P.shard_of(keys, S)
    files = []
    for i in range(S):
        sel = s == i
        rows = M.rows_array(keys[sel], w[sel], None if st is None else st[sel], None if qt is None else qt[sel])
        files.append(P.build_part(rows, 0 if st is None else 8, source_keys=int(sel.sum()) + extra_source,
                                  shard_index=i, num_shards=S, **ARGS))
    return files


def _keys(n, seed):
    rng = np.random.default_rng(seed)
    ks = rng.integers(0, 2 ** 63, n, dtype=np.uint64) * np.uint64(2) + rng.integers(0, 2, n, dtype=np.uint64)
    edges = []
    for S in (2, 3, 8):
        for s in range(S):
            lo, hi = P.shard_range(s, S)
            edges += [lo, hi]
    ks = np.unique(np.concatenate([ks, np.array(edges, np.uint64)]))
    return ks[ks != np.uint64(P.M64)]


def test_shard_ranges_tile_the_key_space_as_shard_of_does():
    for S in (1, 2, 3, 7, 8):
        width = P.M64 // S
        prev_hi = -1
        for s in range(S):
            lo, hi = P.shard_range(s, S)
            assert lo == prev_hi + 1 and lo == s * width
            assert P.shard_of([lo], S)[0] == s and P.shard_of([hi], S)[0] == s
            prev_hi = hi
        assert prev_hi == P.M64 - 1  # the last shard takes the tail [S width, 2^64 - 2]; 2^64 - 1 is the empty marker
    assert P.shard_of([P.M64 - 1], 3)[0] == 2 and P.shard_of([P.M64 // 3 * 3], 3)[0] == 2


def test_part_file_layout_and_round_trip():
    keys = np.array([9, 3, 2 ** 63 + 1, 4], np.uint64)
    w = np.array([0.5, -1.0, 0.25, 2.0], np.float32)
    rows = M.rows_array(keys, w)
    whole = M.build_file(rows, 0, source_keys=6, **ARGS)
    part = P.build_part(rows, 0, source_keys=6, shard_index=0, num_shards=1, **ARGS)
    assert part[:4] == b"XFSP" and len(part) == len(whole) + 8
    assert struct.unpack_from("<Q", part, 8)[0] == 112
    assert part[16:96] == whole[16:96]  # XFSM's fields
    assert struct.unpack_from("<iiQ", part, 96) == (0, 1, M.section_sum(part[:104]))
    assert part[112:] == whole[104:]  # the same chunks
    h, back = P.parse_part(part)
    assert back.tobytes() == rows.tobytes() and h["keys"] == 4 and h["pruned_keys"] == 2
    for pos in (5, 20, 97, 101, 106, 112 + 8, len(part) - 1):
        bad = bytearray(part)
        bad[pos] ^= 0x10
        with pytest.raises(ValueError):
            P.parse_part(bytes(bad))
    for cut in (0, 50, 104, 112, len(part) - 1):
        with pytest.raises(ValueError):
            P.parse_part(part[:cut])
    with pytest.raises(ValueError):
        P.parse_part(whole)


def _resum(data):
    """data with its header and chunk checksums recomputed: damage the checksums do not see"""
    data = bytearray(data)
    data[104:112] = struct.pack("<Q", M.section_sum(bytes(data[:104])))
    pos, chunk = 112, 0
    while pos < len(data):
        first, n, _, _ = struct.unpack_from("<QQQQ", data, pos)
        body = bytes(data[pos + 32:pos + 32 + n * 16])
        struct.pack_into("<Q", data, pos + 16, M.section_sum(body, chunk << 40))
        pos += 32 + len(body)
        chunk += 1
    return bytes(data)


def test_a_part_file_whose_checksums_pass_can_still_be_refused():
    keys = _keys(200, 1)
    files = _split(keys, np.ones(keys.size, np.float32), 3)
    P.parse_part(_resum(files[1]))  # the re-summing itself changes nothing
    # a key of shard 2 in shard 1's file, placed last so that the keys still ascend
    bad = bytearray(files[1])
    lo2, _ = P.shard_range(2, 3)
    struct.pack_into("<Q", bad, len(bad) - 16, lo2)
    with pytest.raises(ValueError, match="outside"):
        P.parse_part(_resum(bad))
    # keys out of order
    bad = bytearray(files[1])
    a, b = bytes(bad[112 + 32:112 + 48]), bytes(bad[112 + 48:112 + 64])
    bad[112 + 32:112 + 48], bad[112 + 48:112 + 64] = b, a
    with pytest.raises(ValueError, match="ascending"):
        P.parse_part(_resum(bad))
    # a shard that does not exist
    bad = bytearray(files[1])
    struct.pack_into("<i", bad, 96, 3)
    with pytest.raises(ValueError, match="shard"):
        P.parse_part(_resum(bad))


@pytest.mark.parametrize("S", [1, 2, 3, 8])
@pytest.mark.parametrize("fm", [False, True])
def test_merge_is_the_whole_models_file(S, fm):
    keys = _keys(3000, S)
    rng = np.random.default_rng(S)
    w = rng.standard_normal(keys.size).astype(np.float32)
    st = rng.standard_normal(keys.size).astype(np.float32) if fm else None
    qt = rng.random(keys.size).astype(np.float32) if fm else None
    files = _split(keys, w, S, st, qt, extra_source=5)
    want = M.build_file(M.rows_array(keys, w, st, qt), 8 if fm else 0, source_keys=keys.size + 5 * S, **ARGS)
    assert P.merge(files) == want
    assert P.merge(files[::-1]) == want  # the order the parts come in does not matter
    h, rows = M.parse_file(want)
    assert h["pruned_keys"] == 5 * S
    # the rows are the parts' rows one after another, in shard order
    assert rows.tobytes() == b"".join(P.parse_part(f)[1].tobytes() for f in files)
    # the fingerprint of the model is the sum of the parts': a sum over rows
    assert sum(P.parse_part(f)[0]["keys"] for f in files) == keys.size


def test_merge_refusals():
    keys = _keys(500, 7)
    w = np.ones(keys.size, np.float32)
    files = _split(keys, w, 3)
    P.merge(files)
    with pytest.raises(ValueError, match="every part"):
        P.merge(files[:2])
    with pytest.raises(ValueError, match="repeated"):
        P.merge([files[0], files[1], files[1]])
    with pytest.raises(ValueError, match="every part"):
        P.merge(files + _split(keys, w, 2)[:1])
    with pytest.raises(ValueError):
        P.merge([M.build_file(M.rows_array(keys, w), 0, source_keys=keys.size, **ARGS)])  # a whole model
    s = P.shard_of(keys, 3)
    other = P.build_part(M.rows_array(keys[s == 2], w[s == 2]), 0, optimizer=1, absent=M.ABSENT_DEFAULT, v_init=1,
                         v_const=0.0, seed=11, source_keys=int((s == 2).sum()), shard_index=2, num_shards=3)
    with pytest.raises(ValueError, match="optimizer"):
        P.merge(files[:2] + [other])
