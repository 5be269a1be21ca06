"""The numpy statement of serving model deltas (tests/delta_model.py) on random row sets: apply(A, diff(A, B)) == B, the
fingerprint is order-free, and the XFSD builder and parser agree."""
import struct

import numpy as np
import pytest

import delta_model as D
import serving_model as SM


def _rows(rng, n, fm, key_space=5000):
    keys = rng.choice(np.arange(1, key_space, dtype=np.uint64), n, replace=False)
    w = rng.standard_normal(n).astype(np.float32)
    if fm:
        return SM.rows_array(keys, w, rng.standard_normal(n).astype(np.float32), rng.random(n).astype(np.float32))
    return SM.rows_array(keys, w)


def _pair(rng, na, nb, fm):
    """B made from A: some rows kept, some changed by one bit, some dropped, some new"""
    a = _rows(rng, na, fm)
    b = a[rng.random(a.size) < 0.7].copy()
    flip = rng.random(b.size) < 0.3
    b["w"][flip] = (b["w"][flip].view(np.uint32) ^ np.uint32(1)).view(np.float32)
    extra = _rows(rng, nb, fm, key_space=20000)
    extra = extra[~np.isin(extra["key"], a["key"])]
    out = np.concatenate([b, extra])
    return a, out[np.argsort(out["key"])]


@pytest.mark.parametrize("fm", [0, 1])
@pytest.mark.parametrize("sizes", [(0, 0), (0, 300), (300, 0), (300, 300), (1000, 50)])
def test_apply_of_diff_is_the_next_model(fm, sizes):
    rng = np.random.default_rng(sizes[0] * 7 + sizes[1] + fm)
    a, b = _pair(rng, sizes[0], sizes[1], fm)
    if sizes[1] == 0:
        b = b[:0]
    up, de = D.diff(a, b)
    got = D.apply(a, up, de)
    assert got.tobytes() == b.tobytes()
    assert D.fingerprint(got) == D.fingerprint(b)
    assert np.all(np.diff(up["key"].astype(object)) > 0) and np.all(np.diff(de.astype(object)) > 0)
    assert not np.isin(de, b["key"]).any() and np.isin(de, a["key"]).all()
    if sizes == (0, 0):
        assert D.fingerprint(a) == 0 and up.size == 0 and de.size == 0
    if sizes[0] == 0:
        assert up.tobytes() == b.tobytes()
    if sizes[1] == 0:
        assert np.array_equal(de, a["key"])


@pytest.mark.parametrize("fm", [0, 1])
def test_diff_of_a_model_with_itself_is_empty(fm):
    a = _rows(np.random.default_rng(3), 500, fm)
    up, de = D.diff(a, a)
    assert up.size == 0 and de.size == 0


@pytest.mark.parametrize("fm", [0, 1])
def test_a_one_bit_change_is_an_upsert(fm):
    a = _rows(np.random.default_rng(4), 100, fm)
    b = a.copy()
    field = "qt" if fm else "w"
    b[field][17] = (b[field][17].view(np.uint32) ^ np.uint32(1 << 31)).view(np.float32)  # -0 against +0 included
    up, de = D.diff(a, b)
    assert up["key"].tolist() == [a["key"][17]] and de.size == 0
    assert D.fingerprint(a) != D.fingerprint(b)


@pytest.mark.parametrize("fm", [0, 1])
def test_fingerprint_is_order_free(fm):
    rng = np.random.default_rng(5)
    a = _rows(rng, 777, fm)
    assert D.fingerprint(a) == D.fingerprint(a[rng.permutation(a.size)])
    # the chain over a row's words is order-dependent: swapping two words of a row changes it
    words = a.view("<u8").reshape(a.size, -1).copy()
    words[0, [0, 1]] = words[0, [1, 0]]
    assert D.fingerprint(words.view(a.dtype).ravel()) != D.fingerprint(a)


def test_fingerprint_of_a_hand_row():
    row = SM.rows_array(np.array([5], np.uint64), np.array([1.5], np.float32))
    w0, w1 = 5, int(np.float32(1.5).view(np.uint32))
    h = SM.splitmix64(np.uint64(w1) ^ SM.splitmix64(np.uint64(w0)))
    assert D.fingerprint(row) == int(h)


@pytest.mark.parametrize("fm", [0, 1])
def test_builder_and_parser_round_trip(fm):
    a, b = _pair(np.random.default_rng(6), 400, 200, fm)
    K = 8 if fm else 0
    data = D.delta_file(a, b, b.size + 9, K, 0, 1, 1, 0.0, 11)
    h, up, de = D.parse_file(data)
    want_up, want_de = D.diff(a, b)
    assert up.tobytes() == want_up.tobytes() and np.array_equal(de, want_de)
    assert (h["magic"], h["version"], h["header_bytes"], h["row_bytes"]) == (b"XFSD", 1, 144, 32 if fm else 16)
    assert (h["fm"], h["latent_dim"], h["absent"], h["seed"]) == (fm, K, 1, 11)
    assert (h["base_keys"], h["result_keys"], h["source_keys"], h["pruned_keys"]) == (a.size, b.size, b.size + 9, 9)
    assert h["base_fingerprint"] == D.fingerprint(a) and h["result_fingerprint"] == D.fingerprint(b)
    assert (h["upserts"], h["deletes"]) == (up.size, de.size)
    assert len(data) == 144 + 2 * 32 + up.nbytes + de.nbytes
    codes = ["4s"] + list(D.HEADER.format[3:])  # one struct code per field
    for i, name in enumerate(D.FIELDS):
        assert struct.calcsize("<" + "".join(codes[:i])) == D.OFFSETS[name]
    assert D.apply(a, up, de).tobytes() == b.tobytes()


def test_parser_refuses_damage_and_malformed_contents():
    a, b = _pair(np.random.default_rng(7), 300, 100, 0)
    data = D.delta_file(a, b, b.size, 0, 0, 0, 0, 0.0, 1)
    for cut in (0, 100, 144 + 10, len(data) - 1):
        with pytest.raises(ValueError):
            D.parse_file(data[:cut])
    with pytest.raises(ValueError):
        D.parse_file(data + b"\0" * 8)
    for pos in (5, 60, 150, len(data) - 3):
        x = bytearray(data)
        x[pos] ^= 1
        with pytest.raises(ValueError):
            D.parse_file(bytes(x))
    up, de = D.diff(a, b)
    assert up.size > 3 and de.size > 3
    bad_pad = up.copy()
    bad_pad["pad"][1] = 1
    dup = up.copy()
    dup["key"][2] = dup["key"][1]
    reserved = up.copy()
    reserved["key"][-1] = D.EMPTY
    for u, d in ((up[::-1], de), (up, de[::-1]), (dup, de), (reserved, de), (bad_pad, de),
                 (up, np.sort(np.append(de[1:], up["key"][0])))):
        bad = D.build_file(u, d, 0, 0, 0, 0, 0.0, 1, a.size, D.fingerprint(a), b.size, b.size, D.fingerprint(b))
        with pytest.raises(ValueError):
            D.parse_file(bad)
