"""The numpy statement of multi-view machine serving models (mvm_serving_model.py) checked on hand-built rows, against
the float64 definition, and against the canonical statement whose row it shares."""
import struct

import numpy as np
import pytest

import canonical_serving_model as CM
import compact_serving_model as CS
import delta_model as DM
import mvm_serving_model as MV
import serving_model as SM


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


@pytest.mark.parametrize("K,f32,f16", [(4, 32, 32), (8, 64, 32), (16, 96, 64), (32, 160, 96)])
def test_row_layout(K, f32, f16):
    for precision, want in ((MV.PRECISION_F32, f32), (MV.PRECISION_F16, f16)):
        dt = MV.row_dtype(K, precision)
        assert dt.itemsize == MV.row_bytes(K, precision) == want
        assert CS.row_bytes(CM.FM_CANONICAL, K, precision) == want  # the canonical row's bytes
        assert dt.fields["zero"][1] == 8 and dt.fields["v"][1] == 16
        # lane c's piece v[4c .. 4c+3] lies where it does in a canonical row
        vb = 2 if precision == MV.PRECISION_F16 else 4
        assert all(16 + 4 * c * vb == (16 + 16 * c if vb == 4 else 16 + 8 * c) for c in range(K // 4))


def test_rows_are_canonical_rows_with_w_zero():
    rng = np.random.default_rng(1)
    keys = rng.choice(1 << 40, 50, replace=False).astype(np.uint64)
    v = rng.normal(size=(50, 16)).astype(np.float32)
    mv, cm = MV.rows_array(keys, v), CM.rows_array(keys, np.zeros(50, np.float32), v)
    assert mv.tobytes() == cm.tobytes()
    assert MV.fingerprint(mv) == CM.fingerprint(cm) == DM.fingerprint(mv)
    assert np.all(mv["key"][1:] > mv["key"][:-1])


def test_padding_rule_includes_bytes_8_to_15():
    keys = np.arange(1, 5, dtype=np.uint64)
    for K, precision in ((4, MV.PRECISION_F16), (8, MV.PRECISION_F32), (16, MV.PRECISION_F16)):
        rows = MV.rows_array(keys, np.ones((4, K), np.float32), precision)
        assert MV.padding_zero(rows).all()
        for byte in (8, 11, 12, 15):
            raw = bytearray(rows.tobytes())
            raw[byte] = 1
            dirty = np.frombuffer(bytes(raw), rows.dtype)
            assert not MV.padding_zero(dirty)[0] and MV.padding_zero(dirty)[1:].all()
        if "pad" in rows.dtype.names:
            dirty = rows.copy()
            dirty["pad"][2, -1] = 1
            assert not MV.padding_zero(dirty)[2]
    # the tail of F32 K = 8 is 64 - 48 = 16 bytes, of F16 K = 16 64 - 48 = 16 bytes; K = 4 F32 has none
    assert "pad" not in MV.row_dtype(4).names and MV.row_dtype(8).fields["pad"][0].itemsize == 16


def test_prune_rules_ignore_w():
    v = np.array([[0, 0, 0, 0], [0, -0.0, 0, 0], [0, 0, 1e-30, 0], [1, 2, 3, 4]], np.float32)
    ready = np.array([False, True, True, False])
    assert MV.pruned(SM.ABSENT_DEFAULT, ready, v).tolist() == [True, False, False, True]
    assert MV.pruned(SM.ABSENT_ZERO, ready, v).tolist() == [True, True, False, False]


def test_file_bytes_with_fm_3(tmp_path):
    rng = np.random.default_rng(2)
    keys = rng.choice(1 << 50, 300, replace=False).astype(np.uint64)
    for K, precision in ((16, MV.PRECISION_F32), (32, MV.PRECISION_F16)):
        rows = MV.rows_array(keys, rng.normal(size=(300, K)).astype(np.float32), precision)
        data = MV.model_file(rows, K, precision, 0, SM.ABSENT_DEFAULT, 1, 0.0, 7, 320)
        assert struct.unpack_from("<i", data, 36)[0] == 3 and struct.unpack_from("<I", data, 60)[0] == precision
        assert struct.unpack_from("<I", data, 32)[0] == MV.row_bytes(K, precision)
        h, back = MV.parse_model_file(data)
        assert back.tobytes() == rows.tobytes() and h["keys"] == 300 and h["pruned_keys"] == 20
        # the canonical statement's file differs in fm only (and so in the header checksum)
        canon = CS.model_file(CS.convert(CM.rows_array(rows["key"], np.zeros(300, np.float32), rows["v"].astype(np.float32)),
                                         precision), CM.FM_CANONICAL, K, precision, 0, SM.ABSENT_DEFAULT, 1, 0.0, 7, 320)
        assert canon[:36] == data[:36] and canon[40:96] == data[40:96] and canon[104:] == data[104:]
        dirty = bytearray(data)
        dirty[104 + 32 + 9] = 1  # byte 9 of the first row, with its chunk's checksum now wrong
        with pytest.raises(ValueError):
            MV.parse_model_file(bytes(dirty))
        # deltas: fm = 3 at byte 16
        b = rows.copy()
        b["v"][::3] = b["v"][::3] * 2
        d = MV.delta_file(rows, b[5:], 300, K, precision, 0, SM.ABSENT_DEFAULT, 1, 0.0, 7)
        hd = dict(zip(DM.FIELDS, DM.HEADER.unpack(d[:DM.HEADER.size])))
        assert hd["fm"] == 3 and struct.unpack_from("<I", d, 52)[0] == precision
        assert hd["upserts"] == DM.diff(rows, b[5:])[0].size and hd["deletes"] == 5


def test_convert_rounds_v_and_copies_the_zero_word():
    keys = np.arange(1, 4, dtype=np.uint64)
    v = np.array([[1 / 3, 65519.0, -0.0, 1e-8], [np.nan, 2.0, 3.0, 4.0], [0.1, 0.2, 0.3, 0.4]], np.float32)
    rows = MV.rows_array(keys, v)
    h = MV.convert(rows, MV.PRECISION_F16)
    assert np.array_equal(h["v"].view(np.uint16), CS.to_half(v).view(np.uint16)) and not h["zero"].any()
    back = MV.convert(h, MV.PRECISION_F32)
    assert np.array_equal(_bits(back["v"]), _bits(CS.rounded(v)))
    big = rows.copy()
    big["v"][1, 2] = 65520.0
    with pytest.raises(CS.Overflow) as e:
        MV.convert(big, MV.PRECISION_F16)
    assert e.value.count == 1 and e.value.key == 2


def _hand(rows_fields):
    """CSR of rows given as lists of (field, x, v)"""
    rp = np.zeros(len(rows_fields) + 1, np.uint32)
    rp[1:] = np.cumsum([len(r) for r in rows_fields])
    toks = [t for r in rows_fields for t in r]
    f = np.array([t[0] for t in toks], np.uint8)
    x = np.array([t[1] for t in toks], np.float32)
    v = np.array([t[2] for t in toks], np.float32).reshape(len(toks), -1)
    return rp, f, x, v


def test_forward_on_hand_built_rows():
    rp, f, x, v = _hand([
        [(0, 1.0, [1, 2, 3, 4]), (1, 2.0, [1, 1, 1, 1])],            # P = (2, 4, 6, 8): y = 20
        [],                                                          # no tokens: y = 0
        [(5, 1.0, [1, 2, 3, 4]), (5, -1.0, [0.5, 0.5, 0.5, 0.5])],   # one field: y = sum of its sums = 8
        [(31, 0.5, [2, 2, 2, 2]), (3, 1.0, [1, -1, 1, -1]), (31, 1.0, [0, 0, 0, 1])],  # S3 = (1,-1,1,-1), S31 = (1,1,1,2): y = -1
        [(7, 1.0, [40, 0, 0, 0])],                                   # y = 40: pctr = 1
        [(7, 1.0, [-40, 0, 0, 0])],                                  # y = -40: pctr = 1e-6
    ])
    y, p = MV.forward(rp, f, x, v)
    assert y.tolist() == [20.0, 0.0, 8.0, -1.0, 40.0, -40.0]
    assert p[1] == np.float32(0.5) and p[4] == 1.0 and p[5] == np.float32(1e-6)
    assert p[0] == np.float32(np.exp(20.0 * 0.9999999998311266) / (1 + np.exp(20.0 * 0.9999999998311266)))
    # fields are read & 31, and no values is all ones
    y2, _ = MV.forward(rp, f.astype(np.int64) + 32, None, v * x[:, None])
    assert _bits(y2).tolist() == _bits(y).tolist()


def test_forward_adds_in_token_order_and_multiplies_fields_ascending():
    # three tokens of one field whose sum depends on the order: (1 + 1e8) - 1e8 = 0 in float32, 1 + (1e8 - 1e8) = 1
    K = 4
    rp = np.array([0, 3, 6], np.uint32)
    f = np.zeros(6, np.uint8)
    v = np.zeros((6, K), np.float32)
    v[:, 0] = [1.0, 1e8, -1e8, 1e8, -1e8, 1.0]
    y, _ = MV.forward(rp, f, None, v)
    assert y.tolist() == [0.0, 1.0]
    # the product runs over the present fields in ascending order: P = (((1 * S_a) * S_b) * S_c)
    v2 = np.zeros((3, K), np.float32)
    v2[:, 0] = [3e-30, 3e30, 1e-30]
    for perm in ([0, 1, 2], [2, 0, 1]):
        fp = np.array([2, 9, 20], np.uint8)[perm]
        yy, _ = MV.forward(np.array([0, 3], np.uint32), fp, None, v2[perm])
        want = np.float32(np.float32(np.float32(1) * np.float32(3e-30)) * np.float32(3e30)) * np.float32(1e-30)
        assert _bits(yy)[0] == _bits(np.float32(want))


def test_butterfly_is_the_32_lane_warp_sum():
    rng = np.random.default_rng(3)
    for K in MV.LATENT_DIMS:
        v = rng.normal(size=(1, K)).astype(np.float32) * np.float32(1e3)
        v[0, ::3] *= -1e-4
        y, _ = MV.forward(np.array([0, 1], np.uint32), np.zeros(1, np.uint8), None, v)
        lanes = np.zeros(32, np.float32)
        lanes[:K] = v[0]
        for o in (16, 8, 4, 2, 1):
            lanes = np.array([lanes[i] + lanes[i ^ o] for i in range(32)], np.float32)
        assert _bits(y)[0] == _bits(lanes)[0]


def _random_rows(rng, lens, fields_of, K):
    rp = np.zeros(len(lens) + 1, np.uint32)
    rp[1:] = np.cumsum(lens)
    nnz = int(rp[-1])
    f = fields_of(rp)
    x = rng.uniform(0.25, 1.5, nnz).astype(np.float32) * rng.choice([-1, 1], nnz).astype(np.float32)
    v = rng.normal(0, 0.6, (nnz, K)).astype(np.float32)
    return rp, f, x, v


@pytest.mark.parametrize("K", MV.LATENT_DIMS)
def test_forward_within_tolerance_of_float64(K):
    rng = np.random.default_rng(K)
    lens = [0, 1, 3, 31, 32, 33, 65, 129, 300] + [9] * 40
    rp, f, x, v = _random_rows(rng, lens, lambda rp: rng.integers(0, 6, int(rp[-1])).astype(np.uint8), K)
    f[rp[5]:rp[6]] = 31
    y, p = MV.forward(rp, f, x, v)
    y64 = MV.forward64(rp, f, x, v)
    scale = np.maximum(1.0, np.abs(y64))
    assert np.all(np.abs(y.astype(np.float64) - y64) <= 1e-4 * scale)
    import fm_model as FMM
    assert np.all(np.abs(p.astype(np.float64) - FMM.sigmoid(y64)) <= 1e-5)


@pytest.mark.parametrize("K", [4, 32])
def test_permuting_tokens_without_repeated_fields_keeps_every_bit(K):
    rng = np.random.default_rng(10 + K)
    lens = [1, 2, 5, 17, 32] * 4
    rp, f, x, v = _random_rows(rng, lens, lambda rp: np.concatenate(
        [rng.permutation(32)[:n] for n in np.diff(rp)]).astype(np.uint8), K)
    y, p = MV.forward(rp, f, x, v)
    perm = np.concatenate([rp[r] + rng.permutation(rp[r + 1] - rp[r]) for r in range(rp.size - 1)]).astype(np.int64)
    y2, p2 = MV.forward(rp, f[perm], x[perm], v[perm])
    assert np.array_equal(_bits(y), _bits(y2)) and np.array_equal(_bits(p), _bits(p2))


def test_zero_rows_of_either_sign_read_alike_nan_and_inf_included():
    """A pruned ZERO row (v = -0 allowed) and an absent key (v = +0) give the same bits: the sums start at +0 and never
    become -0, and 0 x is the same NaN for either sign when x is NaN or Inf."""
    rng = np.random.default_rng(4)
    K = 8
    rp, f, x, v = _random_rows(rng, [4, 7, 3, 12], lambda rp: rng.integers(0, 3, int(rp[-1])).astype(np.uint8), K)
    zero = np.array([1, 5, 6, 13, 20])
    x[5], x[13] = np.nan, np.inf
    vp, vn = v.copy(), v.copy()
    vp[zero] = 0.0
    vn[zero] = -0.0
    vn[zero[0], ::2] = 0.0
    yp, pp = MV.forward(rp, f, x, vp)
    yn, pn = MV.forward(rp, f, x, vn)
    assert np.array_equal(_bits(yp), _bits(yn)) and np.array_equal(_bits(pp), _bits(pn))
    assert np.isnan(yp[1]) and np.isnan(yp[2])  # 0 x NaN, 0 x Inf


def test_collision_free_rows():
    K = 16  # T = 8 tokens per pass
    rp = np.array([0, 3, 6, 22, 25], np.uint32)
    f = np.array([1, 1, 2,   4, 4, 4,   *range(8), *range(8),   0, 1, 2], np.uint8)
    assert MV.collision_free(rp, f, K).tolist() == [True, False, True, True]
