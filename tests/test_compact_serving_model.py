"""compact_serving_model.py against hand cases: binary16 rounding (ties to even, the overflow edge, signed zero,
subnormals, NaN), the F16 row layouts, conversion, and the precision word of the XFSM, XFSP and XFSD files, whose F32
bytes are those of the existing builders."""
import struct

import numpy as np
import pytest

import canonical_serving_model as CM
import compact_serving_model as H
import delta_model as DM
import serving_model as SM
import serving_parts_model as P


def _bits16(x):
    return int(H.to_half(np.float32(x)).view(np.uint16))


# ---- rounding ------------------------------------------------------------------------------------------------------
def test_ties_round_to_even():
    assert H.rounded(np.float32(1 + 2.0 ** -11)) == np.float32(1.0)
    assert H.rounded(np.float32(1 + 3 * 2.0 ** -11)) == np.float32(1 + 2.0 ** -9)
    assert H.rounded(np.float32(-(1 + 2.0 ** -11))) == np.float32(-1.0)


def test_the_overflow_edge():
    below = np.nextafter(np.float32(65520.0), np.float32(0))  # 65519.996
    assert float(below) == pytest.approx(65519.996, abs=1e-3)
    assert H.rounded(below) == np.float32(65504.0) and not H.overflows(below)
    for x in (65520.0, -65520.0, 1e6, 3.4e38):
        assert H.overflows(np.float32(x)), x
    for x in (np.inf, -np.inf, np.nan, 65504.0, -65504.0):
        assert not H.overflows(np.float32(x)), x


def test_signed_zero_subnormals_and_nan():
    assert _bits16(-0.0) == 0x8000 and _bits16(0.0) == 0x0000
    assert H.rounded(np.float32(2.0 ** -25)) == np.float32(0.0)  # a tie between 0 and 2^-24: even is 0
    assert H.rounded(np.float32(3 * 2.0 ** -26)) == np.float32(2.0 ** -24)
    assert H.rounded(np.float32(5 * 2.0 ** -25)) == np.float32(2 * 2.0 ** -24)  # tie, to even
    assert H.rounded(np.float32(2.0 ** -20 + 2.0 ** -30)) == np.float32(2.0 ** -20)
    assert np.isnan(H.rounded(np.float32(np.nan)))
    assert H.rounded(np.float32(np.inf)) == np.inf


# ---- rows ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("K,want", [(4, 32), (8, 32), (16, 64), (32, 96), (64, 160), (128, 288)])
def test_canonical_f16_row_bytes(K, want):
    assert H.row_bytes(CM.FM_CANONICAL, K, H.PRECISION_F16) == want == H.canonical_dtype(K, H.PRECISION_F16).itemsize
    assert H.row_bytes(CM.FM_CANONICAL, K, H.PRECISION_F32) == CM.row_bytes(K)
    dt = H.canonical_dtype(K, H.PRECISION_F16)
    assert dt.fields["v"][1] == 16 and dt.fields["zero"][1] == 12  # piece c of v at 16 + 8c


def test_fm_f16_row_is_16_bytes_without_padding():
    assert H.FM_ROW16.itemsize == 16 == H.row_bytes(1, 16, H.PRECISION_F16)
    assert [H.FM_ROW16.fields[f][1] for f in ("key", "w", "st", "qt")] == [0, 8, 12, 14]
    assert H.row_bytes(1, 16, H.PRECISION_F32) == 32 and H.row_bytes(0, 0, H.PRECISION_F32) == 16


def _fm_rows(rng, n=300):
    keys = np.sort(rng.choice(2 ** 40, n, replace=False).astype(np.uint64))
    return SM.rows_array(keys, rng.normal(0, 1, n), rng.normal(0, 3, n), rng.uniform(0, 50, n))


def _canon_rows(rng, K, n=200):
    keys = np.sort(rng.choice(2 ** 40, n, replace=False).astype(np.uint64))
    return CM.rows_array(keys, rng.normal(0, 1, n), rng.normal(0, 0.3, (n, K)))


def test_convert_fm_rows_and_back():
    rng = np.random.default_rng(1)
    rows = _fm_rows(rng)
    r16 = H.convert(rows, H.PRECISION_F16)
    assert r16.dtype == H.FM_ROW16 and np.array_equal(r16["key"], rows["key"])
    assert np.array_equal(r16["w"].view(np.uint32), rows["w"].view(np.uint32))
    assert np.array_equal(r16["st"].view(np.uint16), rows["st"].astype(np.float16).view(np.uint16))
    back = H.convert(r16, H.PRECISION_F32)
    assert back.dtype == SM.FM_ROW and not np.any(back["pad"])
    assert np.array_equal(back["qt"], H.rounded(rows["qt"]))
    assert H.convert(r16, H.PRECISION_F16).tobytes() == r16.tobytes()  # the same precision: a copy
    assert H.convert(back, H.PRECISION_F16).tobytes() == r16.tobytes()  # rounding is idempotent
    with pytest.raises(ValueError):
        H.convert(SM.rows_array(rows["key"], rows["w"]), H.PRECISION_F16)


@pytest.mark.parametrize("K", CM.LATENT_DIMS)
def test_convert_canonical_rows(K):
    rng = np.random.default_rng(K)
    rows = _canon_rows(rng, K)
    r16 = H.convert(rows, H.PRECISION_F16)
    assert r16.dtype.itemsize == H.row_bytes(CM.FM_CANONICAL, K, H.PRECISION_F16) and H.padding_zero(r16).all()
    assert np.array_equal(H.convert(r16, H.PRECISION_F32)["v"], H.rounded(rows["v"]))


def test_overflow_names_the_count_and_the_smallest_key():
    rows = SM.rows_array(np.array([50, 9, 30, 7], np.uint64), np.ones(4), [1.0, 7e4, 1.0, 1.0], [1.6e5, 1.6e5, 2.0, 65519.0])
    with pytest.raises(H.Overflow) as e:
        H.convert(rows, H.PRECISION_F16)
    assert e.value.count == 3 and e.value.key == 9
    v = np.zeros((3, 16), np.float32)
    v[2, 5] = -7e4
    v[1, :] = np.nan  # NaN stays NaN: not an overflow
    canon = CM.rows_array(np.array([3, 4, 5], np.uint64), np.zeros(3), v)
    with pytest.raises(H.Overflow) as e:
        H.convert(canon, H.PRECISION_F16)
    assert e.value.count == 1 and e.value.key == 5
    v[2, 5] = 65504
    assert np.isnan(H.convert(CM.rows_array(np.array([3, 4, 5], np.uint64), np.zeros(3), v), H.PRECISION_F16)["v"][1]).all()


# ---- files ---------------------------------------------------------------------------------------------------------
def test_f32_files_equal_the_existing_builders():
    rng = np.random.default_rng(3)
    fm = _fm_rows(rng)
    args = (0, 1, 1, 0.0, 11, fm.size + 40)
    assert H.model_file(fm, 1, 16, H.PRECISION_F32, *args) == SM.build_file(fm, 16, *args)
    lr = SM.rows_array(fm["key"], fm["w"])
    assert H.model_file(lr, 0, 0, H.PRECISION_F32, *args) == SM.build_file(lr, 0, *args)
    c = _canon_rows(rng, 16)
    assert H.model_file(c, 2, 16, H.PRECISION_F32, *args) == CM.model_file(c, 16, *args)
    assert H.part_file(fm, 1, 16, H.PRECISION_F32, *args, 1, 3) == P.build_part(fm, 16, *args, 1, 3)
    b = fm[::2].copy()
    b["w"][:10] += 1
    assert H.delta_file(fm, b, b.size + 5, 1, 16, H.PRECISION_F32, *args[:5]) == \
        DM.delta_file(fm, b, b.size + 5, 16, *args[:5])
    cb = c[1:].copy()
    assert H.delta_file(c, cb, cb.size, 2, 16, H.PRECISION_F32, *args[:5]) == CM.delta_file(c, cb, cb.size, 16, *args[:5])


def test_f16_files_carry_the_precision_word():
    rng = np.random.default_rng(4)
    fm = H.convert(_fm_rows(rng), H.PRECISION_F16)
    args = (0, 0, 1, 0.0, 11, fm.size)
    data = H.model_file(fm, 1, 16, H.PRECISION_F16, *args)
    assert struct.unpack_from("<I", data, 60)[0] == 1 and struct.unpack_from("<I", data, 32)[0] == 16
    h, rows = H.parse_model_file(data)
    assert h["precision"] == 1 and rows.tobytes() == fm.tobytes()
    part = H.part_file(fm, 1, 16, H.PRECISION_F16, *args, 0, 2)
    assert struct.unpack_from("<I", part, 60)[0] == 1 and H.parse_model_file(part)[1].tobytes() == fm.tobytes()
    c = H.convert(_canon_rows(rng, 64), H.PRECISION_F16)
    cdata = H.model_file(c, 2, 64, H.PRECISION_F16, *args[:5], c.size)
    assert struct.unpack_from("<I", cdata, 32)[0] == 160 and H.parse_model_file(cdata)[1].tobytes() == c.tobytes()
    d = H.delta_file(fm, fm[1:], fm.size - 1, 1, 16, H.PRECISION_F16, *args[:5])
    hd = dict(zip(DM.FIELDS, DM.HEADER.unpack(d[:DM.HEADER.size])))
    assert hd["zero"] == 1 and hd["row_bytes"] == 16 and hd["deletes"] == 1 and hd["upserts"] == 0


def test_parse_refuses_what_the_loader_refuses():
    rng = np.random.default_rng(5)
    fm = H.convert(_fm_rows(rng, 20), H.PRECISION_F16)
    args = (0, 0, 1, 0.0, 11, fm.size)

    def resum(x):
        x = bytearray(x)
        struct.pack_into("<Q", x, 96, SM.section_sum(bytes(x[:96])))
        return bytes(x)

    good = H.model_file(fm, 1, 16, H.PRECISION_F16, *args)
    for bad in (resum(good[:60] + struct.pack("<I", 2) + good[64:]),  # precision 2
                resum(good[:32] + struct.pack("<I", 32) + good[36:])):  # F16 with F32 row bytes
        with pytest.raises(ValueError):
            H.parse_model_file(bad)
    lr = SM.rows_array(fm["key"], fm["w"])
    lr16 = resum(SM.build_file(lr, 0, *args)[:60] + struct.pack("<I", 1) + SM.build_file(lr, 0, *args)[64:])
    with pytest.raises(ValueError, match="precision"):
        H.parse_model_file(lr16)
    c = H.convert(_canon_rows(rng, 16, 5), H.PRECISION_F16)
    c["pad"][2, 3] = 1
    with pytest.raises(ValueError, match="padding"):
        H.parse_model_file(H.model_file(c, 2, 16, H.PRECISION_F16, *args[:5], c.size))


def test_the_bound_holds_on_random_rows():
    rng = np.random.default_rng(6)
    rp = np.array([0, 0, 1, 5, 50, 200], np.int64)
    n = rp[-1]
    w, st, qt = (rng.normal(0, s, n).astype(np.float32) for s in (1, 2, 1))
    qt = np.abs(qt)
    a32, a16, field, ev = H.fm_bound(rp, w, st, qt)
    assert np.all(np.abs(a16 - a32) <= field + 1e-12) and np.all(ev >= 0) and field[-1] > 0
    x = rng.uniform(-1, 2, n).astype(np.float32)
    v = rng.normal(0, 0.5, (n, 8)).astype(np.float32)
    c32, c16, cf, cev = H.canonical_bound(rp, x, w, v)
    assert np.all(np.abs(c16 - c32) <= cf + 1e-12) and np.all(cev >= 0) and cf[-1] > 0
