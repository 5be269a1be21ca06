"""CPU checks of the field-aware FM serving statement (ffm_serving_model.py): the row and file layout with fm = 4, the
prune rule's claim that a pruned row reads as the absent policy's row bit for bit, and the candidate kernel's fold
algebra."""
import struct

import numpy as np
import pytest

import canonical_serving_model as CM
import compact_serving_model as CS
import ffm_serving_model as FS
import serving_model as SM


def test_row_layout_and_padding():
    for L in FS.LATENT_DIMS:
        assert FS.row_bytes(L) == CM.row_bytes(L) == (16 + 4 * L + 31) // 32 * 32
        assert FS.row_bytes(L, CS.PRECISION_F16) == (16 + 2 * L + 31) // 32 * 32
    assert [FS.row_bytes(L) for L in FS.LATENT_DIMS] == [32, 64, 96, 160, 288, 544]
    rows = CM.rows_array(np.array([9, 3], np.uint64), np.array([1.5, -0.0], np.float32),
                         np.arange(32, dtype=np.float32).reshape(2, 16))
    assert rows.dtype.itemsize == 96 and rows["key"].tolist() == [3, 9] and CM.padding_zero(rows).all()
    raw = bytearray(rows.tobytes())
    raw[12] = 1
    assert not CM.padding_zero(np.frombuffer(bytes(raw), rows.dtype))[0]


def test_model_and_delta_files_with_fm_4():
    L = 16
    rows = CM.rows_array(np.arange(1, 40, dtype=np.uint64) * 977, np.linspace(-1, 1, 39).astype(np.float32),
                         np.random.default_rng(0).normal(size=(39, L)).astype(np.float32))
    data = FS.model_file(rows, L, CS.PRECISION_F32, 0, 0, 1, 0.0, 7, 45)
    assert struct.unpack_from("<i", data, 36)[0] == FS.FM_FFM
    h, back = FS.parse_model_file(data)
    assert back.tobytes() == rows.tobytes() and h["pruned_keys"] == 6 and h["row_bytes"] == 96
    with pytest.raises(ValueError):
        CM.parse_model_file(data)  # not a canonical model's file
    # the canonical file differs in fm alone, at byte 36 and in the header checksum
    canon = CM.model_file(rows, L, 0, 0, 1, 0.0, 7, 45)
    assert canon[104:] == data[104:] and canon[:36] == data[:36] and canon[40:96] == data[40:96]
    with pytest.raises(ValueError):
        FS.parse_model_file(canon)
    # a damaged padding byte, with checksums that pass
    raw = bytearray(rows.tobytes())
    raw[96 * 3 + 12] = 1
    with pytest.raises(ValueError):
        FS.parse_model_file(FS.model_file(np.frombuffer(bytes(raw), rows.dtype), L, CS.PRECISION_F32, 0, 0, 1, 0.0, 7, 45))
    # F16 rows: 16 + 2L bytes rounded up to 32
    r16 = CS.convert(rows, CS.PRECISION_F16)
    h16, back16 = FS.parse_model_file(FS.model_file(r16, L, CS.PRECISION_F16, 0, 0, 1, 0.0, 7, 45))
    assert h16["precision"] == 1 and h16["row_bytes"] == 64 and back16.tobytes() == r16.tobytes()
    # the delta: the canonical one's bytes with fm = 4 at byte 16
    d = FS.delta_file(rows[:30], rows[5:], 50, L, CS.PRECISION_F32, 0, 0, 1, 0.0, 7)
    dc = CM.delta_file(rows[:30], rows[5:], 50, L, 0, 0, 1, 0.0, 7)
    assert struct.unpack_from("<i", d, 16)[0] == FS.FM_FFM and struct.unpack_from("<i", dc, 16)[0] == CM.FM_CANONICAL
    assert d[144:] == dc[144:] and d[:16] == dc[:16] and d[20:136] == dc[20:136]
    assert SM.HEADER.size == 104


def _tokens(rng, n, L, w_zero=False):
    F = L // 4
    return (rng.normal(0, 1, n).astype(np.float32), rng.normal(0, 1, (n, L)).astype(np.float32),
            rng.integers(0, F, n).astype(np.uint8), rng.uniform(-2, 2, n).astype(np.float32))


@pytest.mark.parametrize("L", [4, 16, 64])
def test_a_pruned_row_reads_as_the_absent_row(L):
    """Under ZERO a row with w == +-0 and every v_k == +-0 is pruned and read as zeros; under DEFAULT a row with
    w == +-0 and its initial v is pruned and read as w = +0 and the same v.  Either gives the same T, Σwx and Q bits,
    wherever the token sits and whatever its value, NaN and +-Inf included."""
    rng = np.random.default_rng(L)
    w, v, f, x = _tokens(rng, 12, L)
    init = rng.normal(0, 0.01, L).astype(np.float32)
    signed = np.where(rng.random(L) < 0.5, np.float32(-0.0), np.float32(0.0)).astype(np.float32)
    for value in (np.float32(0.7), np.float32(-3.0), np.float32(0.0), np.float32(np.nan), np.float32(np.inf),
                  np.float32(-np.inf)):
        for pos in (0, 5, 12):
            for pruned_v, absent_v in ((signed, np.zeros(L, np.float32)), (init, init)):
                for pruned_w in (np.float32(0.0), np.float32(-0.0)):
                    def row(wi, vi):
                        ww = np.insert(w, pos, wi)
                        vv = np.insert(v, pos, vi[None, :], axis=0)
                        return FS.fold(FS.empty_state(L), ww, vv, np.insert(f, pos, f[0]), np.insert(x, pos, value))
                    a, b = row(pruned_w, pruned_v), row(np.float32(0.0), absent_v)
                    assert FS.same_state(a, b), (value, pos, pruned_w)
    # the sums never become -0, so the claim does not rest on the order of the zeros
    s = FS.fold(FS.empty_state(L), np.full(3, -0.0, np.float32), np.full((3, L), -0.0, np.float32),
                np.zeros(3, np.uint8), np.ones(3, np.float32))
    assert not np.signbit(s[0]).any() and not np.signbit(s[1]) and not np.signbit(s[2])


@pytest.mark.parametrize("L", [4, 8, 32, 128])
def test_candidate_fold_equals_the_concatenated_row(L):
    """Fold the context once, copy T to T0; each candidate continues from that state, and restoring the rows of its own
    fields from T0 gives back the context's state; the continued state equals the fold of "context, then candidate"."""
    rng = np.random.default_rng(L + 1)
    F = L // 4
    ctx = _tokens(rng, 9, L)
    ctx[2][::2] = 0  # several context tokens of one field
    s_ctx = FS.fold(FS.empty_state(L), *ctx)
    T0 = s_ctx[0].copy()
    T = s_ctx[0].copy()
    for c in range(6):
        cand = _tokens(rng, [0, 1, 3, 7, 12, 2][c], L)
        if cand[2].size:
            cand[2][0] = ctx[2][0]  # a field shared with the context
            cand[2][-1] = cand[2][0]
        cont = FS.fold((T, s_ctx[1], s_ctx[2], s_ctx[3]), *cand)
        flat = FS.fold(FS.empty_state(L), *(np.concatenate([a, b]) for a, b in zip(ctx, cand)))
        assert FS.same_state(cont, flat), c
        T = cont[0].copy()
        for f in np.unique(cand[2].astype(np.int64) & (F - 1)):
            T[f] = T0[f]
        assert np.array_equal(FS.bits(T), FS.bits(T0)), c


def test_candidate_batch_and_concatenation():
    rng = np.random.default_rng(3)
    pool = np.arange(100, 200, dtype=np.uint64)
    cb = FS.candidate_batch(rng, pool, 8, [2, 0, 3], [4, 0, 1], [0, 2, 5])
    ctx_ptr, ctx_keys, cand_ptr, row_ptr, keys, ctx_vals, vals, ctx_fields, fields = cb
    assert cand_ptr.tolist() == [0, 2, 2, 5] and ctx_ptr.tolist() == [0, 4, 4, 5]
    assert row_ptr.tolist() == [0, 0, 2, 7, 7, 9] and (fields < 8).all() and (ctx_fields < 8).all()
    rp, k, f, x = FS.concatenated(*cb)
    assert np.diff(rp.astype(np.int64)).tolist() == [4, 6, 6, 1, 3]
    assert k[:4].tolist() == ctx_keys[:4].tolist() and k[4:8].tolist() == ctx_keys[:4].tolist()
    assert k[8:10].tolist() == keys[:2].tolist() and x[-2:].tolist() == vals[-2:].tolist()
