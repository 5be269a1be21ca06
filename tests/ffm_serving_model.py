"""A numpy statement of field-aware FM serving models (xf_table_freeze_ffm, csrc/serve.cu): the row is the canonical one
(canonical_serving_model, compact_serving_model at F16); the XFSM / XFSD bytes with fm = 4; the forward's state (field
sums T, Σwx, Q, present fields) as a float32 left fold in token order, which the prune rule and the candidate kernel
rest on; and the candidate batches the GPU tests score.  The float64 reference of the forward is ffm_model.FFM64.forward.
"""
import struct

import numpy as np

import canonical_serving_model as CM
import compact_serving_model as CS
import delta_model as DM
import serving_model as SM

FM_FFM = 4  # the fm field of xf_model_info, XFSM and XFSD
LATENT_DIMS = CM.LATENT_DIMS
PIECE = 4  # coordinates per field vector: F = L / 4 fields


def row_bytes(L, precision=CS.PRECISION_F32):
    """The canonical row's bytes: 16 + 4L (F32) or 16 + 2L (F16), rounded up to 32."""
    return CS.row_bytes(CM.FM_CANONICAL, L, precision)


def row_dtype(L, precision=CS.PRECISION_F32):
    """{u64 key, f32 w, u32 0, v[L] (f4 or f2), zero padding}: the canonical row."""
    return CS.canonical_dtype(L, precision)


# ---- files ---------------------------------------------------------------------------------------------------------
def model_file(rows, L, precision, optimizer, absent, v_init, v_const, seed, source_keys):
    """The bytes of the XFSM file holding `rows` (sorted by key, row_dtype(L, precision)): the canonical file with
    fm = 4 at byte 36 and the precision at byte 60."""
    rb = row_bytes(L, precision)
    assert rows.dtype.itemsize == rb
    n = rows.size
    head = [b"XFSM", 1, SM.HEADER.size, n, SM.capacity_for(n), rb, FM_FFM, L, optimizer, absent, v_init, v_const,
            precision, seed, source_keys, source_keys - n, SM.CHUNK_BYTES // rb, 0]
    head[-1] = SM.section_sum(SM.HEADER.pack(*head)[:96])
    return CS._sections([SM.HEADER.pack(*head)], [(rows, SM.CHUNK_BYTES // rb, rb)])


def parse_model_file(data):
    """(header dict, rows) of a field-aware FM's XFSM file; ValueError for what xf_model_load refuses of it: a damaged
    file, fm other than 4, a latent_dim outside LATENT_DIMS, row bytes other than L's, keys that do not ascend, non-zero
    padding."""
    if len(data) < SM.HEADER.size or data[:4] != b"XFSM":
        raise ValueError("not an XFSM file")
    h = dict(zip(SM.FIELDS, SM.HEADER.unpack(data[:SM.HEADER.size])))
    if h["header_checksum"] != SM.section_sum(data[:96]):
        raise ValueError("header checksum")
    L, precision = h["latent_dim"], h["zero"]
    if h["fm"] != FM_FFM or L not in LATENT_DIMS or precision not in (CS.PRECISION_F32, CS.PRECISION_F16):
        raise ValueError("header fields")
    rb = row_bytes(L, precision)
    if h["row_bytes"] != rb or h["chunk_rows"] != SM.CHUNK_BYTES // rb or h["capacity"] != SM.capacity_for(h["keys"]):
        raise ValueError("header fields")
    dt = row_dtype(L, precision)
    parts, pos, first, chunk = [], SM.HEADER.size, 0, 0
    while first < h["keys"]:
        f0, n, s, z = struct.unpack("<QQQQ", data[pos:pos + 32]) if pos + 32 <= len(data) else (None,) * 4
        body = data[pos + 32:pos + 32 + (n or 0) * rb]
        if f0 != first or z != 0 or not n or len(body) != n * rb or s != SM.section_sum(body, chunk << 40):
            raise ValueError("chunk %d" % chunk)
        parts.append(np.frombuffer(body, dt))
        pos += 32 + len(body)
        first += n
        chunk += 1
    if pos != len(data):
        raise ValueError("trailing bytes")
    rows = np.concatenate(parts) if parts else np.zeros(0, dt)
    if rows.size and (np.any(rows["key"][1:] <= rows["key"][:-1]) or not CS.padding_zero(rows).all()):
        raise ValueError("keys not ascending or non-zero padding")
    h["precision"] = precision
    return h, rows


def delta_file(a, b, b_source_keys, L, precision, optimizer, absent, v_init, v_const, seed):
    """The XFSD file of the delta from rows a to rows b: fm = 4 at byte 16, the precision at byte 52."""
    rb = row_bytes(L, precision)
    up, de = DM.diff(a, b)
    de = np.ascontiguousarray(de, np.uint64)
    head = [b"XFSD", 1, DM.HEADER.size, FM_FFM, L, optimizer, absent, v_init, v_const, seed, rb, precision, a.size,
            DM.fingerprint(a), b.size, b_source_keys, b_source_keys - b.size, DM.fingerprint(b), up.size, de.size,
            SM.CHUNK_BYTES // rb, DM.CHUNK_KEYS, 0]
    head[-1] = SM.section_sum(DM.HEADER.pack(*head)[:136])
    return CS._sections([DM.HEADER.pack(*head)], [(up, SM.CHUNK_BYTES // rb, rb), (de, DM.CHUNK_KEYS, 8)])


# ---- the forward's state -------------------------------------------------------------------------------------------
def _fma(a, b, c):
    """fma in float32 through float64: the product is exact there, the sum is rounded twice.  The folds below are
    compared with themselves, so this is enough for their algebra."""
    return np.float32(np.float64(a) * np.float64(b) + np.float64(c))


def empty_state(L):
    """T[a][b] (F x F x 4), Σwx, Q, present fields: all +0."""
    F = L // PIECE
    return np.zeros((F, F, PIECE), np.float32), np.float32(0.0), np.float32(0.0), np.zeros(F, bool)


def fold(state, w, v, fields, x):
    """The state after the tokens (w [n], v [n, L], fields [n], x [n]) in token order, op by op as the kernels:
        a = v x;  T[f][*] = T[f][*] + a;  Q = Q + fma(a3, a3, fma(a2, a2, fma(a1, a1, a0 a0))) of piece f;
        Σwx = Σwx + w x;  field f present."""
    T, wx, Q, present = state
    T, present = T.copy(), present.copy()
    F = T.shape[0]
    with np.errstate(all="ignore"):
        for i in range(len(fields)):
            f = int(fields[i]) & (F - 1)
            xi = np.float32(x[i])
            a = (np.asarray(v[i], np.float32) * xi).reshape(F, PIECE)
            T[f] = T[f] + a
            s = a[f]
            Q = np.float32(Q + _fma(s[3], s[3], _fma(s[2], s[2], _fma(s[1], s[1], s[0] * s[0]))))
            wx = np.float32(wx + np.float32(w[i]) * xi)
            present[f] = True
    return T, wx, Q, present


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def same_state(s, t):
    """Whether two states hold the same bits."""
    return (np.array_equal(bits(s[0]), bits(t[0])) and bits(s[1]) == bits(t[1]) and bits(s[2]) == bits(t[2])
            and np.array_equal(s[3], t[3]))


# ---- candidate batches ----------------------------------------------------------------------------------------------
def candidate_batch(rng, pool, F, counts, ctx_lens, cand_lens):
    """(ctx_ptr, ctx_keys, cand_ptr, row_ptr, keys, ctx_vals, vals, ctx_fields, fields) in Model.predict_candidates'
    order: request q has ctx_lens[q] context tokens and counts[q] candidates, whose lengths cycle through cand_lens.
    Field ids below F, each side holding repeated fields and sharing fields with the other."""
    def side(n):
        k = pool[rng.integers(0, pool.size, n)].astype(np.uint64)
        f = rng.integers(0, F, n).astype(np.uint8)
        f[::3] = f[0] if n else 0
        x = rng.uniform(-1.2, 1.5, n).astype(np.float32)
        return k, f, x

    ctx = [side(n) for n in ctx_lens]
    lens = [cand_lens[i % len(cand_lens)] for i in range(sum(counts))]
    cand = [side(n) for n in lens]
    ptr = lambda ls: np.concatenate([[0], np.cumsum(ls)]).astype(np.uint32)
    cat = lambda parts, j, dt: np.concatenate([p[j] for p in parts]).astype(dt) if parts else np.zeros(0, dt)
    return (ptr(ctx_lens), cat(ctx, 0, np.uint64), ptr(counts), ptr(lens), cat(cand, 0, np.uint64),
            cat(ctx, 2, np.float32), cat(cand, 2, np.float32), cat(ctx, 1, np.uint8), cat(cand, 1, np.uint8))


def concatenated(ctx_ptr, ctx_keys, cand_ptr, row_ptr, keys, ctx_vals, vals, ctx_fields, fields):
    """The flat batch (row_ptr, keys, fields, vals) whose row c is candidate c's request's context, then its tokens."""
    rows, lens = [], []
    for q in range(cand_ptr.size - 1):
        a, b = int(ctx_ptr[q]), int(ctx_ptr[q + 1])
        for c in range(int(cand_ptr[q]), int(cand_ptr[q + 1])):
            s, e = int(row_ptr[c]), int(row_ptr[c + 1])
            rows.append((np.concatenate([ctx_keys[a:b], keys[s:e]]), np.concatenate([ctx_fields[a:b], fields[s:e]]),
                         np.concatenate([ctx_vals[a:b], vals[s:e]])))
            lens.append(b - a + e - s)
    rp = np.concatenate([[0], np.cumsum(lens)]).astype(np.uint32)
    cat = lambda j, dt: np.concatenate([r[j] for r in rows]).astype(dt) if rows else np.zeros(0, dt)
    return rp, cat(0, np.uint64), cat(1, np.uint8), cat(2, np.float32)
