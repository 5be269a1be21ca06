"""A numpy statement of half-precision serving models (xf_model_convert, csrc/serve.cu): the F16 rows of FM and canonical
models, the conversion between precisions, the precision word of the XFSM, XFSP and XFSD files, and the bound on how
far an F16 model's predictions may move from the F32 model's.  The GPU tests hold the library to it;
test_compact_serving_model.py checks it against hand cases and against the F32 builders of the other models.

At F16, w stays float32 and only the latent fields (FM st, qt; canonical every v_k) are IEEE binary16, rounded to
nearest even as numpy's astype(np.float16) and CUDA's __float2half_rn both do, subnormals included.  A field finite in
float32 and not in binary16 (|x| >= 65520) is refused, never saturated; a NaN stays a NaN."""
import struct

import numpy as np

import canonical_serving_model as CM
import delta_model as DM
import fm_model as FMM
import serving_model as SM
import serving_parts_model as P

PRECISION_F32, PRECISION_F16 = 0, 1
FM_ROW16 = np.dtype([("key", "<u8"), ("w", "<f4"), ("st", "<f2"), ("qt", "<f2")])
assert FM_ROW16.itemsize == 16


class Overflow(ValueError):
    """Fields finite in float32 that binary16 cannot hold: their number and the smallest key that holds one."""

    def __init__(self, count, key):
        super().__init__("%d latent fields do not fit binary16; smallest key %d" % (count, key))
        self.count, self.key = count, key


def to_half(x):
    """float32 values rounded to nearest even in binary16 (no check)."""
    with np.errstate(over="ignore", invalid="ignore"):
        return np.asarray(x, np.float32).astype(np.float16)


def overflows(x):
    """Which float32 values are finite and round to an infinity in binary16 (|x| >= 65520)."""
    x = np.asarray(x, np.float32)
    return np.isfinite(x) & ~np.isfinite(to_half(x).astype(np.float32))


def rounded(x):
    """The float32 value of each field's binary16 rounding: what an F16 model serves for it."""
    return to_half(x).astype(np.float32)


def row_bytes(fm, K, precision):
    """Bytes of a row: LR 16 (F32 only); FM 32 at F32, 16 at F16; canonical 16 + 4K (F32) or 16 + 2K (F16), rounded
    up to 32."""
    if fm == CM.FM_CANONICAL:
        return (16 + (2 if precision == PRECISION_F16 else 4) * K + 31) // 32 * 32
    if fm == 1:
        return 16 if precision == PRECISION_F16 else 32
    assert precision == PRECISION_F32, "an LR model is F32 only"
    return 16


def canonical_dtype(K, precision):
    """{u64 key, f32 w, u32 0, v[K] (f4 or f2), zero padding}"""
    if precision == PRECISION_F32:
        return CM.row_dtype(K)
    pad = row_bytes(CM.FM_CANONICAL, K, precision) - 16 - 2 * K
    fields = [("key", "<u8"), ("w", "<f4"), ("zero", "<u4"), ("v", "<f2", (K,))]
    if pad:
        fields.append(("pad", "u1", (pad,)))
    return np.dtype(fields)


def row_dtype(fm, K, precision):
    if fm == CM.FM_CANONICAL:
        return canonical_dtype(K, precision)
    if fm == 1:
        return FM_ROW16 if precision == PRECISION_F16 else SM.FM_ROW
    return SM.LR_ROW


def _latent(rows):
    return ("st", "qt") if "st" in rows.dtype.names else ("v",)


def convert(rows, precision):
    """Rows (sorted by key) of an FM or canonical model at `precision`: keys and w as they are, latent fields rounded
    (to F16) or widened exactly (to F32); the same precision gives a copy.  Overflow for fields binary16 cannot hold;
    ValueError for LR rows."""
    names = rows.dtype.names
    if "st" not in names and "v" not in names:
        raise ValueError("an LR model has no latent fields to narrow")
    fm = 1 if "st" in names else CM.FM_CANONICAL
    K = 0 if fm == 1 else rows.dtype["v"].shape[0]
    out = np.zeros(rows.size, row_dtype(fm, K, precision))
    out["key"], out["w"] = rows["key"], rows["w"]
    over = np.zeros(rows.size, np.int64)
    for f in _latent(rows):
        x = np.asarray(rows[f])
        if precision == PRECISION_F16 and x.dtype != np.float16:
            o = overflows(x)
            over += o.reshape(rows.size, -1).sum(axis=1)
            out[f] = to_half(x)
        else:
            out[f] = x.astype(out.dtype[f].base)
    if over.any():
        raise Overflow(int(over.sum()), int(rows["key"][over > 0].min()))
    return out


def padding_zero(rows):
    """Whether every padding byte of the rows is zero (an F16 FM row has none)."""
    names = rows.dtype.names
    ok = np.ones(rows.size, bool)
    if "zero" in names:
        ok &= np.asarray(rows["zero"]) == 0
    if "pad" in names:
        pad = np.asarray(rows["pad"]).reshape(rows.size, -1)
        ok &= ~np.any(pad != 0, axis=1)
    return ok


# ---- files ---------------------------------------------------------------------------------------------------------
def _sections(out, sections, chunk=0):
    for data, per, width in sections:
        for first in range(0, data.size, per):
            body = np.ascontiguousarray(data[first:first + per]).tobytes()
            out.append(struct.pack("<QQQQ", first, len(body) // width, SM.section_sum(body, chunk << 40), 0))
            out.append(body)
            chunk += 1
    return b"".join(out)


def model_header(n, fm, K, precision, optimizer, absent, v_init, v_const, seed, source_keys):
    """The 104-byte XFSM header; byte 60 holds the precision."""
    rb = row_bytes(fm, K, precision)
    head = [b"XFSM", 1, SM.HEADER.size, n, SM.capacity_for(n), rb, fm, K, optimizer, absent, v_init, v_const, precision,
            seed, source_keys, source_keys - n, SM.CHUNK_BYTES // rb, 0]
    head[-1] = SM.section_sum(SM.HEADER.pack(*head)[:96])
    return SM.HEADER.pack(*head)


def model_file(rows, fm, K, precision, optimizer, absent, v_init, v_const, seed, source_keys):
    """The bytes of an XFSM file holding `rows` (sorted by key, row_dtype(fm, K, precision))."""
    rb = row_bytes(fm, K, precision)
    assert rows.dtype.itemsize == rb
    head = model_header(rows.size, fm, K, precision, optimizer, absent, v_init, v_const, seed, source_keys)
    return _sections([head], [(rows, SM.CHUNK_BYTES // rb, rb)])


def part_file(rows, fm, K, precision, optimizer, absent, v_init, v_const, seed, source_keys, shard_index, num_shards):
    """The bytes of the XFSP file of shard shard_index of num_shards holding `rows`: XFSM's bytes [0, 96), precision
    included, then the shard."""
    whole = model_file(rows, fm, K, precision, optimizer, absent, v_init, v_const, seed, source_keys)
    head = list(SM.HEADER.unpack(whole[:SM.HEADER.size]))[:-1]
    head[0], head[2] = b"XFSP", P.PART_HEADER.size
    head += [shard_index, num_shards, 0]
    head[-1] = SM.section_sum(P.PART_HEADER.pack(*head)[:104])
    return P.PART_HEADER.pack(*head) + whole[SM.HEADER.size:]


def parse_model_file(data):
    """(header dict, rows) of an XFSM or XFSP file of any precision; ValueError for what xf_model_load refuses of it:
    a damaged file, a precision other than 0 or 1, row bytes other than those of (fm, K, precision), keys that do not
    ascend, non-zero padding."""
    part = data[:4] == b"XFSP"
    hs = P.PART_HEADER if part else SM.HEADER
    if len(data) < hs.size or data[:4] not in (b"XFSM", b"XFSP"):
        raise ValueError("not a model file")
    h = dict(zip(P.PART_FIELDS if part else SM.FIELDS, hs.unpack(data[:hs.size])))
    if h["header_checksum"] != SM.section_sum(data[:hs.size - 8]):
        raise ValueError("header checksum")
    fm, K, precision = h["fm"], h["latent_dim"], h["zero"]
    if precision not in (PRECISION_F32, PRECISION_F16) or (fm == 0 and precision != PRECISION_F32):
        raise ValueError("precision")
    if fm == CM.FM_CANONICAL and K not in CM.LATENT_DIMS:
        raise ValueError("latent_dim")
    rb = row_bytes(fm, K, precision)
    if h["row_bytes"] != rb or h["chunk_rows"] != SM.CHUNK_BYTES // rb or h["capacity"] != SM.capacity_for(h["keys"]):
        raise ValueError("header fields")
    dt = row_dtype(fm, K, precision)
    parts, pos, first, chunk = [], hs.size, 0, 0
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
    if rows.size and np.any(rows["key"][1:] <= rows["key"][:-1]):
        raise ValueError("keys not ascending")
    if fm != CM.FM_CANONICAL and precision == PRECISION_F32:
        if rows.size and np.any(np.ascontiguousarray(rows["pad"]) != 0):
            raise ValueError("non-zero padding")
    elif not padding_zero(rows).all():
        raise ValueError("non-zero padding")
    h["precision"] = precision
    return h, rows


def delta_file(a, b, b_source_keys, fm, K, precision, optimizer, absent, v_init, v_const, seed):
    """The XFSD file of the delta from rows a to rows b of one precision; byte 52 holds the precision."""
    rb = row_bytes(fm, K, precision)
    up, de = DM.diff(a, b)
    de = np.ascontiguousarray(de, np.uint64)
    head = [b"XFSD", 1, DM.HEADER.size, fm, K, optimizer, absent, v_init, v_const, seed, rb, precision, a.size,
            DM.fingerprint(a), b.size, b_source_keys, b_source_keys - b.size, DM.fingerprint(b), up.size, de.size,
            SM.CHUNK_BYTES // rb, DM.CHUNK_KEYS, 0]
    head[-1] = SM.section_sum(DM.HEADER.pack(*head)[:136])
    return _sections([DM.HEADER.pack(*head)], [(up, SM.CHUNK_BYTES // rb, rb), (de, DM.CHUNK_KEYS, 8)])


# ---- the bound -----------------------------------------------------------------------------------------------------
def _rows_of(rp, per_token):
    """float64 sums over each CSR row of per-token values [nnz] or [nnz, K]"""
    rp = np.asarray(rp, np.int64)
    x = np.asarray(per_token, np.float64)
    c = np.concatenate([np.zeros((1,) + x.shape[1:]), np.cumsum(x, axis=0)])
    return c[rp[1:]] - c[rp[:-1]]


def fm_bound(rp, w, st, qt):
    """For FM rows over tokens with float32 fields w, st, qt [nnz] (what each token reads from the F32 model):
    (arg32, arg16, field, eval): each row's argument wx + S^2 - Q in float64 from the F32 fields and from their
    binary16 roundings, the bound (2|S| + dS) dS + dQ on their difference (dS = sum |st - r(st)|, dQ = sum
    |qt - r(qt)|), and a bound on either kernel's float32 evaluation error, in fm_model.gamma's style."""
    t = np.diff(np.asarray(rp, np.int64))
    w, st, qt = (np.asarray(a, np.float64) for a in (w, st, qt))
    rs, rq = rounded(st).astype(np.float64), rounded(qt).astype(np.float64)
    W, S, Q = _rows_of(rp, w), _rows_of(rp, st), _rows_of(rp, qt)
    S16, Q16 = _rows_of(rp, rs), _rows_of(rp, rq)
    arg32, arg16 = W + S * S - Q, W + S16 * S16 - Q16
    dS, dQ = _rows_of(rp, np.abs(st - rs)), _rows_of(rp, np.abs(qt - rq))
    field = (2 * np.abs(S) + dS) * dS + dQ
    g = FMM.gamma(t)
    Wa = _rows_of(rp, np.abs(w))
    Sa = np.maximum(_rows_of(rp, np.abs(st)), _rows_of(rp, np.abs(rs)))
    Qa = np.maximum(_rows_of(rp, np.abs(qt)), _rows_of(rp, np.abs(rq)))
    eS = g * Sa
    Smax = np.maximum(np.abs(S), np.abs(S16))
    ev = g * Wa + (2 * Smax + eS) * eS + g * Qa + FMM.gamma(3) * (Wa + (Smax + eS) ** 2 + Qa)
    return arg32, arg16, field, FMM.SAFETY * ev


def canonical_bound(rp, x, w, v):
    """The same for canonical rows over tokens with values x [nnz], w [nnz] and v [nnz, K] (float32, what each token
    reads from the F32 model): arg = wx + (sum_k S_k^2 - Q) / 2 with S_k = sum x v_k and Q = sum (x v_k)^2.  The field
    term is (sum_k (2|S_k| + dS_k) dS_k + dQ) / 2 with dS_k = sum |x| |v_k - r(v_k)| and dQ = sum x^2 |v_k^2 - r(v_k)^2|."""
    t = np.diff(np.asarray(rp, np.int64))
    K = np.asarray(v).shape[1]
    x, w, v = np.asarray(x, np.float64), np.asarray(w, np.float64), np.asarray(v, np.float64)
    rv = rounded(v).astype(np.float64)
    a, ar = x[:, None] * v, x[:, None] * rv
    W = _rows_of(rp, w * x)
    Sk, Sk16 = _rows_of(rp, a), _rows_of(rp, ar)
    Q, Q16 = _rows_of(rp, (a * a).sum(axis=1)), _rows_of(rp, (ar * ar).sum(axis=1))
    arg32 = W + 0.5 * ((Sk * Sk).sum(axis=1) - Q)
    arg16 = W + 0.5 * ((Sk16 * Sk16).sum(axis=1) - Q16)
    dS = _rows_of(rp, np.abs(x)[:, None] * np.abs(v - rv))
    dQ = _rows_of(rp, ((x * x)[:, None] * np.abs(v * v - rv * rv)).sum(axis=1))
    field = 0.5 * (((2 * np.abs(Sk) + dS) * dS).sum(axis=1) + dQ)
    # evaluation: products (1 rounding), S_k over t terms, Q over t K terms, s2 over K terms, wx over t, 3 at the end
    Wa = _rows_of(rp, np.abs(w * x))
    Ska = np.maximum(_rows_of(rp, np.abs(a)), _rows_of(rp, np.abs(ar)))
    Qa = np.maximum(Q, Q16)
    eS = FMM.gamma(t + 1)[:, None] * Ska
    s2 = ((np.maximum(np.abs(Sk), np.abs(Sk16)) + eS) ** 2).sum(axis=1)
    ev = (FMM.gamma(t + 1) * Wa + (2 * Ska * eS + eS * eS).sum(axis=1) + FMM.gamma(t * K + 2) * Qa
          + FMM.gamma(K + 1) * s2 + FMM.gamma(3) * (Wa + 0.5 * (s2 + Qa)))
    return arg32, arg16, field, FMM.SAFETY * ev
