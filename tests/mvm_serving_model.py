"""A numpy statement of multi-view machine serving models (xf_table_freeze_mvm, csrc/serve.cu): the row {key, u64 0,
v[K], zero padding} at F32 and F16, its padding rule, the two prune rules, the XFSM / XFSD bytes with fm = 3, the
fingerprint, and the forward in float32, op for op in the order header section 6 states.  The GPU tests hold the library
to it; test_mvm_serving_model.py checks it on hand-built rows and against the float64 definition."""
import struct

import numpy as np

import compact_serving_model as CS
import delta_model as DM
import serving_model as SM

FM_MVM = 3  # the fm field of xf_model_info, XFSM and XFSD
LATENT_DIMS = (4, 8, 16, 32)
FIELDS = 32  # field ids are below 32; the kernels read fields[j] & 31
PRECISION_F32, PRECISION_F16 = CS.PRECISION_F32, CS.PRECISION_F16
P_MIN = np.float32(1e-6)


def row_bytes(K, precision=PRECISION_F32):
    """The canonical row's bytes: 16 + 4K (F32) or 16 + 2K (F16), rounded up to 32."""
    return (16 + (2 if precision == PRECISION_F16 else 4) * K + 31) // 32 * 32


def row_dtype(K, precision=PRECISION_F32):
    """{u64 key, u64 0, v[K] (f4 or f2), zero padding}: lane c's piece of v at 16 + 16c (F32) or 16 + 8c (F16)."""
    vb = 2 if precision == PRECISION_F16 else 4
    pad = row_bytes(K, precision) - 16 - vb * K
    fields = [("key", "<u8"), ("zero", "<u8"), ("v", "<f2" if vb == 2 else "<f4", (K,))]
    if pad:
        fields.append(("pad", "u1", (pad,)))
    dt = np.dtype(fields)
    assert dt.itemsize == row_bytes(K, precision)
    return dt


def rows_array(keys, v, precision=PRECISION_F32):
    """Packed rows sorted by key (v: [n, K] float32, rounded to binary16 at F16)."""
    keys = np.asarray(keys, np.uint64)
    v = np.asarray(v, np.float32).reshape(keys.size, -1)
    order = np.argsort(keys, kind="stable")
    rows = np.zeros(keys.size, row_dtype(v.shape[1], precision))
    rows["key"] = keys[order]
    rows["v"] = CS.to_half(v[order]) if precision == PRECISION_F16 else v[order]
    return rows


def padding_zero(rows):
    """Whether every padding byte is zero: bytes 8 .. 15 (the row holds no w) and the tail after v."""
    ok = np.asarray(rows["zero"]) == 0
    if "pad" in rows.dtype.names:
        ok &= ~np.any(np.asarray(rows["pad"]).reshape(rows.size, -1) != 0, axis=1)
    return ok


def pruned(absent, v_ready, v):
    """Rows prune = 1 leaves out, w playing no part: under DEFAULT a latent block that is not materialised; under ZERO
    every resolved v_k == +-0 (v: the resolved latent rows, [n, K])."""
    if absent == SM.ABSENT_DEFAULT:
        return ~np.asarray(v_ready, bool)
    return np.all(np.asarray(v, np.float32) == 0, axis=1)


def fingerprint(rows):
    """The order-free fingerprint over the row's row_bytes / 8 words (delta_model.fingerprint's chain)."""
    return DM.fingerprint(rows)


def convert(rows, precision):
    """The rows at `precision`: v rounded to nearest even (to F16) or widened exactly (to F32), the zero word copied;
    compact_serving_model.Overflow for fields binary16 cannot hold."""
    K = rows.dtype["v"].shape[0]
    out = np.zeros(rows.size, row_dtype(K, precision))
    out["key"], out["zero"] = rows["key"], rows["zero"]
    x = np.asarray(rows["v"])
    if precision == PRECISION_F16 and x.dtype != np.float16:
        over = CS.overflows(x).sum(axis=1)
        if over.any():
            raise CS.Overflow(int(over.sum()), int(rows["key"][over > 0].min()))
        out["v"] = CS.to_half(x)
    else:
        out["v"] = x.astype(out.dtype["v"].base)
    return out


# ---- files ---------------------------------------------------------------------------------------------------------
def model_file(rows, K, precision, optimizer, absent, v_init, v_const, seed, source_keys):
    """The bytes of the XFSM file holding `rows` (rows_array): fm = 3 at byte 36, the precision at byte 60."""
    rb = row_bytes(K, precision)
    assert rows.dtype.itemsize == rb
    n = rows.size
    head = [b"XFSM", 1, SM.HEADER.size, n, SM.capacity_for(n), rb, FM_MVM, K, optimizer, absent, v_init, v_const,
            precision, seed, source_keys, source_keys - n, SM.CHUNK_BYTES // rb, 0]
    head[-1] = SM.section_sum(SM.HEADER.pack(*head)[:96])
    return CS._sections([SM.HEADER.pack(*head)], [(rows, SM.CHUNK_BYTES // rb, rb)])


def parse_model_file(data):
    """(header dict, rows) of a multi-view machine's XFSM file; ValueError for what xf_model_load refuses of it."""
    if len(data) < SM.HEADER.size or data[:4] != b"XFSM":
        raise ValueError("not an XFSM file")
    h = dict(zip(SM.FIELDS, SM.HEADER.unpack(data[:SM.HEADER.size])))
    if h["header_checksum"] != SM.section_sum(data[:96]):
        raise ValueError("header checksum")
    K, precision = h["latent_dim"], h["zero"]
    if h["fm"] != FM_MVM or K not in LATENT_DIMS or precision not in (PRECISION_F32, PRECISION_F16):
        raise ValueError("header fields")
    rb = row_bytes(K, precision)
    if h["row_bytes"] != rb or h["chunk_rows"] != SM.CHUNK_BYTES // rb or h["capacity"] != SM.capacity_for(h["keys"]):
        raise ValueError("header fields")
    dt = row_dtype(K, precision)
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
    if rows.size and (np.any(rows["key"][1:] <= rows["key"][:-1]) or not padding_zero(rows).all()):
        raise ValueError("keys not ascending or non-zero padding")
    h["precision"] = precision
    return h, rows


def delta_file(a, b, b_source_keys, K, precision, optimizer, absent, v_init, v_const, seed):
    """The XFSD file of the delta from rows a to rows b: fm = 3 at byte 16, the precision at byte 52."""
    rb = row_bytes(K, precision)
    up, de = DM.diff(a, b)
    de = np.ascontiguousarray(de, np.uint64)
    head = [b"XFSD", 1, DM.HEADER.size, FM_MVM, K, optimizer, absent, v_init, v_const, seed, rb, precision, a.size,
            DM.fingerprint(a), b.size, b_source_keys, b_source_keys - b.size, DM.fingerprint(b), up.size, de.size,
            SM.CHUNK_BYTES // rb, DM.CHUNK_KEYS, 0]
    head[-1] = SM.section_sum(DM.HEADER.pack(*head)[:136])
    return CS._sections([DM.HEADER.pack(*head)], [(up, SM.CHUNK_BYTES // rb, rb), (de, DM.CHUNK_KEYS, 8)])


# ---- the forward ---------------------------------------------------------------------------------------------------
def sigmoid(y):
    """xf_sigmoid (table.cuh) of float32 arguments: 1e-6 below -30, 1 above 30, else exp in double, rounded to float."""
    y = np.asarray(y, np.float32)
    with np.errstate(over="ignore", invalid="ignore"):
        ex = np.exp(y.astype(np.float64) * 0.9999999998311266)
        mid = (ex / (1.0 + ex)).astype(np.float32)
    return np.where(y < -30.0, P_MIN, np.where(y > 30.0, np.float32(1.0), mid)).astype(np.float32)


def forward(rp, fields, x, v):
    """(y, pctr) float32 of each CSR row, the model's forward op for op: v [nnz, K] the rows the tokens read (the absent
    policy applied), fields [nnz] (read & 31), x [nnz] or None (all 1).
        S[f][k] = +0;  for j in token order: S[f_j][k] = S[f_j][k] + (v_jk * x_j)
        P_k = 1;  for the present fields f ascending: P_k = P_k * S[f][k]     (no tokens: P_k = 0)
        y = the 32-lane butterfly sum (xor 16, 8, 4, 2, 1) of P_0 .. P_K-1 and zeros;  pctr = sigmoid(y)
    Every operation is one float32 rounding to nearest, as numpy's float32 arithmetic is."""
    rp = np.asarray(rp, np.int64)
    v = np.asarray(v, np.float32)
    nnz, K = v.shape
    B = rp.size - 1
    f = np.asarray(fields, np.int64) & (FIELDS - 1)
    x = np.ones(nnz, np.float32) if x is None else np.asarray(x, np.float32)
    with np.errstate(all="ignore"):
        a = v * x[:, None]  # one float32 product per (token, k)
        lens = np.diff(rp)
        S = np.zeros((B, FIELDS, K), np.float32)
        present = np.zeros((B, FIELDS), bool)
        for t in range(int(lens.max()) if B else 0):
            r = np.nonzero(lens > t)[0]
            j = rp[r] + t
            S[r, f[j]] = S[r, f[j]] + a[j]  # the rows are distinct: one add per (row, field, k) per t
            present[r, f[j]] = True
        P = np.ones((B, K), np.float32)
        for q in range(FIELDS):
            m = present[:, q]
            P[m] = P[m] * S[m, q]
        P[~present.any(axis=1)] = 0
        lanes = np.zeros((B, 32), np.float32)
        lanes[:, :K] = P
        idx = np.arange(32)
        for o in (16, 8, 4, 2, 1):
            lanes = lanes + lanes[:, idx ^ o]
        y = lanes[:, 0].copy()
    return y, sigmoid(y)


def forward64(rp, fields, x, v):
    """y of each row in float64 by the definition: sum_k prod_{fields present} (sum_{tokens of the field} v_k x)."""
    rp = np.asarray(rp, np.int64)
    v = np.asarray(v, np.float64)
    B, K = rp.size - 1, v.shape[1]
    f = np.asarray(fields, np.int64) & (FIELDS - 1)
    x = np.ones(v.shape[0]) if x is None else np.asarray(x, np.float64)
    row_of = np.repeat(np.arange(B), np.diff(rp))
    S = np.zeros((B, FIELDS, K))
    np.add.at(S, (row_of, f), v * x[:, None])
    present = np.zeros((B, FIELDS), bool)
    present[row_of, f] = True
    Sp = np.where(present[:, :, None], S, 1.0)
    return np.where(present.any(axis=1), Sp.prod(axis=1).sum(axis=1), 0.0)


def collision_free(rp, fields, K):
    """Rows on which the table's predict is reproducible, so the model equals it bit for bit: no field holds more than
    two tokens, or no pass of the step kernel (T = 128 / K consecutive tokens from the row's first) holds two tokens of
    one field."""
    rp = np.asarray(rp, np.int64)
    f = np.asarray(fields, np.int64) & (FIELDS - 1)
    T = 128 // K
    out = np.zeros(rp.size - 1, bool)
    for r in range(rp.size - 1):
        fr = f[rp[r]:rp[r + 1]]
        if fr.size == 0 or np.bincount(fr, minlength=FIELDS).max() <= 2:
            out[r] = True
            continue
        out[r] = all(np.unique(fr[p:p + T]).size == fr[p:p + T].size for p in range(0, fr.size, T))
    return out
