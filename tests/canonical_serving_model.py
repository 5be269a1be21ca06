"""A numpy statement of canonical serving models (xf_table_freeze_canonical, csrc/serve.cu): the row stride and packing,
the two prune rules, the XFSM / XFSD headers of a canonical model and its fingerprint.  The GPU tests hold the library
to it; test_canonical_serving_model.py checks it against hand-built rows."""
import struct

import numpy as np

import delta_model as DM
import serving_model as SM

FM_CANONICAL = 2  # the fm field of xf_model_info, XFSM and XFSD
LATENT_DIMS = (4, 8, 16, 32, 64, 128)


def row_bytes(K):
    """16 + 4K rounded up to 32: every row starts on a sector, v starts 16 bytes in."""
    return (16 + 4 * K + 31) // 32 * 32


def row_dtype(K):
    """{u64 key, f32 w, u32 0, f32 v[K], zero padding}"""
    pad = row_bytes(K) - 16 - 4 * K
    fields = [("key", "<u8"), ("w", "<f4"), ("zero", "<u4"), ("v", "<f4", (K,))]
    if pad:
        fields.append(("pad", "u1", (pad,)))
    dt = np.dtype(fields)
    assert dt.itemsize == row_bytes(K)
    return dt


def rows_array(keys, w, v):
    """Packed canonical rows sorted by key."""
    keys = np.asarray(keys, np.uint64)
    v = np.asarray(v, np.float32).reshape(keys.size, -1)
    order = np.argsort(keys, kind="stable")
    rows = np.zeros(keys.size, row_dtype(v.shape[1]))
    rows["key"] = keys[order]
    rows["w"] = np.asarray(w, np.float32)[order]
    rows["v"] = v[order]
    return rows


def padding_zero(rows):
    """Whether every padding byte of the rows (bytes 12 .. 15 and 16 + 4K .. row bytes) is zero."""
    ok = np.asarray(rows["zero"]) == 0
    if "pad" in rows.dtype.names:
        ok &= ~np.any(np.asarray(rows["pad"]) != 0, axis=1)
    return ok


def pruned(w, absent, v_ready, v):
    """Rows prune = 1 leaves out: w == 0 and, under DEFAULT, a latent block that is not materialised; under ZERO,
    every resolved v_k == 0 (v: the resolved latent rows, [n, K])."""
    zero_w = np.asarray(w, np.float32) == np.float32(0.0)  # +0 and -0
    if absent == SM.ABSENT_DEFAULT:
        return zero_w & ~np.asarray(v_ready, bool)
    return zero_w & np.all(np.asarray(v, np.float32) == 0, axis=1)


def fingerprint(rows):
    """The order-free fingerprint: n = row bytes / 8 words per row, the chain of delta_model.fingerprint."""
    return DM.fingerprint(rows)


def model_file(rows, K, optimizer, absent, v_init, v_const, seed, source_keys):
    """The bytes of a canonical XFSM file holding `rows` (rows_array)."""
    n = rows.size
    rb = row_bytes(K)
    chunk_rows = SM.CHUNK_BYTES // rb
    head = [b"XFSM", 1, SM.HEADER.size, n, SM.capacity_for(n), rb, FM_CANONICAL, K, optimizer, absent, v_init, v_const, 0,
            seed, source_keys, source_keys - n, chunk_rows, 0]
    head[-1] = SM.section_sum(SM.HEADER.pack(*head)[:96])
    out = [SM.HEADER.pack(*head)]
    for chunk, first in enumerate(range(0, n, chunk_rows)):
        body = rows[first:first + chunk_rows].tobytes()
        out.append(struct.pack("<QQQQ", first, len(body) // rb, SM.section_sum(body, chunk << 40), 0))
        out.append(body)
    return b"".join(out)


def parse_model_file(data):
    """(header dict, rows) of a canonical XFSM file; ValueError if it is not one or breaks the format."""
    if len(data) < SM.HEADER.size or data[:4] != b"XFSM":
        raise ValueError("not an XFSM file")
    h = dict(zip(SM.FIELDS, SM.HEADER.unpack(data[:SM.HEADER.size])))
    if h["header_checksum"] != SM.section_sum(data[:96]):
        raise ValueError("header checksum")
    K = h["latent_dim"]
    if h["fm"] != FM_CANONICAL or K not in LATENT_DIMS or h["row_bytes"] != row_bytes(K) or \
            h["chunk_rows"] != SM.CHUNK_BYTES // row_bytes(K) or h["capacity"] != SM.capacity_for(h["keys"]):
        raise ValueError("header fields")
    dt = row_dtype(K)
    parts, pos, first, chunk = [], SM.HEADER.size, 0, 0
    while first < h["keys"]:
        f0, n, s, z = struct.unpack("<QQQQ", data[pos:pos + 32]) if pos + 32 <= len(data) else (None,) * 4
        body = data[pos + 32:pos + 32 + (n or 0) * dt.itemsize]
        if f0 != first or z != 0 or not n or len(body) != n * dt.itemsize or s != SM.section_sum(body, chunk << 40):
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
    return h, rows


def delta_header(K, optimizer, absent, v_init, v_const, seed, base, result, result_source_keys, upserts, deletes):
    """The 144-byte XFSD header of a canonical delta, checksum included."""
    rb = row_bytes(K)
    head = [b"XFSD", 1, DM.HEADER.size, FM_CANONICAL, K, optimizer, absent, v_init, v_const, seed, rb, 0, base.size,
            fingerprint(base), result.size, result_source_keys, result_source_keys - result.size, fingerprint(result),
            upserts, deletes, SM.CHUNK_BYTES // rb, DM.CHUNK_KEYS, 0]
    head[-1] = SM.section_sum(DM.HEADER.pack(*head)[:136])
    return DM.HEADER.pack(*head)


def delta_file(a, b, b_source_keys, K, optimizer, absent, v_init, v_const, seed):
    """The XFSD file of the delta from canonical rows a to rows b."""
    up, de = DM.diff(a, b)
    de = np.ascontiguousarray(de, np.uint64)
    out = [delta_header(K, optimizer, absent, v_init, v_const, seed, a, b, b_source_keys, up.size, de.size)]
    chunk = 0
    for data, per, width in ((up, SM.CHUNK_BYTES // row_bytes(K), row_bytes(K)), (de, DM.CHUNK_KEYS, 8)):
        for first in range(0, data.size, per):
            body = np.ascontiguousarray(data[first:first + per]).tobytes()
            out.append(struct.pack("<QQQQ", first, len(body) // width, SM.section_sum(body, chunk << 40), 0))
            out.append(body)
            chunk += 1
    return b"".join(out)
