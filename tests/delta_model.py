"""A numpy statement of serving model deltas (csrc/delta.cu): the fingerprint, diff, apply, and the XFSD file.  Rows are
serving_model.rows_array arrays (sorted by key).  The GPU tests hold the library to it and build damaged and malformed
files with it; test_delta_model.py checks it on random row sets."""
import struct

import numpy as np

import serving_model as SM

HEADER = struct.Struct("<4sIQiiiiifQIIQQQQQQQQQQQ")  # the 144-byte header, fields in file order
FIELDS = ("magic", "version", "header_bytes", "fm", "latent_dim", "optimizer", "absent", "v_init", "v_const", "seed",
          "row_bytes", "zero", "base_keys", "base_fingerprint", "result_keys", "source_keys", "pruned_keys",
          "result_fingerprint", "upserts", "deletes", "chunk_rows", "chunk_keys", "header_checksum")
OFFSETS = dict(magic=0, version=4, header_bytes=8, fm=16, latent_dim=20, optimizer=24, absent=28, v_init=32, v_const=36,
               seed=40, row_bytes=48, zero=52, base_keys=56, base_fingerprint=64, result_keys=72, source_keys=80,
               pruned_keys=88, result_fingerprint=96, upserts=104, deletes=112, chunk_rows=120, chunk_keys=128,
               header_checksum=136)
assert HEADER.size == 144
CHUNK_KEYS = SM.CHUNK_BYTES // 8
EMPTY = np.uint64(2 ** 64 - 1)


def fingerprint(rows):
    """Sum mod 2^64 over the rows of h_n, h_0 = 0, h_{i+1} = splitmix64(h_i ^ w_i) over the row's 8-byte words."""
    if rows.size == 0:
        return 0
    words = np.ascontiguousarray(rows).view("<u8").reshape(rows.size, -1)
    h = np.zeros(rows.size, np.uint64)
    for i in range(words.shape[1]):
        h = SM.splitmix64(h ^ words[:, i])
    with np.errstate(over="ignore"):
        return int(np.sum(h, dtype=np.uint64))


def _raw(rows):
    """each row's bytes as one comparable value"""
    return np.ascontiguousarray(rows).view("V%d" % rows.dtype.itemsize).ravel()


def diff(a, b):
    """(upserts, deletes) from rows a to rows b: b's rows whose key a lacks or whose bytes differ, and a's keys b lacks."""
    ia = np.searchsorted(a["key"], b["key"])
    ia_c = np.minimum(ia, max(a.size - 1, 0))
    found = (ia < a.size) & (a["key"][ia_c] == b["key"]) if a.size else np.zeros(b.size, bool)
    same = np.zeros(b.size, bool)
    if a.size:
        same[found] = _raw(a[ia_c[found]]) == _raw(b[found])
    upserts = b[~same]
    deletes = a["key"][~np.isin(a["key"], b["key"])]
    return upserts, deletes


def apply(a, upserts, deletes):
    """rows a with the deletes removed and the upserts set, sorted by key"""
    keep = ~np.isin(a["key"], deletes) & ~np.isin(a["key"], upserts["key"])
    out = np.concatenate([a[keep], upserts])
    return out[np.argsort(out["key"], kind="stable")]


def build_file(upserts, deletes, latent_dim, optimizer, absent, v_init, v_const, seed, base_keys, base_fingerprint,
               result_keys, source_keys, result_fingerprint):
    """The bytes of an XFSD file holding `upserts` (rows) and `deletes` (keys) as given: nothing is sorted or checked,
    so that malformed contents with valid checksums can be built."""
    fm = 1 if latent_dim > 0 else 0
    row_bytes = 32 if fm else 16
    deletes = np.ascontiguousarray(deletes, np.uint64)
    chunk_rows = SM.CHUNK_BYTES // row_bytes
    head = [b"XFSD", 1, HEADER.size, fm, latent_dim, optimizer, absent, v_init, v_const, seed, row_bytes, 0, base_keys,
            base_fingerprint, result_keys, source_keys, source_keys - result_keys, result_fingerprint, upserts.size,
            deletes.size, chunk_rows, CHUNK_KEYS, 0]
    head[-1] = SM.section_sum(HEADER.pack(*head)[:136])
    out = [HEADER.pack(*head)]
    chunk = 0
    for data, per, width in ((upserts, chunk_rows, row_bytes), (deletes, CHUNK_KEYS, 8)):
        for first in range(0, data.size, per):
            body = np.ascontiguousarray(data[first:first + per]).tobytes()
            out.append(struct.pack("<QQQQ", first, len(body) // width, SM.section_sum(body, chunk << 40), 0))
            out.append(body)
            chunk += 1
    return b"".join(out)


def delta_file(a, b, b_source_keys, latent_dim, optimizer, absent, v_init, v_const, seed):
    """The XFSD file of the delta from rows a to rows b (b frozen from a table of b_source_keys keys)."""
    up, de = diff(a, b)
    return build_file(up, de, latent_dim, optimizer, absent, v_init, v_const, seed, a.size, fingerprint(a), b.size,
                      b_source_keys, fingerprint(b))


def parse_file(data):
    """(header dict, upserts, deletes) of an XFSD file; ValueError if it is not one, is truncated, a checksum fails or
    its contents break the format."""
    if len(data) < HEADER.size or data[:4] != b"XFSD":
        raise ValueError("not an XFSD file")
    h = dict(zip(FIELDS, HEADER.unpack(data[:HEADER.size])))
    if h["header_checksum"] != SM.section_sum(data[:136]):
        raise ValueError("header checksum")
    dt = SM.FM_ROW if h["fm"] else SM.LR_ROW
    if h["row_bytes"] != dt.itemsize or h["chunk_rows"] != SM.CHUNK_BYTES // dt.itemsize or h["chunk_keys"] != CHUNK_KEYS:
        raise ValueError("header fields")
    if h["source_keys"] - h["result_keys"] != h["pruned_keys"]:
        raise ValueError("header counts")
    pos, chunk, sections = HEADER.size, 0, []
    for n, per, d in ((h["upserts"], h["chunk_rows"], dt), (h["deletes"], CHUNK_KEYS, np.dtype("<u8"))):
        parts, first = [], 0
        while first < n:
            if pos + 32 > len(data):
                raise ValueError("truncated")
            f0, c, s, z = struct.unpack("<QQQQ", data[pos:pos + 32])
            body = data[pos + 32:pos + 32 + c * d.itemsize]
            if f0 != first or z != 0 or c != min(per, n - first) or len(body) != c * d.itemsize or \
                    s != SM.section_sum(body, chunk << 40):
                raise ValueError("chunk %d" % chunk)
            parts.append(np.frombuffer(body, d))
            pos += 32 + len(body)
            first += c
            chunk += 1
        sections.append(np.concatenate(parts) if parts else np.zeros(0, d))
    if pos != len(data):
        raise ValueError("trailing bytes")
    up, de = sections
    for keys in (up["key"], de):
        if keys.size and (np.any(keys[1:] <= keys[:-1]) or np.any(keys == EMPTY)):
            raise ValueError("keys not strictly ascending below 2^64 - 1")
    if up.size and np.any(np.ascontiguousarray(up["pad"]) != 0):
        raise ValueError("non-zero padding")
    if np.isin(de, up["key"]).any():
        raise ValueError("a key both upserted and deleted")
    return h, up, de
