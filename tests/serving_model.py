"""A numpy statement of the serving model (csrc/serve.cu): what a frozen FM row holds, which rows a freeze prunes, and
the XFSM file.  The GPU tests hold the library to it; test_serving_model.py checks it against hand cases."""
import struct

import numpy as np

ABSENT_DEFAULT, ABSENT_ZERO = 0, 1
HEADER = struct.Struct("<4sIQQQIiiiiifIQQQQQ")  # the 104-byte header, fields in file order
FIELDS = ("magic", "version", "header_bytes", "keys", "capacity", "row_bytes", "fm", "latent_dim", "optimizer", "absent",
          "v_init", "v_const", "zero", "seed", "source_keys", "pruned_keys", "chunk_rows", "header_checksum")
OFFSETS = dict(magic=0, version=4, header_bytes=8, keys=16, capacity=24, row_bytes=32, fm=36, latent_dim=40, optimizer=44,
               absent=48, v_init=52, v_const=56, zero=60, seed=64, source_keys=72, pruned_keys=80, chunk_rows=88,
               header_checksum=96)
CHUNK_BYTES = 64 << 20
LR_ROW = np.dtype([("key", "<u8"), ("w", "<f4"), ("pad", "<u4")])
FM_ROW = np.dtype([("key", "<u8"), ("w", "<f4"), ("st", "<f4"), ("qt", "<f4"), ("pad", "<u4", (3,))])
assert HEADER.size == 104 and LR_ROW.itemsize == 16 and FM_ROW.itemsize == 32


def fm_sums(v):
    """(st, qt) of latent rows v[n, K] in float32, in the kernels' association: k ascending, st += v_k and
    qt = qt + (v_k * v_k), every operation rounded to float32."""
    v = np.asarray(v, np.float32)
    if v.ndim == 1:
        v = v[None, :]
    st = np.zeros(v.shape[0], np.float32)
    qt = np.zeros(v.shape[0], np.float32)
    for k in range(v.shape[1]):
        st = (st + v[:, k]).astype(np.float32)
        qt = (qt + (v[:, k] * v[:, k]).astype(np.float32)).astype(np.float32)
    return st, qt


def pruned(w, fm, absent, v_ready=None, st=None, qt=None):
    """Which rows a freeze with prune = 1 leaves out: those that read exactly as an absent key does."""
    w = np.asarray(w, np.float32)
    zero_w = w == np.float32(0.0)  # +0 and -0
    if not fm:
        return zero_w
    if absent == ABSENT_DEFAULT:
        return zero_w & ~np.asarray(v_ready, bool)
    return zero_w & (np.asarray(st, np.float32) == 0) & (np.asarray(qt, np.float32) == 0)


def capacity_for(keys):
    c = 1024
    while c < 2 * keys:
        c *= 2
    return c


_M = (1 << 64) - 1


def splitmix64(x):
    x = np.asarray(x, np.uint64)
    with np.errstate(over="ignore"):
        x = x + np.uint64(0x9E3779B97F4A7C15)
        x = (x ^ (x >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        x = (x ^ (x >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return x ^ (x >> np.uint64(31))


def section_sum(data, off0=0):
    """Sum mod 2^64 of splitmix64(word ^ offset) over the 8-byte words of `data`, the first word at offset off0."""
    words = np.frombuffer(bytes(data), "<u8")
    offs = np.uint64(off0) + np.arange(words.size, dtype=np.uint64) * np.uint64(8)
    with np.errstate(over="ignore"):
        return int(np.sum(splitmix64(words ^ offs), dtype=np.uint64))


def rows_array(keys, w, st=None, qt=None):
    """Packed rows sorted by key: LR when st is None."""
    keys = np.asarray(keys, np.uint64)
    order = np.argsort(keys, kind="stable")
    rows = np.zeros(keys.size, LR_ROW if st is None else FM_ROW)
    rows["key"] = keys[order]
    rows["w"] = np.asarray(w, np.float32)[order]
    if st is not None:
        rows["st"] = np.asarray(st, np.float32)[order]
        rows["qt"] = np.asarray(qt, np.float32)[order]
    return rows


def build_file(rows, latent_dim, optimizer, absent, v_init, v_const, seed, source_keys):
    """The bytes of an XFSM file that holds `rows` (rows_array)."""
    fm = 1 if latent_dim > 0 else 0
    row_bytes = rows.dtype.itemsize
    n = rows.size
    chunk_rows = CHUNK_BYTES // row_bytes
    head = [b"XFSM", 1, HEADER.size, n, capacity_for(n), row_bytes, fm, latent_dim, optimizer, absent, v_init, v_const, 0,
            seed, source_keys, source_keys - n, chunk_rows, 0]
    head[-1] = section_sum(HEADER.pack(*head)[:96])
    out = [HEADER.pack(*head)]
    for chunk, first in enumerate(range(0, n, chunk_rows)):
        body = rows[first:first + chunk_rows].tobytes()
        out.append(struct.pack("<QQQQ", first, len(body) // row_bytes, section_sum(body, chunk << 40), 0))
        out.append(body)
    return b"".join(out)


def parse_file(data):
    """(header dict, rows) of an XFSM file; ValueError if it is not one, is truncated, a checksum fails, or a row's
    padding is not zero."""
    if len(data) < HEADER.size or data[:4] != b"XFSM":
        raise ValueError("not an XFSM file")
    h = dict(zip(FIELDS, HEADER.unpack(data[:HEADER.size])))
    if h["header_checksum"] != section_sum(data[:96]):
        raise ValueError("header checksum")
    dt = FM_ROW if h["fm"] else LR_ROW
    if h["row_bytes"] != dt.itemsize or h["capacity"] != capacity_for(h["keys"]):
        raise ValueError("header fields")
    parts, pos, first, chunk = [], HEADER.size, 0, 0
    while first < h["keys"]:
        if pos + 32 > len(data):
            raise ValueError("truncated")
        f0, n, s, z = struct.unpack("<QQQQ", data[pos:pos + 32])
        body = data[pos + 32:pos + 32 + n * dt.itemsize]
        if f0 != first or z != 0 or n == 0 or len(body) != n * dt.itemsize or s != section_sum(body, chunk << 40):
            raise ValueError("chunk %d" % chunk)
        parts.append(np.frombuffer(body, dt))
        pos += 32 + len(body)
        first += n
        chunk += 1
    if pos != len(data):
        raise ValueError("trailing bytes")
    rows = np.concatenate(parts) if parts else np.zeros(0, dt)
    if np.any(np.diff(rows["key"].astype(object)) <= 0):
        raise ValueError("keys not ascending")
    if rows.size and np.any(np.ascontiguousarray(rows["pad"]) != 0):
        raise ValueError("non-zero padding")
    return h, rows
