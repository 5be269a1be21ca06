"""Where the device table puts a key: the probe sequence of table.cuh (xf_probe_slot) and the bucket rule of
capi.cu (xf_table::alloc_table) restated in Python, and builders of keys whose placement is chosen exactly.

xf_probe_slot multiplies the key by an odd constant A mod 2^64, m = key * A; the home bucket is the top
(log2cap - bshift) bits of m and the walk through the home bucket starts at slot (m >> 9) & (2^bshift - 1).  A is
odd, so key = m * A^-1 mod 2^64 gives any m we choose:
  * top 40 bits of m all ones: the key homes in the LAST bucket at every capacity up to 2^40, so its chain wraps to
    slot 0, and keys built this way stay clustered through every growth;
  * top 40 bits zero: the key homes in bucket 0;
  * the same top bits and the same bits 9..12: every such key has the same probe sequence at every capacity and
    bucket size (bshift <= 4), so n of them form one chain n slots long.
The bits of m that no placement reads (0..8 and 13..23) number the keys, so the builders give up to 2^20 distinct
keys per (cluster, start slot)."""
import numpy as np

A = 0x9E3779B97F4A7C15      # xf_probe_slot's multiplier
A_INV = 0xF1DE83E19937733D  # its inverse mod 2^64
M64 = (1 << 64) - 1
EMPTY_KEY = M64             # XF_EMPTY_KEY: the empty-slot marker, reserved
TOP_ONES = ((1 << 40) - 1) << 24
FREE_BITS = 20              # bits 0..8 and 13..23 of m


def m_of(key):
    return (int(key) * A) & M64


def key_of(m):
    return (int(m) * A_INV) & M64


def probe_slot(key, i, log2cap, bshift):
    """xf_probe_slot: the slot of probe number i of `key` in a table of 2^log2cap slots and buckets of 2^bshift."""
    m = m_of(key)
    hb = m >> (64 - (log2cap - bshift))
    b1 = (1 << bshift) - 1
    j0 = (m >> 9) & b1
    k = i >> bshift
    j = ((j0 + i) & b1) if k == 0 else (i & b1)
    return (((hb + k) << bshift) | j) & ((1 << log2cap) - 1)


def home_slot(key, log2cap, bshift):
    return probe_slot(key, 0, log2cap, bshift)


def row_stride(K, opt_ftrl, canon=False):
    """xf_row_stride: bytes per row (K = 0: 32)."""
    if K <= 0:
        return 32
    acc = (32 + 4 * K + 15) & ~15
    ca = acc + 16 + (8 * K if opt_ftrl else 0)
    return (ca + (4 * K if canon else 0) + 31) & ~31


def bucket_log2(stride, log2cap, env=None):
    """alloc_table's bucket size: the rows that share one 128-byte line, XFLOW_BUCKET_LOG2 (`env`, clamped to 0..4)
    overriding, and plain linear probing (0) in tables of fewer than 16 buckets."""
    bs = 0
    while (stride << (bs + 1)) <= 128:
        bs += 1
    if env is not None and env != "":
        bs = min(max(int(env), 0), 4)
    if bs + 4 > log2cap:
        bs = 0
    return bs


def _m(top, n, j0s, start):
    j0s = tuple(j0s)
    out = []
    for c in range(start, start + n):
        assert c < (1 << FREE_BITS), "out of free bits"
        j0 = j0s[c % len(j0s)]
        assert 0 <= j0 < 16
        out.append(top | ((c >> 9) << 13) | (j0 << 9) | (c & 0x1FF))
    return out


def _keys(ms):
    keys = np.array([key_of(m) for m in ms], np.uint64)
    assert not (keys == np.uint64(EMPTY_KEY)).any()
    return keys


def tail(n, j0s=(0, 1, 2, 3), start=0):
    """n keys homed in the last bucket (their chains wrap to slot 0), start slots cycling through j0s.  Keys
    numbered from `start`, so disjoint ranges give disjoint keys."""
    return _keys(_m(TOP_ONES, n, j0s, start))


def head(n, j0s=(0, 1, 2, 3), start=0):
    """n keys homed in bucket 0."""
    return _keys(_m(0, n, j0s, start))


def one_chain(n, start=0):
    """n keys with one probe sequence (last bucket, start slot 0): the i-th key inserted sits at probe depth i."""
    return tail(n, (0,), start)


def twin_of_empty():
    """The key whose probe sequence is that of EMPTY_KEY (2^64 - 1) at every capacity and bucket size."""
    return np.uint64(key_of(m_of(EMPTY_KEY) ^ 1))
