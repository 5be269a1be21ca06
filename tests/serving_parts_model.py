"""A numpy statement of model parts (xf_table_freeze_part, csrc/serve.cu): the shard ranges, the XFSP file and the merge
of part files into the XFSM file of the whole model.  The GPU tests hold the library to it; test_serving_parts_model.py
checks it against hand cases."""
import struct

import numpy as np

import serving_model as M

PART_HEADER = struct.Struct("<4sIQQQIiiiiifIQQQQiiQ")  # the 112-byte XFSP header, fields in file order
PART_FIELDS = M.FIELDS[:-1] + ("shard_index", "num_shards", "header_checksum")
PART_OFFSETS = dict(M.OFFSETS, shard_index=96, num_shards=100, header_checksum=104)
COMPAT = ("fm", "latent_dim", "optimizer", "absent", "v_init", "v_const", "seed")  # what the parts of one model share
M64 = (1 << 64) - 1
assert PART_HEADER.size == 112


def shard_range(s, S):
    """Inclusive key range of shard s of S (xf_shard_of, postoffice.cc:134-143); the last shard runs to 2^64 - 2."""
    width = M64 // S
    return s * width, (M64 - 1 if s == S - 1 else (s + 1) * width - 1)


def shard_of(keys, S):
    """xf_shard_of over a key array"""
    keys = np.asarray(keys, np.uint64)
    return np.minimum(keys // np.uint64(M64 // S), np.uint64(S - 1)).astype(np.int64)


def build_part(rows, latent_dim, optimizer, absent, v_init, v_const, seed, source_keys, shard_index, num_shards):
    """The bytes of the XFSP file of shard shard_index of num_shards that holds `rows` (serving_model.rows_array)."""
    whole = M.build_file(rows, latent_dim, optimizer, absent, v_init, v_const, seed, source_keys)
    head = list(M.HEADER.unpack(whole[:M.HEADER.size]))[:-1]
    head[0], head[2] = b"XFSP", PART_HEADER.size
    head += [shard_index, num_shards, 0]
    head[-1] = M.section_sum(PART_HEADER.pack(*head)[:104])
    return PART_HEADER.pack(*head) + whole[M.HEADER.size:]


def parse_part(data):
    """(header dict, rows) of an XFSP file; ValueError for what xf_model_load refuses: another format, a damaged or
    truncated file, keys that do not ascend strictly, keys outside the shard's range, a shard that does not exist."""
    if len(data) < PART_HEADER.size or data[:4] != b"XFSP":
        raise ValueError("not an XFSP file")
    h = dict(zip(PART_FIELDS, PART_HEADER.unpack(data[:PART_HEADER.size])))
    if h["header_checksum"] != M.section_sum(data[:104]) or h["header_bytes"] != PART_HEADER.size:
        raise ValueError("header checksum")
    if not 0 <= h["shard_index"] < h["num_shards"]:
        raise ValueError("no such shard")
    # the rows as XFSM holds them: parse them behind a whole-model header that carries the same fields
    whole = list(M.HEADER.unpack(data[:M.HEADER.size]))
    whole[0], whole[2], whole[-1] = b"XFSM", M.HEADER.size, 0
    whole[-1] = M.section_sum(M.HEADER.pack(*whole)[:96])
    _, rows = M.parse_file(M.HEADER.pack(*whole) + data[PART_HEADER.size:])
    lo, hi = shard_range(h["shard_index"], h["num_shards"])
    if rows.size and (int(rows["key"][0]) < lo or int(rows["key"][-1]) > hi):
        raise ValueError("a key outside the shard")
    return h, rows


def merge(files):
    """The XFSM bytes of the whole model of XFSP files `files` (any order); ValueError for what xf_model_merge refuses."""
    parsed = [parse_part(f) for f in files]
    n = len(parsed)
    if n == 0 or any(h["num_shards"] != n for h, _ in parsed):
        raise ValueError("a merge takes every part of one split")
    if sorted(h["shard_index"] for h, _ in parsed) != list(range(n)):
        raise ValueError("a shard is repeated or missing")
    h0 = parsed[0][0]
    for h, _ in parsed:
        for f in COMPAT:
            if h[f] != h0[f]:
                raise ValueError("the parts differ in " + f)
    parsed.sort(key=lambda p: p[0]["shard_index"])
    # the ranges ascend with the shard: the rows of the parts in shard order are sorted by key
    rows = np.concatenate([r for _, r in parsed])
    return M.build_file(rows, h0["latent_dim"], h0["optimizer"], h0["absent"], h0["v_init"], h0["v_const"], h0["seed"],
                        sum(h["source_keys"] for h, _ in parsed))
