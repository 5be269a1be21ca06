"""numpy restatement of candidate ranking (xf_model_rank_candidates_*, include/xflow_b200.h): request q's candidate i
(local index) with score p_i has the key r_i = ord(p_i) << 32 | (2^32 - 1 - i), ord(NaN) = 0, ord(p) = bits(p) ^ 2^31
for a clear sign bit and ~bits(p) for a set one; larger keys rank first.  The top min(k, n_q) fill a request's k slots,
the rest hold index 0xFFFFFFFF and pctr bits 0x7FC00000."""
import numpy as np

PAD_INDEX = np.uint32(0xFFFFFFFF)
PAD_PCTR_BITS = np.uint32(0x7FC00000)


def rank_keys(p):
    """The keys of one request's scores (float32 [n])."""
    b = np.ascontiguousarray(p, np.float32).view(np.uint32).astype(np.uint64)
    nan = (b & 0x7FFFFFFF) > 0x7F800000
    o = np.where(b & 0x80000000, ~b & 0xFFFFFFFF, b ^ 0x80000000)
    o = np.where(nan, np.uint64(0), o)
    i = np.arange(b.size, dtype=np.uint64)
    return (o << np.uint64(32)) | (np.uint64(0xFFFFFFFF) - i)


def rank_model(pctr, cand_ptr, k):
    """(index uint32 [R, k], pctr float32 [R, k]) of every request of the batch, from its scores pctr [candidates]."""
    pctr = np.ascontiguousarray(pctr, np.float32)
    cand_ptr = np.asarray(cand_ptr, np.int64)
    R = cand_ptr.size - 1
    index = np.full((R, k), PAD_INDEX, np.uint32)
    bits = np.full((R, k), PAD_PCTR_BITS, np.uint32)
    for q in range(R):
        p = pctr[cand_ptr[q]:cand_ptr[q + 1]]
        top = np.argsort(rank_keys(p), kind="stable")[::-1][:k]  # the keys are distinct
        index[q, :top.size] = top
        bits[q, :top.size] = p.view(np.uint32)[top]
    return index, bits.view(np.float32)
