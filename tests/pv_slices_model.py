"""CPU statement of sliced progressive validation (include/xflow_b200.h section 8, xf_pv_set_slices): a row belongs to
slice s when at least one of its tokens has a key the map sends to s, once however many of its tokens do; each slice's
report is that of an unsliced pv (tests/validation_model.py) with the slice mantissa bits fed exactly its rows."""
import numpy as np

import validation_model as V


def slice_rows(row_ptr, keys, slice_map, num_slices):
    """For each slice, the ascending indices of the rows in it.  slice_map: {key: slice}."""
    row_ptr = np.asarray(row_ptr, np.int64)
    keys = np.asarray(keys, np.uint64)
    members = [[] for _ in range(num_slices)]
    for r in range(row_ptr.size - 1):
        named = {slice_map[k] for k in keys[row_ptr[r]:row_ptr[r + 1]].tolist() if k in slice_map}
        for s in named:
            members[s].append(r)
    return [np.asarray(m, np.int64) for m in members]


def slice_reports(pctr, labels, weights, row_ptr, keys, slice_map, num_slices, ms):
    """Each slice's report: V.Pv(ms) fed the slice's rows."""
    pctr = np.asarray(pctr, np.float32)
    labels = np.asarray(labels)
    weights = np.ones(pctr.size, np.float32) if weights is None else np.asarray(weights, np.float32)
    return [V.Pv(ms).add(pctr[rows], labels[rows], weights[rows]).report()
            for rows in slice_rows(row_ptr, keys, slice_map, num_slices)]
