"""Ranking quality at a cutoff on the device (pytest -m gpu): xf_group_metric_topk and _groups_topk against the CPU
statement tests/group_topk_model.py byte for byte, under permutation, re-cutting and two streams, beside the finish
it evaluates, on a frozen model's ranked candidates, and through its refusals."""
import math

import numpy as np
import pytest

import group_topk_model as T
from test_gpu_group_metric import Rows, _case
from xflow_b200 import api

pytestmark = pytest.mark.gpu

ERR_ARG, ERR_STATE = "error -1:", "error -6:"
KS = (1, 10, 1000, 65536)
FIELDS = ("ndcg", "precision", "recall")


def _torch():
    import torch
    return torch


def _same(a, b):
    """Equal bytes, NaN included (any NaN matches any NaN)."""
    a, b = np.ascontiguousarray(a, np.float64), np.ascontiguousarray(b, np.float64)
    if a.shape != b.shape or not np.array_equal(np.isnan(a), np.isnan(b)):
        return False
    keep = ~np.isnan(a)
    return a[keep].tobytes() == b[keep].tobytes()


def _check(got, groups, want, wgroups):
    for key in ("k", "groups", "scored_groups", "scored_rows"):
        assert got[key] == want[key], (key, got[key], want[key])
    for key in FIELDS:
        for name in (key, key + "_mean"):
            assert _same([got[name]], [want[name]]), (name, got[name], want[name])
        assert _same(groups[key], wgroups[key]), key


@pytest.mark.parametrize("name", ["ties16", "zipf", "one_group", "one_row_groups"])
def test_matches_the_model(name):
    p, y, g = _case(name, 7)
    r = Rows(p, y, g)
    m = api.GroupMetric()
    r.add(m)
    fin = m.finish()
    for k in KS:
        want, wgroups = T.evaluate(p, y, g, k)
        got = m.topk(k)
        _check(got, m.groups_topk(), want, wgroups)
        assert got["groups"] == fin["groups"] and got["scored_groups"] == fin["scored_groups"]
        assert got["scored_rows"] == fin["scored_rows"]
    if name == "one_group":   # runs of about 100 rows: some straddle k
        assert T.runs(p, y, g)[5].max() > 50
    if name == "one_row_groups":
        assert math.isnan(got["ndcg"]) and got["scored_groups"] == 0
    m.close()


def test_permutation_cuts_and_streams_give_the_same_bytes():
    torch = _torch()
    p, y, g = _case("ties16", 5)
    one = api.GroupMetric()
    Rows(p, y, g).add(one)
    one.finish()
    raw = {k: one.topk_bytes(k) for k in (3, 1000)}
    groups = one.groups_topk()                      # of k = 1000
    perm = np.random.default_rng(6).permutation(p.size)
    r = Rows(p[perm], y[perm], g[perm])
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    cuts = [0, 1, 999, 50_000, 50_001, 120_000, p.size]
    two = api.GroupMetric()
    for i, (a, b) in enumerate(zip(cuts, cuts[1:])):
        r.add(two, a, b, stream=(s1 if i % 2 else s2).cuda_stream)
    two.finish()
    assert two.topk_bytes(3) == raw[3] and two.topk_bytes(1000) == raw[1000]
    got = two.groups_topk()
    for key in FIELDS:
        assert groups[key].tobytes() == got[key].tobytes(), key
    one.close()
    two.close()


def test_topk_changes_neither_groups_nor_finish():
    p, y, g = _case("zipf", 3)
    m = api.GroupMetric()
    Rows(p, y, g).add(m)
    raw = m.finish_bytes()
    before = m.groups()
    a = m.topk_bytes(10)
    after = m.groups()
    for key in before:
        assert before[key].tobytes() == after[key].tobytes(), key
    assert m.topk_bytes(65536) != a and m.topk_bytes(10) == a   # a second topk replaces the first
    assert m.finish_bytes() == raw
    for key, v in m.groups().items():
        assert v.tobytes() == before[key].tobytes(), key
    m.close()


def test_precision_of_ranked_candidates():
    """A frozen FM model scores the candidates of 2000 requests.  Where a request's scores are distinct,
    precision_g * min(k, n_g) is the number of positives among rank_candidates' top k for that request."""
    rng = np.random.default_rng(9)
    K, space = 8, 4000
    keys = api.hash_decimal_ids(np.arange(space, dtype=np.uint64))
    t = api.Table(latent_dim=K, optimizer=api.OPT_FTRL, seed=3, capacity=1 << 14)
    t.import_(keys, w=rng.normal(0, 0.5, space).astype(np.float32),
              v=rng.normal(0, 0.3, (space, K)).astype(np.float32))
    model = t.freeze()
    R = 2000
    counts = rng.integers(1, 60, R)
    ctx_ptr = np.r_[0, np.cumsum(np.full(R, 3))].astype(np.uint32)
    ctx_keys = keys[rng.integers(0, space, int(ctx_ptr[-1]))]
    cand_ptr = np.r_[0, np.cumsum(counts)].astype(np.uint32)
    C = int(cand_ptr[-1])
    row_ptr = np.r_[0, np.cumsum(rng.integers(1, 4, C))].astype(np.uint32)
    cand_keys = keys[rng.integers(0, space, int(row_ptr[-1]))]
    scores = model.predict_candidates(ctx_ptr, ctx_keys, cand_ptr, row_ptr, cand_keys)
    labels = (rng.random(C) < 0.25).astype(np.uint8)
    request = np.repeat(np.arange(R, dtype=np.uint64), counts)
    m = api.GroupMetric()
    Rows(scores, labels, request).add(m)
    m.finish()
    ids = m.groups()["ids"]
    assert np.array_equal(ids, np.arange(R, dtype=np.uint64))
    checked = 0
    for k in (1, 5, 20):
        index, _ = model.rank_candidates(ctx_ptr, ctx_keys, cand_ptr, row_ptr, cand_keys, k)
        m.topk(k)
        prec = m.groups_topk()["precision"]
        for q in range(R):
            s = scores[cand_ptr[q]:cand_ptr[q + 1]]
            lab = labels[cand_ptr[q]:cand_ptr[q + 1]]
            if np.unique(s).size < s.size or not lab.any():
                continue
            top = index[q][index[q] != 0xFFFFFFFF]
            hits = int((lab[top] != 0).sum())
            assert _same([prec[q]], [hits / min(k, s.size)]), (k, q)
            checked += 1
    assert checked > R
    m.close()
    model.close()
    t.close()


def test_refusals_and_the_empty_metric():
    L = api.lib()
    p, y, g = _case("small", 4)
    r = Rows(p, y, g)
    m = api.GroupMetric()
    with pytest.raises(api.XflowError, match=ERR_STATE):   # before any finish
        m.topk(10)
    empty = m.finish()
    e = m.topk(10)
    assert e["groups"] == e["scored_groups"] == e["scored_rows"] == 0 and e["k"] == 10
    assert all(math.isnan(e[key]) for key in ("ndcg", "ndcg_mean", "precision", "precision_mean", "recall",
                                              "recall_mean"))
    assert m.groups_topk(0)["ndcg"].size == 0 and empty["groups"] == 0
    r.add(m)
    with pytest.raises(api.XflowError, match=ERR_STATE):   # after an add
        m.topk(10)
    raw = m.finish_bytes()
    G_ = m.last_groups
    with pytest.raises(api.XflowError, match=ERR_STATE):   # groups_topk before a topk
        m.groups_topk()
    top = m.topk_bytes(10)
    want = m.groups_topk()
    for k in (0, 65537):
        with pytest.raises(api.XflowError, match=ERR_ARG + ".*k = %d" % k):
            m.topk(k)
    with pytest.raises(api.XflowError, match=ERR_ARG):
        m.groups_topk(G_ + 1)
    assert L.xf_group_metric_groups_topk(m.h, G_, None, None, None) == 0
    got = m.groups_topk()                                  # the refusals left the last topk in place
    for key in FIELDS:
        assert got[key].tobytes() == want[key].tobytes(), key
    assert m.finish_bytes() == raw and m.topk_bytes(10) == top
    m.finish()                                             # a finish ends the last topk's values
    with pytest.raises(api.XflowError, match=ERR_STATE):
        m.groups_topk()
    m.reset()
    with pytest.raises(api.XflowError, match=ERR_STATE):   # after a reset
        m.topk(10)
    with pytest.raises(api.XflowError, match=ERR_STATE):
        m.groups_topk()
    r.add(m)
    assert m.finish_bytes() == raw and m.topk_bytes(10) == top
    m.close()


def test_discounts_are_the_50_digit_table():
    assert np.array_equal(api.group_discounts(), T.discounts())
