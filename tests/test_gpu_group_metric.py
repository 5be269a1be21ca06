"""The grouped test metric on the device (pytest -m gpu): xf_group_metric_* against the CPU statement
tests/group_metric_model.py, against xf_metric and the progressive validation on the same rows, under permutation,
re-cutting and two streams, on a frozen model's candidate scores, and through its lifecycle and refusals."""
import math

import numpy as np
import pytest

import group_metric_model as G
from xflow_b200 import api

pytestmark = pytest.mark.gpu

ERR_ARG, ERR_STATE = "error -1:", "error -6:"
TOP = np.uint64(2 ** 64 - 1)
SPECIAL = np.array([np.nan, np.inf, -np.inf, -0.0, 0.0, 1.0, 1e-30, 0.5], np.float32)


def _torch():
    import torch
    return torch


def _dev(a):
    return _torch().from_numpy(np.ascontiguousarray(a).view(np.uint8)).cuda()


class Rows:
    """(p, y, g) on the host and the device."""

    def __init__(self, p, y, g):
        self.p = np.ascontiguousarray(p, np.float32)
        self.y = np.ascontiguousarray(y, np.uint8)
        self.g = np.ascontiguousarray(g, np.uint64)
        self.d = [_dev(self.p), _dev(self.y), _dev(self.g)]
        _torch().cuda.synchronize()
        self.n = self.p.size

    def add(self, m, a=0, b=None, stream=0):
        b = self.n if b is None else b
        m.add_device(self.d[0].data_ptr() + 4 * a, self.d[1].data_ptr() + a, self.d[2].data_ptr() + 8 * a, b - a,
                     stream=stream)


def _case(name, seed):
    rng = np.random.default_rng(seed)
    if name == "ties16":  # 16 prediction levels, specials, labels 2 and 255, one-row / one-class groups, extreme ids
        n = 200_000
        p = np.linspace(0.05, 0.95, 16).astype(np.float32)[rng.integers(0, 16, n)]
        g = rng.integers(0, 20_000, n).astype(np.uint64) * np.uint64(0x9E3779B97F4A7C15)
        y = rng.choice(np.array([0, 1, 2, 255], np.uint8), n, p=[0.6, 0.3, 0.05, 0.05])
        pick = rng.random(n) < 0.02
        p[pick] = SPECIAL[rng.integers(0, SPECIAL.size, int(pick.sum()))]
        g[:40], g[40:80] = np.uint64(0), TOP
        g[80:200] = np.uint64(12345)
        y[80:200] = 0                                   # an all-negative group
        g[200:300] = np.uint64(67890)
        y[200:300] = 2                                  # an all-positive group
        p[300:310] = np.nan
        g[300:310] = np.uint64(555)                     # a group of NaN rows only does not exist
        g[310:1310] = np.arange(10 ** 12, 10 ** 12 + 1000, dtype=np.uint64)  # one-row groups
    elif name == "small":
        n = 10_000
        p = rng.random(n).astype(np.float32)
        g = rng.integers(0, 300, n).astype(np.uint64)
        y = (rng.random(n) < 0.3 + 0.4 * p).astype(np.uint8)
    elif name == "zipf":
        n = 1_000_000
        g = (rng.zipf(1.3, n) % (1 << 40)).astype(np.uint64)
        p = rng.random(n).astype(np.float32)
        y = (rng.random(n) < p).astype(np.uint8)
    elif name == "one_group":
        n = 1_000_000
        g = np.full(n, TOP, np.uint64)
        p = np.round(rng.random(n), 4).astype(np.float32)
        y = (rng.random(n) < p).astype(np.uint8)
    elif name == "one_row_groups":
        n = 1_000_000
        g = np.arange(n, dtype=np.uint64) * np.uint64(0x9E3779B97F4A7C15)  # distinct, 0 among them
        g[1] = TOP
        assert np.unique(g).size == n
        g = rng.permutation(g)
        p = rng.random(n).astype(np.float32)
        y = (rng.random(n) < 0.5).astype(np.uint8)
    elif name == "large":
        n = 5_000_000
        g = rng.integers(0, 100_000, n).astype(np.uint64)
        p = rng.random(n).astype(np.float32)
        p[rng.random(n) < 0.001] = -0.0
        y = (rng.random(n) < p).astype(np.uint8)
    return p, y, g


def _bits(a):
    return np.ascontiguousarray(a, np.float64).tobytes()


def _check_against_model(got, groups, want, wgroups):
    for k in ("rows", "positives", "negatives", "nan_rows", "groups", "scored_groups", "scored_rows"):
        assert got[k] == want[k], (k, got[k], want[k])
    for k in ("gauc", "gauc_mean"):
        assert _bits([got[k]]) == _bits([want[k]]) or (math.isnan(got[k]) and math.isnan(want[k])), (k, got[k], want[k])
    if want["rows"]:
        assert abs(got["logloss"] - want["logloss"]) <= 1e-12 * abs(want["logloss"])
    for k in ("ids", "rows", "positives"):
        assert np.array_equal(groups[k], wgroups[k]), k
    assert np.array_equal(groups["auc"], wgroups["auc"], equal_nan=True)
    assert np.all(np.abs(groups["logloss"] - wgroups["logloss"]) <= 1e-12 * np.abs(wgroups["logloss"]))


@pytest.mark.parametrize("name", ["small", "ties16", "zipf", "one_group", "one_row_groups", "large"])
def test_matches_the_model(name):
    p, y, g = _case(name, 7)
    want, wgroups = G.evaluate(p, y, g)
    r = Rows(p, y, g)
    m = api.GroupMetric()
    r.add(m)
    got = m.finish()
    groups = m.groups()
    _check_against_model(got, groups, want, wgroups)
    if name == "ties16":
        assert got["nan_rows"] > 10 and 555 not in groups["ids"].tolist()
        assert groups["ids"][0] == 0 and groups["ids"][-1] == TOP
        assert got["scored_groups"] < got["groups"]
    if name == "one_group":
        assert got["groups"] == 1
    if name == "one_row_groups":
        assert got["groups"] == p.size and got["scored_groups"] == 0 and math.isnan(got["gauc"])
    m.close()


def test_one_group_is_xf_metric_and_the_logloss_is_the_pvs():
    rng = np.random.default_rng(3)
    n = 300_000
    p = np.round(rng.random(n), 3).astype(np.float32)
    y = (rng.random(n) < p).astype(np.uint8)
    r = Rows(p, y, np.full(n, 42, np.uint64))
    m = api.GroupMetric()
    r.add(m)
    got = m.finish()
    out = (api.C.c_double * 6)()
    rc = api.lib().xf_auc_logloss_device(api.C.c_void_p(r.d[0].data_ptr()), api.C.c_void_p(r.d[1].data_ptr()), n, 0,
                                         None, out)
    assert rc == 0
    assert _bits(m.groups()["auc"]) == _bits([out[5]])
    # the logloss of an unweighted pv fed the same rows, byte for byte (NaN, +-Inf and -0 rows included)
    p2, y2, g2 = _case("ties16", 11)
    for rows in (r, Rows(p2, y2, g2)):
        pv = api.ProgressiveValidation()
        pv.add_device(rows.d[0].data_ptr(), rows.d[1].data_ptr(), rows.n)
        m.reset()
        rows.add(m)
        assert _bits([m.finish()["logloss"]]) == _bits([pv.report()["logloss"]])
        pv.close()
    m.close()


def test_permutation_cuts_and_streams_give_the_same_bytes():
    torch = _torch()
    p, y, g = _case("ties16", 5)
    one = api.GroupMetric()
    Rows(p, y, g).add(one)
    raw, groups = one.finish_bytes(), one.groups()
    perm = np.random.default_rng(6).permutation(p.size)
    r = Rows(p[perm], y[perm], g[perm])
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    cuts = [0, 1, 999, 50_000, 50_001, 120_000, p.size]
    two = api.GroupMetric()
    for k, (a, b) in enumerate(zip(cuts, cuts[1:])):  # the adds grow the buffers while the other stream copies
        r.add(two, a, b, stream=(s1 if k % 2 else s2).cuda_stream)
    assert two.finish_bytes() == raw
    got = two.groups()
    for k in groups:
        assert groups[k].tobytes() == got[k].tobytes(), k
    assert two.finish_bytes() == raw   # finish does not reset
    one.close()
    two.close()


def test_per_request_auc_of_candidate_scores():
    """A frozen FM model scores the candidates of 3000 requests; with the request index as the group, every request's
    AUC is the model's."""
    rng = np.random.default_rng(9)
    K, space = 8, 4000
    keys = api.hash_decimal_ids(np.arange(space, dtype=np.uint64))
    t = api.Table(latent_dim=K, optimizer=api.OPT_FTRL, seed=3, capacity=1 << 14)
    t.import_(keys, w=rng.normal(0, 0.5, space).astype(np.float32),
              v=rng.normal(0, 0.3, (space, K)).astype(np.float32))
    model = t.freeze()
    R = 3000
    counts = rng.integers(1, 40, R)
    ctx_ptr = np.r_[0, np.cumsum(np.full(R, 3))].astype(np.uint32)
    ctx_keys = keys[rng.integers(0, space, int(ctx_ptr[-1]))]
    cand_ptr = np.r_[0, np.cumsum(counts)].astype(np.uint32)
    C = int(cand_ptr[-1])
    row_ptr = np.r_[0, np.cumsum(rng.integers(1, 4, C))].astype(np.uint32)
    cand_keys = keys[rng.integers(0, space, int(row_ptr[-1]))]
    scores = model.predict_candidates(ctx_ptr, ctx_keys, cand_ptr, row_ptr, cand_keys)
    labels = (rng.random(C) < 0.25).astype(np.uint8)
    request = np.repeat(np.arange(R, dtype=np.uint64), counts)
    want, wgroups = G.evaluate(scores, labels, request)
    m = api.GroupMetric()
    Rows(scores, labels, request).add(m)
    got = m.finish()
    groups = m.groups()
    _check_against_model(got, groups, want, wgroups)
    assert got["groups"] == R and got["scored_groups"] > R // 2
    m.close()
    model.close()
    t.close()


def test_lifecycle_and_refusals():
    torch = _torch()
    L = api.lib()
    p, y, g = _case("small", 4)
    r = Rows(p, y, g)
    m = api.GroupMetric()
    empty = m.finish()
    assert empty["rows"] == empty["groups"] == empty["nan_rows"] == 0
    assert all(math.isnan(empty[k]) for k in ("logloss", "gauc", "gauc_mean"))
    assert m.groups(0)["ids"].size == 0
    r.add(m)
    raw = m.finish_bytes()
    G_ = m.last_groups
    with pytest.raises(api.XflowError, match=ERR_ARG):
        m.groups(G_ + 1)
    # NULL arrays are allowed in groups()
    assert L.xf_group_metric_groups(m.h, G_, None, None, None, None, None) == 0
    # refusals leave the metric as it was
    dp = api.C.c_void_p(r.d[0].data_ptr())
    dy = api.C.c_void_p(r.d[1].data_ptr())
    dg = api.C.c_void_p(r.d[2].data_ptr())
    for args in ((None, dy, dg), (dp, None, dg), (dp, dy, None)):
        assert L.xf_group_metric_add_device(m.h, *args, 10, None) == -1
        assert b"NULL" in L.xf_last_error()
    assert L.xf_group_metric_add_device(m.h, dp, dy, dg, (1 << 31) - r.n, None) == -1
    err = L.xf_last_error().decode()
    assert "2^31" in err and str(r.n) in err and str((1 << 31) - r.n) in err
    assert L.xf_group_metric_add_device(m.h, dp, dy, dg, 1 << 40, None) == -1
    assert L.xf_group_metric_add_device(m.h, None, None, None, 0, None) == 0
    assert m.groups()["ids"].size == G_   # no add came after the finish
    assert m.finish_bytes() == raw
    # an add after a finish makes groups() refuse until the next finish
    r.add(m, 0, 10)
    with pytest.raises(api.XflowError, match=ERR_STATE):
        m.groups(G_)
    # reset clears everything; finish on the empty metric gives NaN ratios
    m.reset()
    with pytest.raises(api.XflowError, match=ERR_STATE):
        m.groups(G_)
    e2 = m.finish()
    assert e2["rows"] == 0 and e2["groups"] == 0 and math.isnan(e2["gauc"]) and math.isnan(e2["logloss"])
    # a reset orders after earlier adds and before later ones, across streams
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    r.add(m, stream=s1.cuda_stream)
    m.reset()
    r.add(m, stream=s2.cuda_stream)
    assert m.finish_bytes() == raw
    m.close()
