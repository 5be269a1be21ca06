"""Candidate scoring on serving models (xf_model_predict_candidates_*, csrc/serve.cu): a request's context scored
against each of its candidates returns, bit for bit, the model's flat predict of the concatenated row "context, then
candidate", on every model kind, precision, absent policy and prune setting, through both entry points."""
import numpy as np
import pytest

from xflow_b200 import api

pytestmark = pytest.mark.gpu

RUN = 16  # candidates per warp run in serve.cu (XF_CAND_RUN)
FIELDS = 32
ERR_ARG, ERR_STATE = "error -1:", "error -6:"
SPACE = 3000
CANON_K = (4, 8, 16, 32, 64, 128)
MVM_K = (4, 8, 16, 32)


def _keys_of(ids):
    return api.hash_decimal_ids(np.asarray(ids, np.uint64))


HELD = _keys_of(np.arange(SPACE))                      # rows the model holds
PULLED = _keys_of(np.arange(5 * SPACE, 5 * SPACE + 300))  # default rows: pruned
UNSEEN = _keys_of(np.arange(9 * SPACE, 9 * SPACE + 500))  # never in the table
POOL = np.concatenate([HELD, PULLED, UNSEEN])


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _table(kind, K):
    """A table with HELD imported (random w, v; a tenth of LR's w exactly 0) and PULLED pulled."""
    rng = np.random.default_rng(K + 100 * len(kind))
    canonical = kind in ("canon", "mvm")
    t = api.Table(latent_dim=K, optimizer=api.OPT_FTRL, v_init=api.VINIT_COUNTER, seed=3, capacity=1 << 14,
                  canonical_fm=1 if canonical else 0)
    w = rng.normal(0, 0.3, HELD.size).astype(np.float32)
    w[::10] = 0.0
    scale = 0.7 if kind == "mvm" else 0.2
    v = rng.normal(0, scale, (HELD.size, K)).astype(np.float32) if K else None
    t.import_(HELD, w=np.zeros_like(w) if kind == "mvm" else w, v=v)
    t.pull(PULLED, want_v=False)
    return t


def _freeze(t, kind, absent, prune):
    if kind == "mvm":
        return t.freeze_mvm(absent=absent, prune=prune)
    if kind == "canon":
        return t.freeze_canonical(absent=absent, prune=prune)
    return t.freeze(absent=absent, prune=prune)


KINDS = [("lr", 0), ("fm", 8)] + [("canon", K) for K in CANON_K] + [("mvm", K) for K in MVM_K]
_CACHE = {}


def _models(kind, K):
    """Every model of one table: (absent, prune, precision) -> Model."""
    if (kind, K) not in _CACHE:
        t = _table(kind, K)
        ms = {}
        for absent in (api.ABSENT_DEFAULT, api.ABSENT_ZERO):
            for prune in (True, False):
                m = _freeze(t, kind, absent, prune)
                ms[(absent, prune, api.PRECISION_F32)] = m
                if kind != "lr":
                    ms[(absent, prune, api.PRECISION_F16)] = m.convert(api.PRECISION_F16)
        t.close()
        _CACHE[(kind, K)] = ms
    return _CACHE[(kind, K)]


def _ids(cases):
    return ["%s%d" % c for c in cases]


# ---- batches ---------------------------------------------------------------------------------------------------------
class Batch:
    """R requests: contexts (ctx_ptr, ctx_keys, ctx_vals, ctx_fields) and candidates (cand_ptr, row_ptr, keys, vals,
    fields); vals and fields are None where a side has none."""

    def __init__(self, ctx_lens, cand_counts, cand_lens, rng, kind, vals=True, keys_from=None):
        R = len(ctx_lens)
        assert len(cand_counts) == R and sum(cand_counts) == len(cand_lens)
        self.ctx_ptr = _ptr(ctx_lens)
        self.cand_ptr = _ptr(cand_counts)
        self.row_ptr = _ptr(cand_lens)
        pool = POOL if keys_from is None else keys_from
        self.ctx_keys = pool[rng.integers(0, pool.size, int(self.ctx_ptr[-1]))].astype(np.uint64)
        self.keys = pool[rng.integers(0, pool.size, int(self.row_ptr[-1]))].astype(np.uint64)
        # keys repeat between a request's context and its candidates
        for q in range(R):
            a, b = int(self.ctx_ptr[q]), int(self.ctx_ptr[q + 1])
            for c in range(int(self.cand_ptr[q]), int(self.cand_ptr[q + 1])):
                x, y = int(self.row_ptr[c]), int(self.row_ptr[c + 1])
                if b > a and y > x and rng.random() < 0.5:
                    self.keys[x + int(rng.integers(0, y - x))] = self.ctx_keys[a + int(rng.integers(0, b - a))]
        value = kind in ("canon", "mvm") and vals
        self.ctx_vals = _vals(rng, self.ctx_keys.size) if value else None
        self.vals = _vals(rng, self.keys.size) if value else None
        if kind == "mvm":
            # fields 0 .. 7 on both sides, 8 .. 15 the context's only, 16 .. 31 the candidates' only
            self.ctx_fields = rng.integers(0, 16, self.ctx_keys.size).astype(np.uint8)
            self.fields = np.where(rng.random(self.keys.size) < 0.5, rng.integers(0, 8, self.keys.size),
                                   rng.integers(16, 32, self.keys.size)).astype(np.uint8)
            # field sums stay near 1 in long rows
            if value:
                for v, p in ((self.ctx_vals, self.ctx_ptr), (self.vals, self.row_ptr)):
                    n = np.diff(p.astype(np.int64))
                    v *= np.repeat(1.0 / np.sqrt(np.maximum(n, 1)), n).astype(np.float32)
        else:
            self.ctx_fields = self.fields = None

    @property
    def R(self):
        return self.cand_ptr.size - 1

    @property
    def N(self):
        return self.row_ptr.size - 1

    def flat(self):
        """The concatenated rows: (row_ptr, keys, vals, fields)."""
        lens, keys, vals, fields = [], [], [], []
        for q in range(self.R):
            a, b = int(self.ctx_ptr[q]), int(self.ctx_ptr[q + 1])
            for c in range(int(self.cand_ptr[q]), int(self.cand_ptr[q + 1])):
                x, y = int(self.row_ptr[c]), int(self.row_ptr[c + 1])
                lens.append(b - a + y - x)
                keys += [self.ctx_keys[a:b], self.keys[x:y]]
                if self.vals is not None or self.ctx_vals is not None:
                    vals += [_side(self.ctx_vals, a, b), _side(self.vals, x, y)]
                if self.fields is not None:
                    fields += [self.ctx_fields[a:b], self.fields[x:y]]
        cat = lambda xs, t: np.concatenate(xs).astype(t) if xs else np.zeros(0, t)
        return (_ptr(lens), cat(keys, np.uint64), cat(vals, np.float32) if vals else None,
                cat(fields, np.uint8) if self.fields is not None else None)


def _ptr(lens):
    p = np.zeros(len(lens) + 1, np.uint32)
    p[1:] = np.cumsum(np.asarray(lens, np.int64))
    return p


def _side(v, a, b):
    return np.ones(b - a, np.float32) if v is None else v[a:b]


def _vals(rng, n):
    """Feature values with negatives and exact zeros."""
    x = rng.uniform(-1.5, 2.0, n).astype(np.float32)
    x[rng.random(n) < 0.1] = 0.0
    return x


def _flat_predict(m, kind, b):
    rp, keys, vals, fields = b.flat()
    if kind == "mvm":
        return m.predict_host_fields(rp, keys, fields, vals)
    return m.predict_host(rp, keys, vals)


def _host(m, b):
    return m.predict_candidates(b.ctx_ptr, b.ctx_keys, b.cand_ptr, b.row_ptr, b.keys, ctx_vals=b.ctx_vals, vals=b.vals,
                                ctx_fields=b.ctx_fields, fields=b.fields)


def _dev(a, torch, dtype=None):
    if a is None:
        return None
    a = np.ascontiguousarray(a)
    if a.dtype == np.uint64:
        a = a.view(np.int64)
    elif a.dtype == np.uint32:
        a = a.view(np.int32)
    return torch.from_numpy(a.copy()).cuda()


class DeviceBatch:
    """A batch's arrays on the device (kept alive with the object)."""

    def __init__(self, b, torch):
        self.b = b
        self.t = {k: _dev(getattr(b, k), torch) for k in ("ctx_ptr", "ctx_keys", "ctx_vals", "ctx_fields", "cand_ptr",
                                                          "row_ptr", "keys", "vals", "fields")}

    def addr(self, k):
        x = self.t[k]
        return 0 if x is None else x.data_ptr()

    def run(self, m, out, stream):
        b = self.b
        m.predict_candidates_device(b.R, self.addr("ctx_ptr"), self.addr("ctx_keys"), b.ctx_keys.size,
                                    self.addr("cand_ptr"), b.N, self.addr("row_ptr"), self.addr("keys"), b.keys.size,
                                    out.data_ptr(), stream=stream.cuda_stream, d_ctx_vals=self.addr("ctx_vals"),
                                    d_vals=self.addr("vals"), d_ctx_fields=self.addr("ctx_fields"),
                                    d_fields=self.addr("fields"))


def _device(m, b):
    torch = pytest.importorskip("torch")
    d = DeviceBatch(b, torch)
    out = torch.full((max(b.N, 1),), -1.0, dtype=torch.float32, device="cuda")
    s = torch.cuda.Stream()
    torch.cuda.synchronize()
    d.run(m, out, s)
    s.synchronize()
    return out.cpu().numpy()[:b.N]


def _check(m, kind, b, what=""):
    want = _flat_predict(m, kind, b)
    got_h = _host(m, b)
    got_d = _device(m, b)
    assert got_h.shape == want.shape == (b.N,), what
    assert np.array_equal(_bits(got_h), _bits(want)), what
    assert np.array_equal(_bits(got_d), _bits(want)), what
    return want


def _random_batch(rng, kind, R=24, max_cands=40, max_ctx=80, max_len=50, vals=True):
    counts = [int(x) for x in rng.integers(0, max_cands + 1, R)]
    counts[1] = 0
    ctx = [int(x) for x in rng.integers(0, max_ctx + 1, R)]
    ctx[2] = 0
    lens = [int(x) for x in rng.integers(0, max_len + 1, sum(counts))]
    return Batch(ctx, counts, lens, rng, kind, vals=vals)


# ---- 1. random batches on every model ------------------------------------------------------------------------------
@pytest.mark.parametrize("kind,K", KINDS, ids=_ids(KINDS))
def test_random_batches_equal_the_flat_predict(kind, K):
    rng = np.random.default_rng(K + 7)
    spread = []
    for key, m in _models(kind, K).items():
        for vals in ((True, False) if kind in ("canon", "mvm") else (False,)):
            b = _random_batch(rng, kind, vals=vals)
            want = _check(m, kind, b, (key, vals))
            spread.append(len(set(want.tolist())))
    assert max(spread) > 50


# ---- 2. every alignment of the context against the lanes and lane groups -------------------------------------------
@pytest.mark.parametrize("kind,K", KINDS, ids=_ids(KINDS))
def test_alignment(kind, K):
    """Context lengths 0 .. 129 (every residue of 64 and of 2T, T = 128 / K) against candidates of 0, 1, 31, 32, 33
    and 100 tokens; one request per context length."""
    rng = np.random.default_rng(K + 11)
    ctx = list(range(130))
    shapes = [0, 1, 31, 32, 33, 100]
    b = Batch(ctx, [len(shapes)] * len(ctx), shapes * len(ctx), rng, kind)
    for key, m in _models(kind, K).items():
        _check(m, kind, b, key)


# ---- 3. run boundaries -----------------------------------------------------------------------------------------------
SOME = [("lr", 0), ("fm", 8), ("canon", 16), ("canon", 128), ("mvm", 8), ("mvm", 32)]


@pytest.mark.parametrize("kind,K", SOME, ids=_ids(SOME))
def test_run_boundaries(kind, K):
    rng = np.random.default_rng(K + 13)
    ms = _models(kind, K)
    m = ms[(api.ABSENT_DEFAULT, True, api.PRECISION_F32)]
    counts = [RUN - 1, RUN, RUN + 1, 3 * RUN + 5, 0, RUN - 1, 1, 3 * RUN + 5, RUN + 1, RUN]
    ctx = [int(x) for x in rng.integers(0, 70, len(counts))]
    b = Batch(ctx, counts, [int(x) for x in rng.integers(0, 40, sum(counts))], rng, kind)
    for key, mm in ms.items():
        _check(mm, kind, b, key)
    # 10 000 requests of one candidate each
    R = 10000
    b = Batch([int(x) for x in rng.integers(0, 20, R)], [1] * R, [int(x) for x in rng.integers(0, 12, R)], rng, kind)
    _check(m, kind, b, "one candidate each")
    # one request of 100 000 candidates
    N = 100000
    b = Batch([37], [N], [int(x) for x in rng.integers(0, 9, N)], rng, kind)
    _check(m, kind, b, "one request")


# ---- 4. long rows ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind,K", SOME, ids=_ids(SOME))
def test_long_rows(kind, K):
    rng = np.random.default_rng(K + 17)
    for key, m in _models(kind, K).items():
        _check(m, kind, Batch([4097, 5], [3, 2], [7, 0, 40, 4097, 4097], rng, kind), key)


# ---- 5. degenerate batches -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind,K", SOME, ids=_ids(SOME))
def test_degenerate_batches(kind, K):
    rng = np.random.default_rng(K + 19)
    for key, m in _models(kind, K).items():
        # R = 0
        b = Batch([], [], [], rng, kind)
        assert _host(m, b).size == 0 and _device(m, b).size == 0
        # requests, but no candidates at all
        b = Batch([3, 0, 9], [0, 0, 0], [], rng, kind)
        assert _host(m, b).size == 0 and _device(m, b).size == 0
        # an empty context: the flat predict of the candidates themselves
        b = Batch([0, 0], [3, 2], [5, 0, 17, 33, 1], rng, kind)
        want = _check(m, kind, b, key)
        rp = b.row_ptr
        if kind == "mvm":
            alone = m.predict_host_fields(rp, b.keys, b.fields, b.vals)
        else:
            alone = m.predict_host(rp, b.keys, b.vals)
        assert np.array_equal(_bits(want), _bits(alone))
        # empty candidates: the flat predict of the context
        b = Batch([6, 40], [2, 3], [0] * 5, rng, kind)
        want = _check(m, kind, b, key)
        if kind == "mvm":
            ctx = m.predict_host_fields(b.ctx_ptr, b.ctx_keys, b.ctx_fields, b.ctx_vals)
        else:
            ctx = m.predict_host(b.ctx_ptr, b.ctx_keys, b.ctx_vals)
        assert np.array_equal(_bits(want), _bits(np.repeat(ctx, [2, 3])))
        # all empty: sigmoid(0)
        b = Batch([0, 0, 0], [1, 0, 4], [0] * 5, rng, kind)
        assert _host(m, b).tolist() == [0.5] * 5 and _device(m, b).tolist() == [0.5] * 5


# ---- 6. full size ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("K", [0, 16])
def test_full_size(K):
    """R = 256 requests of N = 256 candidates, 64 context tokens and 36 per candidate: flat rows 65 536 x 100."""
    kind = "fm" if K else "lr"
    t = _table(kind, K)
    m = t.freeze()
    rng = np.random.default_rng(23)
    R = N = 256
    b = Batch([64] * R, [N] * R, [36] * (R * N), rng, kind, keys_from=np.concatenate([HELD, UNSEEN]))
    _check(m, kind, b, "full size")
    m.close()
    t.close()


# ---- 7. reproducibility ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind,K", SOME, ids=_ids(SOME))
def test_repeatable_and_streams(kind, K):
    torch = pytest.importorskip("torch")
    rng = np.random.default_rng(K + 29)
    m = _models(kind, K)[(api.ABSENT_DEFAULT, False, api.PRECISION_F32)]
    b1 = _random_batch(rng, kind, R=64)
    b2 = _random_batch(rng, kind, R=64)
    first = [_host(m, b1), _host(m, b2)]
    for _ in range(3):
        assert np.array_equal(_bits(_host(m, b1)), _bits(first[0]))
    assert np.array_equal(_bits(_device(m, b1)), _bits(first[0]))
    # two batches in flight on two streams at once, each issued several times
    d1, d2 = DeviceBatch(b1, torch), DeviceBatch(b2, torch)
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    outs = []
    torch.cuda.synchronize()
    for _ in range(4):
        o1 = torch.full((b1.N,), -1.0, dtype=torch.float32, device="cuda")
        o2 = torch.full((b2.N,), -1.0, dtype=torch.float32, device="cuda")
        torch.cuda.synchronize()
        d1.run(m, o1, s1)
        d2.run(m, o2, s2)
        outs.append((o1, o2))
    s1.synchronize()
    s2.synchronize()
    for o1, o2 in outs:
        assert np.array_equal(_bits(o1.cpu().numpy()), _bits(first[0]))
        assert np.array_equal(_bits(o2.cpu().numpy()), _bits(first[1]))


# ---- 8. refusals -----------------------------------------------------------------------------------------------------
def _raw(m, b, **over):
    """xf_model_predict_candidates_host on the batch's arrays with fields of the struct replaced."""
    arr = {k: getattr(b, k) for k in ("ctx_ptr", "ctx_keys", "ctx_vals", "ctx_fields", "cand_ptr", "row_ptr", "keys",
                                      "vals", "fields")}
    addr = {k: (None if v is None else v.ctypes.data) for k, v in arr.items()}
    f = dict(requests=b.R, ctx_nnz=b.ctx_keys.size, candidates=b.N, nnz=b.keys.size, **addr)
    f.update(over)
    s = api.CandidateBatch(**f)
    out = np.empty(max(b.N, 1), np.float32)
    return api.lib().xf_model_predict_candidates_host(m.h, api.C.byref(s), api._p(out)), api.lib().xf_last_error().decode()


def _refused(m, b, code, pattern, **over):
    import re
    rc, msg = _raw(m, b, **over)
    assert rc == code and re.search(pattern, msg), (rc, msg, over)


def test_refusals():
    rng = np.random.default_rng(31)
    lr = _models("lr", 0)[(api.ABSENT_DEFAULT, True, api.PRECISION_F32)]
    mv = _models("mvm", 8)[(api.ABSENT_DEFAULT, True, api.PRECISION_F32)]
    cn = _models("canon", 8)[(api.ABSENT_DEFAULT, True, api.PRECISION_F32)]
    b = Batch([3, 4], [2, 1], [2, 3, 1], rng, "lr")
    bm = Batch([3, 4], [2, 1], [2, 3, 1], rng, "mvm")
    assert _raw(lr, b)[0] == 0 and _raw(mv, bm)[0] == 0
    # null arguments
    for k in ("ctx_ptr", "cand_ptr", "row_ptr", "ctx_keys", "keys"):
        _refused(lr, b, -1, "null argument", **{k: None})
    for k in ("ctx_fields", "fields"):
        _refused(mv, bm, -1, "null argument", **{k: None})
    assert api.lib().xf_model_predict_candidates_host(lr.h, None, None) == -1
    # decreasing pointers
    for k, p in (("ctx_ptr", [3, 2, 7]), ("cand_ptr", [0, 4, 3]), ("row_ptr", [0, 2, 1, 6])):
        bad = np.array(p, np.uint32)
        _refused(lr, b, -1, k + " decreases", **{k: bad.ctypes.data})
    # cand_ptr's ends
    bad0 = np.array([1, 2, 3], np.uint32)
    _refused(lr, b, -1, "cand_ptr runs from 1", cand_ptr=bad0.ctypes.data)
    short = np.array([0, 2, 2], np.uint32)
    _refused(lr, b, -1, "cand_ptr runs from 0 to 2: .*candidates = 3", cand_ptr=short.ctypes.data)
    # past the tokens
    _refused(lr, b, -1, "ctx_ptr ends at 7, past ctx_nnz = 6", ctx_nnz=6)
    _refused(lr, b, -1, "row_ptr ends at 6, past nnz = 5", nnz=5)
    # the reserved key on either side
    for k in ("ctx_keys", "keys"):
        bad = getattr(b, k).copy()
        bad[1] = np.uint64(0xFFFFFFFFFFFFFFFF)
        _refused(lr, b, -1, k + ": key .* at position 1 is reserved", **{k: bad.ctypes.data})
    # field ids of 32 and more on either side
    for k in ("ctx_fields", "fields"):
        bad = getattr(bm, k).copy()
        bad[2] = 32
        _refused(mv, bm, -1, k + ": field id 32 of token 2", **{k: bad.ctypes.data})
    # kinds: values on LR, field ids on LR and canonical
    v = np.ones(b.keys.size, np.float32)
    _refused(lr, b, -1, "ignores feature values", vals=v.ctypes.data)
    _refused(lr, b, -1, "ignores feature values", ctx_vals=np.ones(7, np.float32).ctypes.data)
    f = np.zeros(16, np.uint8)
    _refused(lr, b, -1, "xf_table_freeze_mvm", fields=f.ctypes.data)
    _refused(cn, b, -1, "xf_table_freeze_mvm", ctx_fields=f.ctypes.data)
    # a part
    t = api.Table(capacity=1 << 12)
    t.import_(HELD[:10], w=np.ones(10, np.float32))
    part = t.freeze_part()
    _refused(part, b, -6, "is a part")
    part.close()
    t.close()
    # the Python layer checks sizes
    with pytest.raises(ValueError):
        lr.predict_candidates(b.ctx_ptr[:-1], b.ctx_keys, b.cand_ptr, b.row_ptr, b.keys)
    with pytest.raises(ValueError):
        mv.predict_candidates(bm.ctx_ptr, bm.ctx_keys, bm.cand_ptr, bm.row_ptr, bm.keys, ctx_fields=bm.ctx_fields,
                              fields=bm.fields[:-1])
    # the device entry point: a part, the kinds, null pointers
    torch = pytest.importorskip("torch")
    d = DeviceBatch(b, torch)
    out = torch.empty(b.N, dtype=torch.float32, device="cuda")
    with pytest.raises(api.XflowError, match=ERR_ARG + ".*ignores feature values"):
        lr.predict_candidates_device(b.R, d.addr("ctx_ptr"), d.addr("ctx_keys"), 7, d.addr("cand_ptr"), b.N,
                                     d.addr("row_ptr"), d.addr("keys"), 6, out.data_ptr(), d_vals=out.data_ptr())
    with pytest.raises(api.XflowError, match=ERR_ARG + ".*null argument"):
        mv.predict_candidates_device(b.R, d.addr("ctx_ptr"), d.addr("ctx_keys"), 7, d.addr("cand_ptr"), b.N,
                                     d.addr("row_ptr"), d.addr("keys"), 6, out.data_ptr())
