"""The lazy LR step (xflow_b200/csrc/step_lazy.cu: xf_k_step_lr_lazy) against the exact ledger of tests/lr_ledger.py
(pytest -m gpu).

For every step: export the batch's keys, step, read the residuals back, hold them to residual_bounds (an order-free
interval from the pre-step weights), and require the exported post-step state of every key of the batch to equal
ledger_step() bit for bit.  The residual sums are integers, so the post-step table is a function of the pre-step state
and the kernel's own residuals whatever order its atomics land in: one token deposit lost, doubled or mis-scaled
changes some key's bits.  Each step also checks that keys outside the batch did not change, that the unique-key count
grows by the keys the step trained and the table by the keys it inserted.

The launch gives each row a group of G = 128 threads when the batch averages more than 64 tokens per row and of 64
otherwise; rows longer than G take the long-row path (phase A opens the row with an empty deposit in each later round,
phase B looks again and adds per token).  The grid is the CTAs that fit on the GPU at once, and each group strides over
the rows.  The matrices below cover both widths, every row length around the multiples of 32 and of G, key placements
across warps and rounds, grids around the resident size, the full-size shapes, batches past 2^20 tokens, and every
template instantiation (admission, eviction stamps, importance weights)."""
import numpy as np
import pytest

import lr_ledger as L
from common import assert_close
from oracle import oracle as O
from xflow_b200 import api, datagen

pytestmark = pytest.mark.gpu

LENGTHS = [0, 1, 31, 32, 33, 63, 64, 65, 95, 96, 97, 127, 128, 129, 191, 192, 193, 256, 257, 1000, 4097]
OPT = {"ftrl": api.OPT_FTRL, "sgd": api.OPT_SGD}
FIELDS = ("w", "nw", "zw")


def group_width(rp):
    """The G the launch picks for a batch (xf_launch_step_lr_lazy)."""
    B = rp.size - 1
    return 64 if int(rp[-1]) <= 64 * B else 128


def csr(lens, keys, rng):
    rp = np.zeros(len(lens) + 1, np.uint32)
    rp[1:] = np.cumsum(lens)
    assert keys.size == rp[-1]
    lab = (rng.random(len(lens)) < 0.3).astype(np.uint8)
    return rp, np.ascontiguousarray(keys, np.uint64), lab


def random_keys(rng, n, space):
    return api.hash_decimal_ids(rng.integers(0, space, n).astype(np.uint64))


def mixed_batch(rng, width, space, extra_lens=(), filler=None, rows=None):
    """Every length of LENGTHS (and extra_lens), shuffled among filler rows that set the batch's average tokens per row
    to <= 64 (width 64) or > 64 (width 128)."""
    lens = list(LENGTHS) + list(extra_lens)
    if filler is None:
        filler = (1, 40) if width == 64 else (66, 220)
    n = rows if rows is not None else (600 if width == 64 else 300)
    lens += list(rng.integers(filler[0], filler[1], n - len(lens)))
    lens = np.asarray(lens, np.int64)
    rng.shuffle(lens)
    rp, keys, lab = csr(lens, random_keys(rng, int(lens.sum()), space), rng)
    assert group_width(rp) == width, (width, int(rp[-1]), lens.size)
    return rp, keys, lab


class Run:
    """A table and trainer driven step by step under the ledger."""

    def __init__(self, opt="ftrl", capacity=1 << 20, max_rows=1 << 17, max_nnz=1 << 23, admission=None, eviction=False,
                 seed=0):
        self.opt = opt
        self.table = api.Table(optimizer=OPT[opt], capacity=capacity)
        if admission is not None:
            self.table.set_admission(**admission)
        if eviction:
            self.table.set_eviction(max_idle_batches=1 << 20)
        self.admitted = admission is not None
        self.eviction = eviction
        self.tr = api.Trainer(self.table, max_rows=max_rows, max_nnz=max_nnz, keep_loss=True)
        self.rng = np.random.default_rng(1000 + seed)
        self.seen = np.zeros(0, np.uint64)
        self.steps = 0

    def import_some(self, keys, frac=0.3):
        """Import a state on a fraction of `keys` whose FTRL weight is not f(z, n) (SGD: just a weight)."""
        uk = np.unique(keys)
        pick = uk[self.rng.random(uk.size) < frac]
        n = pick.size
        # weights up to a few units: rows far from pctr = 0.5 have residuals finer than the unit, so a wrong unit shows
        w = (self.rng.standard_normal(n) * 10.0 ** self.rng.uniform(-3, 0.7, n)).astype(np.float32)
        nw = (10.0 ** self.rng.uniform(-6, 0, n)).astype(np.float32) if self.opt == "ftrl" else None
        zw = (self.rng.standard_normal(n) * 0.01).astype(np.float32) if self.opt == "ftrl" else None
        self.table.import_(pick, w=w, nw=nw, zw=zw)
        e = self.table.export(pick)
        assert np.array_equal(e["w"].view(np.uint32), w.view(np.uint32))
        if self.opt == "ftrl":
            assert np.mean(w != L.ftrl_w(zw, nw)) > 0.9
        return pick

    def step(self, rp, keys, lab, e=None, predict_first=False, what=""):
        """One step under the ledger; returns (residuals, ledger)."""
        t, tr = self.table, self.tr
        rp = np.asarray(rp, np.uint32)
        B = lab.size
        what = "%s step %d (B=%d, nnz=%d, G=%d)" % (what, self.steps, B, int(rp[-1]), group_width(rp))
        uk = np.unique(keys)
        inv = np.searchsorted(uk, keys)
        pctr = tr.predict_host(rp, keys) if predict_first else None   # predict inserts absent keys (no policy)
        pre = t.export(uk)
        pre_present = pre["present"].astype(bool)
        outside = np.setdiff1d(self.seen, uk)
        if outside.size > 4000:
            outside = outside[self.rng.choice(outside.size, 4000, replace=False)]
        out_pre = t.export(outside) if outside.size else None
        size0, uniq0, adm0 = t.size(), tr.stats()["unique_keys"], t.admission_stats()
        if e is None:
            tr.step_host(rp, keys, lab)
        else:
            tr.step_host_weighted(rp, keys, lab, e)
        res = tr.get_loss(B)
        post = t.export(uk)
        present = post["present"].astype(bool)
        keep = present[inv] if self.admitted else None
        live = np.ones(B, bool) if e is None else np.asarray(e, np.float32) > 0
        # residuals: zero-weight rows are skipped, every other one lies in the order-free interval
        assert np.all(res[~live] == 0), what + ": a row of weight 0 has a residual"
        w_tok = pre["w"][inv] if keep is None else np.where(keep, pre["w"][inv], np.float32(0))
        lo, hi = L.residual_bounds(w_tok, rp, keys, lab)
        r = res.astype(np.float64)
        bad = live & ~((r >= lo) & (r <= hi))
        assert not bad.any(), "%s: %d residuals outside their bounds, e.g. row %d: %r not in [%r, %r]" % (
            what, int(bad.sum()), int(np.argmax(bad)), r[bad][0], lo[bad][0], hi[bad][0])
        if pctr is not None:
            neg = live & (lab == 0)
            assert np.array_equal(pctr[neg].view(np.uint32), res[neg].view(np.uint32)), \
                what + ": predict's pctr differs from the step's residual on rows with label 0"
        # the post-step state, bit for bit
        led = L.ledger_step(pre, rp, keys, res, B, self.opt, e=e, keep=keep)
        assert not (led.trained & ~present).any(), what + ": a trained key has no row"
        for f in FIELDS:
            diff = led[f].view(np.uint32) != post[f].view(np.uint32)
            if diff.any():
                i = int(np.argmax(diff))
                raise AssertionError("%s: %s of %d/%d keys differs from the ledger, e.g. key %d: got %r want %r "
                                     "(pre %r, sum %d, s %d)" % (what, f, int(diff.sum()), uk.size, int(uk[i]),
                                                                 post[f][i], led[f][i], pre[f][i], led.sums[i], led.s))
        # keys outside the batch, the table's size and the unique-key count
        if out_pre is not None:
            out_post = t.export(outside)
            for f in FIELDS + ("present",):
                assert np.array_equal(out_pre[f].view(np.uint8), out_post[f].view(np.uint8)), what + ": outside " + f
        new = led.trained & ~pre_present
        assert np.array_equal(present & ~pre_present, new), what + ": inserted keys"
        assert t.size() - size0 == int(new.sum()), what + ": size"
        assert tr.stats()["unique_keys"] - uniq0 == int(led.trained.sum()), what + ": unique keys"
        adm1 = t.admission_stats()
        assert adm1["batches"] == adm0["batches"] + 1
        if self.admitted:
            rejected = live[np.repeat(np.arange(B), np.diff(rp.astype(np.int64)))] & ~keep
            assert adm1["rejected_tokens"] - adm0["rejected_tokens"] == int(rejected.sum()), what + ": rejected tokens"
            assert adm1["admitted_keys"] - adm0["admitted_keys"] == int(new.sum()), what + ": admitted keys"
        if self.eviction:
            stamps = t.last_touch(uk[led.trained])
            assert np.all(stamps == adm0["batches"]), what + ": last_touch of the trained keys"
        self.seen = np.union1d(self.seen, uk[present])
        if self.seen.size > 200000:
            self.seen = self.seen[self.rng.choice(self.seen.size, 200000, replace=False)]
        self.steps += 1
        return res, led


# ---------------------------------------------------------------------------------------------------------------------
# group width and row length


@pytest.mark.parametrize("opt", ["ftrl", "sgd"])
@pytest.mark.parametrize("width", [64, 128])
def test_row_lengths_at_both_group_widths(width, opt):
    """Rows of every length in LENGTHS (0 .. 4097: both sides of each multiple of 32 and of G) among filler rows, at
    G = 64 (rows of 65 and more take the long-row path: opened by phase A's empty deposit, added to in phase B) and at
    G = 128.  Three steps of different row and token counts whose keys recur, so that every step folds the pending
    steps of the one before with their own divisor and unit; predict before each step equals the step's residuals on
    rows with label 0."""
    rng = np.random.default_rng(width + (opt == "sgd"))
    run = Run(opt, seed=width)
    for s, rows in enumerate((600, 377, 901) if width == 64 else (300, 211, 433)):
        rp, keys, lab = mixed_batch(rng, width, 30000, rows=rows)
        run.step(rp, keys, lab, predict_first=True, what="G=%d" % width)


def _at_switch(rng, B, extra, space=20000):
    """A batch of B rows and exactly 64 B + extra tokens, with rows of every length in LENGTHS."""
    lens = np.asarray(list(LENGTHS) + [0] * (B - len(LENGTHS)), np.int64)
    need = 64 * B + extra - int(lens.sum())
    free = np.arange(len(LENGTHS), B)
    lens[free] = need // free.size
    lens[free[: need % free.size]] += 1
    rng.shuffle(lens)
    rp, keys, lab = csr(lens, random_keys(rng, int(lens.sum()), space), rng)
    assert int(rp[-1]) == 64 * B + extra
    return rp, keys, lab


@pytest.mark.parametrize("extra", [0, 1], ids=["nnz=64B", "nnz=64B+1"])
def test_both_sides_of_the_group_width_switch(extra):
    """nnz = 64 B exactly (G = 64) and 64 B + 1 (G = 128): three steps each, with rows of every length in LENGTHS."""
    rng = np.random.default_rng(40 + extra)
    run = Run("ftrl", seed=40 + extra)
    for B in (700, 513, 1024):
        rp, keys, lab = _at_switch(rng, B, extra)
        assert group_width(rp) == (64 if extra == 0 else 128)
        run.step(rp, keys, lab, predict_first=True, what="switch")


# ---------------------------------------------------------------------------------------------------------------------
# key placement inside a row


def placement_batch(rng, width, hot, space=5000):
    """Rows that place keys across warps and rounds: key A at tokens 0, 32, 64 and 96 of a 128-token row (one leader per
    warp of round 0); key Bk only at tokens >= 128 of a 300-token row (opened by phase A's empty deposit at both G); key
    C at token 5 and again at 150 and 260; a row of 128 and a row of 4097 copies of key D / E; key H in every other row."""
    A, Bk, C, D, E, H = hot
    rows = []
    r = random_keys(rng, 128, space); r[[0, 32, 64, 96]] = A; rows.append(r)
    r = random_keys(rng, 300, space); r[[130, 200, 255, 256, 299]] = Bk; rows.append(r)
    r = random_keys(rng, 300, space); r[[5, 150, 260]] = C; rows.append(r)
    rows.append(np.full(128, D, np.uint64))
    rows.append(np.full(4097, E, np.uint64))
    lo, hi = (1, 30) if width == 64 else (70, 200)
    n = 400 if width == 64 else 200
    for ln in rng.integers(lo, hi, n):
        rows.append(random_keys(rng, int(ln), space))
    for r in rows[:3] + rows[5:]:
        r[rng.integers(0, r.size)] = H
    rows = [rows[i] for i in rng.permutation(len(rows))]
    lens = [r.size for r in rows]
    rp, keys, lab = csr(lens, np.concatenate(rows), rng)
    assert group_width(rp) == width
    return rp, keys, lab


@pytest.mark.parametrize("opt", ["ftrl", "sgd"])
@pytest.mark.parametrize("width", [64, 128])
def test_key_placement_across_warps_and_rounds(width, opt):
    """One key in every warp of round 0 (several CASes on one row), a key only in rounds >= 1, a key in round 0 and in
    later rounds, rows of 128 and 4097 copies of one key, and one key in every row (every group CASes the same row):
    three steps, the same hot keys each time."""
    rng = np.random.default_rng(7 * width + (opt == "sgd"))
    hot = random_keys(rng, 6, 1 << 40)
    run = Run(opt, seed=3 * width)
    for s in range(3):
        rp, keys, lab = placement_batch(rng, width, hot)
        res, led = run.step(rp, keys, lab, what="placement G=%d" % width)
        assert led.trained[np.searchsorted(led.uk, hot)].all()


# ---------------------------------------------------------------------------------------------------------------------
# the resident grid


def _sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def test_grids_around_the_resident_size():
    """B = SMs x c x 256 / G - 1, + 0 and + 1 rows for c = 1 .. 4 CTAs per SM at both G (whatever occupancy the build
    gets, one of these is the grid the launch picks, and the rows past it make some groups take a second row), B = 1, 2
    and 3, and batches of eight rows per group, in which each group strides over many rows and meets empty rows (no
    barrier before the summing point) and long rows (several rounds) in one sequence, reusing its shared slots and
    named barrier.  One table, every batch a ledger step from the state the batch before left."""
    sms = _sm_count()
    rng = np.random.default_rng(9)
    run = Run("ftrl", seed=9)
    sizes = [(w, sms * c * 256 // w + d) for c in (1, 2, 3, 4) for w in (64, 128) for d in (-1, 0, 1)]
    sizes += [(64, 1), (64, 2), (64, 3), (128, 1), (128, 2), (128, 3)]
    sizes += [(64, sms * 4 * 4 * 8), (128, sms * 4 * 2 * 8)]
    for w, B in sizes:
        if B <= 3:
            lens = rng.integers(0, 60, B) if w == 64 else rng.integers(65, 400, B)
        else:
            # empty and long rows among ordinary ones
            pool = [0, 0, 1, 33, 64, 65, 129, 257] if w == 64 else [0, 0, 1, 65, 128, 129, 257, 600]
            lens = rng.integers(1, 50, B) if w == 64 else rng.integers(66, 140, B)
            k = rng.random(B) < 0.15
            lens[k] = rng.choice(pool, int(k.sum()))
        if w == 128 and lens.sum() <= 64 * B:
            lens[0] += 64 * B + 1 - lens.sum()
        rp, keys, lab = csr(lens, random_keys(rng, int(lens.sum()), 50000), rng)
        assert group_width(rp) == w, (w, B)
        run.step(rp, keys, lab, what="grid")


# ---------------------------------------------------------------------------------------------------------------------
# full size


FULL = {"uniform": dict(dist="uniform", ragged=False), "zipf1.05": dict(dist="zipf", ragged=False),
        "ragged": dict(dist="uniform", ragged=True)}


@pytest.mark.parametrize("shape", sorted(FULL))
def test_full_size_batches_under_the_ledger(shape):
    """The metric's shape: B = 65 536 rows of 100 tokens over 10^8 ids (G = 128), uniform, Zipf(1.05) and ragged
    (0 .. 199 tokens per row); three steps each, bit for bit."""
    B, d = 65536, 100
    run = Run("ftrl", capacity=1 << 26, max_rows=B, max_nnz=B * 2 * d, seed=77)
    for s in range(3):
        rp, keys, lab = datagen.make_csr_keys(60 + s, B, d, 10 ** 8, api.hash_decimal_ids, **FULL[shape])
        assert group_width(rp) == 128
        run.step(rp, keys, lab, what="full " + shape)


def test_full_size_100_tokens_per_row_matches_oracle():
    """The metric's shape against the oracle (the reference's arithmetic) within 1e-5, in the style of
    test_full_batch_multi_step_matches_oracle: every residual of two steps and the state of every touched key."""
    B, d = 65536, 100
    gt = api.Table(optimizer=api.OPT_FTRL, capacity=1 << 25)
    ot = O.Table(K=0, opt=O.OPT_FTRL)
    tr = api.Trainer(gt, max_rows=B, max_nnz=B * d, keep_loss=True)
    seen = []
    for step in range(2):
        rp, keys, lab = datagen.make_csr_keys(80 + step, B, d, 10 ** 8, api.hash_decimal_ids)
        tr.step_host(rp, keys, lab)
        _, ol = ot.step(rp.astype(np.int64), keys, lab.astype(np.int32))
        assert_close(tr.get_loss(B), ol, "loss step %d" % step, abs_floor=1e-6)
        seen.append(keys)
    uk = np.unique(np.concatenate(seen))
    ge, oe = gt.export(uk), ot.export(uk)
    assert np.array_equal(ge["present"], oe["present"]) and gt.size() == ot.size()
    for f in FIELDS:
        assert_close(ge[f], oe[f], f)


def test_batch_past_2_20_tokens_then_a_small_one():
    """A G = 128 batch of just over 2^20 tokens (unit 2^-26) on few keys, so that the sums are large, then a small batch
    (unit 2^-27) on the same keys, then the big one again: each pending step folds with its own unit."""
    rng = np.random.default_rng(21)
    run = Run("ftrl", max_nnz=1 << 22, seed=21)
    big = csr(np.full(8192, 129), random_keys(rng, 8192 * 129, 3000), rng)
    small = mixed_batch(rng, 128, 3000)
    for rp, keys, lab in (big, small, big):
        res, led = run.step(rp, keys, lab, what="2^20")
        assert led.s == (26 if keys.size > 1 << 20 else 27)


# ---------------------------------------------------------------------------------------------------------------------
# the kernel's template instantiations: admission x eviction stamps x importance weights


VARIANTS = [(adm, stamp, weight) for adm in (None, "bloom", "poisson") for stamp in (False, True) for weight in (False, True)]


def _variant_id(v):
    adm, stamp, weight = v
    return "-".join([adm or "admit-all", "stamps" if stamp else "no-stamps", "weighted" if weight else "unweighted"])


@pytest.mark.parametrize("width", [64, 128])
@pytest.mark.parametrize("variant", VARIANTS, ids=[_variant_id(v) for v in VARIANTS])
def test_kernel_variants_under_the_ledger(variant, width):
    """Every instantiation of xf_k_step_lr_lazy<ADMIT, STAMP, WEIGHT> at both G, FTRL or SGD, with imported weights on
    part of the keys: Bloom or Poisson admission (keep = present after the step; admission_stats as the admission model
    states), eviction stamps (last_touch = the batch's number for every trained key), and step_host_weighted with weights
    of 0 (no residual, no deposit), fractions and values above 1."""
    adm, stamp, weight = variant
    opt = "sgd" if (stamp and not weight) or (adm == "poisson" and weight) else "ftrl"
    admission = None
    if adm == "bloom":
        admission = dict(mode=api.ADMIT_BLOOM, threshold=2, log2_cells=20, hashes=3, seed=5)
    elif adm == "poisson":
        admission = dict(mode=api.ADMIT_POISSON, probability=0.5, seed=5)
    seed = VARIANTS.index(variant) * 2 + (width == 128)
    rng = np.random.default_rng(500 + seed)
    run = Run(opt, admission=admission, eviction=stamp, seed=seed)
    space = 3000   # keys recur: the Bloom filter admits a key on its third sighting
    first = mixed_batch(rng, width, space)
    run.import_some(first[1])
    for s in range(3):
        rp, keys, lab = first if s == 0 else mixed_batch(rng, width, space, rows=(300 if width == 64 else 200) + 37 * s)
        e = None
        if weight:
            B = lab.size
            e = rng.choice(np.float32([0, 0.25, 0.5, 1, 1.5, 3, 7.75]), B).astype(np.float32)
            e[rng.random(B) < 0.2] = 0
        run.step(rp, keys, lab, e=e, what=_variant_id(variant))
    if adm is not None:
        st = run.table.admission_stats()
        assert st["rejected_tokens"] > 0 and st["admitted_keys"] > 0


# ---------------------------------------------------------------------------------------------------------------------
# invariance and cross-kernel checks


def _imported_pair(keys, opt="ftrl", seed=3):
    rng = np.random.default_rng(seed)
    uk = np.unique(keys)
    w = (rng.standard_normal(uk.size) * 0.05).astype(np.float32)
    nw = (10.0 ** rng.uniform(-6, 0, uk.size)).astype(np.float32)
    zw = (rng.standard_normal(uk.size) * 0.01).astype(np.float32)
    w[::3] = L.ftrl_w(zw[::3], nw[::3])
    out = []
    for _ in range(2):
        t = api.Table(optimizer=OPT[opt], capacity=1 << 20)
        t.import_(uk, w=w, nw=nw, zw=zw)
        out.append((t, api.Trainer(t, max_rows=1 << 14, max_nnz=1 << 22, keep_loss=True)))
    return out


def test_group_width_does_not_change_the_sums():
    """"pctr is the same float whatever G is" (step_lazy.cu): a G = 128 batch X and X' = X with empty rows interleaved
    until the average is <= 64 (G = 64), from the same imported state.  X's rows in X' predict and train with residuals
    identical bit for bit to X's, long rows included."""
    rng = np.random.default_rng(31)
    rp, keys, lab = mixed_batch(rng, 128, 20000, extra_lens=(100, 150, 200, 300, 513))
    B = lab.size
    lens = np.diff(rp.astype(np.int64))
    pad = int(np.ceil(keys.size / 64)) - B + 5
    where = np.sort(rng.integers(0, B + 1, pad))
    lens2 = np.insert(lens, where, 0)
    real = np.ones(lens2.size, bool)
    real[where + np.arange(pad)] = False
    assert np.array_equal(lens2[real], lens)
    lab2 = np.zeros(lens2.size, np.uint8)
    lab2[real] = lab
    rp2 = np.zeros(lens2.size + 1, np.uint32)
    rp2[1:] = np.cumsum(lens2)
    assert group_width(rp) == 128 and group_width(rp2) == 64
    (ta, tra), (tb, trb) = _imported_pair(keys)
    pa, pb = tra.predict_host(rp, keys), trb.predict_host(rp2, keys)
    assert np.array_equal(pa.view(np.uint32), pb[real].view(np.uint32)), "predict differs between G = 128 and G = 64"
    tra.step_host(rp, keys, lab)
    trb.step_host(rp2, keys, lab2)
    ra, rb = tra.get_loss(B), trb.get_loss(lens2.size)
    assert np.array_equal(ra.view(np.uint32), rb[real].view(np.uint32)), "residuals differ between G = 128 and G = 64"
    assert np.all(rb[~real] == 0.5)   # an empty row: pctr = sigmoid(0), label 0


@pytest.mark.parametrize("width", [64, 128])
def test_imported_weight_through_a_zero_step(width):
    """An imported FTRL weight that is not f(z, n) stands for w until the key's first step folds in.  When that step's
    residual sum is exactly 0 (two rows of pctr 0.5 with labels 0 and 1), the weight afterwards is f(z, n), and the
    next step must start from it: its residuals and its post-step state, for tokens in many groups of the batch."""
    rng = np.random.default_rng(90 + width)
    run = Run("ftrl", seed=90 + width)
    k = random_keys(rng, 1, 1 << 40)
    z, n = np.float32([0.02]), np.float32([0.5])
    assert L.ftrl_w(z, n)[0] != 0
    run.table.import_(k, w=np.float32([0.0]), nw=n, zw=z)
    # step 1: the key alone in two rows (wx = 0, pctr = 0.5) of labels 0 and 1: residuals +0.5 and -0.5
    lo, hi = (1, 30) if width == 64 else (70, 200)
    lens = [1, 1] + list(rng.integers(lo, hi, 200))
    rp, keys, lab = csr(lens, np.concatenate([k, k, random_keys(rng, int(sum(lens)) - 2, 10 ** 6)]), rng)
    lab[:2] = [0, 1]
    assert group_width(rp) == width
    res, led = run.step(rp, keys, lab, what="zero step")
    i = int(np.searchsorted(led.uk, k[0]))
    assert res[0] == 0.5 and res[1] == -0.5 and led.sums[i] == 0 and led.trained[i]
    assert run.table.export(k)["w"][0] == L.ftrl_w(z, n)[0]
    # step 2: the key in many rows
    lens = list(rng.integers(lo, hi, 300))
    rp, keys, lab = csr(lens, random_keys(rng, int(sum(lens)), 10 ** 6), rng)
    keys[rp[:-1][np.asarray(lens) > 0]] = k[0]
    run.step(rp, keys, lab, predict_first=True, what="after the zero step")
    run.step(rp, keys, lab, what="and again")


def test_predict_equals_training_residuals_at_both_widths():
    """Predict (mode 1 of the kernel) on a batch equals the training step's residuals bit for bit on rows with label 0,
    at G = 64 and G = 128, with admission off (predict inserts absent keys; the ledger's baselines are taken after)."""
    rng = np.random.default_rng(55)
    run = Run("sgd", seed=55)
    for width in (64, 128, 64, 128):
        rp, keys, lab = mixed_batch(rng, width, 8000)
        run.step(rp, keys, lab, predict_first=True, what="predict")


def test_frozen_model_predicts_as_the_table_after_g128_training():
    """After a G = 128 run, freeze() and the table's own predict agree bit for bit on a query batch that averages more
    than 64 tokens per row and holds rows of 65 .. 4097 tokens, some keys of it absent from the table: the serving
    kernel adds the terms in the order the step kernels add them."""
    rng = np.random.default_rng(66)
    run = Run("ftrl", seed=66)
    run.import_some(mixed_batch(rng, 128, 20000)[1])
    for s in range(3):
        run.step(*mixed_batch(rng, 128, 20000), what="serving")
    lens = [65, 96, 97, 127, 128, 129, 191, 192, 193, 256, 257, 1000, 4097] + list(rng.integers(66, 200, 300))
    rp, keys, _ = csr(lens, random_keys(rng, int(sum(lens)), 25000), rng)
    assert group_width(rp) == 128
    m = run.table.freeze()
    pm = m.predict_host(rp, keys)
    pt = run.tr.predict_host(rp, keys)
    assert np.array_equal(pm.view(np.uint32), pt.view(np.uint32))
