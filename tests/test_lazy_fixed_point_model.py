"""CPU model of the fixed-point residual sums of lazy LR tables (xflow_b200/csrc/table.cuh: xf_fix_shift,
xf_fix_of, xf_lazy_add, xf_lazy_fold).

A lazy row keeps the residual sum of its pending batch in the top 48 bits of a 64-bit word, as a signed integer
in units of 2^-s: every token's residual is rounded to a multiple of 2^-s (xf_fix_of) and added with an integer
atomic, which wraps silently at 48 bits.  The unit is chosen per batch from a bound on its token count nnz: the
largest s <= 27 with nnz * 2^s <= 2^47 - 1, and it is recorded beside the batch's row count, so that the fold of a
pending step scales the sum back with the unit that made it.

Claims checked: (1) the rule never lets a sum leave the 48-bit field, including the extreme batch in which every
token of the batch has |residual| = 1 on one key; (2) the step the fold then applies equals the eager step
(float32 of the exact residual sum, divided by the row count) within the quantisation bound
count * 2^-s / 2 of the sum; (3) a fixed unit of 2^-27 -- what lazy tables used before the rule -- wraps at
2^20 tokens of residual 1 and flips the sign of the step; (4) steps of batches with different units that are
pending at the same time each fold with their own unit."""
import numpy as np
import pytest

F = np.float32
FIELD_BITS = 48


def fix_shift(nnz):
    """xf_fix_shift: the largest s <= 27 with nnz * 2^s <= 2^47 - 1."""
    s = 47 - int(nnz).bit_length()
    return max(0, min(27, s))


def wrap48(x):
    """What the 48-bit field holds after integer adds that sum to x (two's complement, silently wrapping)."""
    m = x & ((1 << FIELD_BITS) - 1)
    return m - (1 << FIELD_BITS) if m >> (FIELD_BITS - 1) else m


def fix_of(residual, s):
    """xf_fix_of: the residual in units of 2^-s, rounded to nearest (ties to even, __double2ll_rn)."""
    return int(np.rint(np.float64(F(residual)) * 2.0 ** s))


def field_sum(residuals, s):
    """The deposits of one key's tokens into its row: per-token rounding, integer adds, 48-bit wrap."""
    r = np.asarray(residuals, np.float32).astype(np.float64)
    fixes = np.rint(r * 2.0 ** s).astype(np.int64)
    return wrap48(int(fixes.sum()))


def fold_grad(gfix, s, rows):
    """xf_lazy_fold: the sum scaled back with its batch's unit, rounded to float once, divided in double."""
    return F(np.float64(F(gfix * 2.0 ** -s)) / rows)


def test_fix_shift_rule():
    assert fix_shift(0) == fix_shift(1) == fix_shift((1 << 20) - 1) == 27
    assert fix_shift(1 << 20) == 26
    assert fix_shift(6_553_600) == 24                      # the bench's 65 536 rows x 100 tokens
    assert fix_shift((1 << 32) - 1) == 15                  # the largest token count a batch can declare
    for nnz in list(range(1, 70)) + [(1 << k) + d for k in range(1, 40) for d in (-1, 0, 1)]:
        s = fix_shift(nnz)
        assert nnz * 2 ** s <= 2 ** 47 - 1
        assert s == 27 or nnz * 2 ** (s + 1) > 2 ** 47 - 1   # the finest unit that fits


@pytest.mark.parametrize("sign", [1.0, -1.0])
def test_extreme_batches_never_wrap(sign):
    # every token of the batch on one key with |residual| = 1: the largest sum a batch of nnz tokens can make.  The
    # constraint is monotone in nnz for a fixed unit, so the ends of every bit length cover all token counts.
    for k in range(0, 33):
        for nnz in {max(1, (1 << k) - 1), 1 << k, (1 << k) + 1}:
            if nnz >= 1 << 32:
                continue
            s = fix_shift(nnz)
            exact = int(sign) * nnz * fix_of(1.0, s)
            assert wrap48(exact) == exact, (nnz, s)
            # the step: the sum is an integer number of tokens, exactly representable at every unit
            assert fold_grad(wrap48(exact), s, 1.0) == F(sign * nnz)


def test_fixed_unit_of_2_27_wraps_at_2_20_tokens():
    nnz = 1 << 20
    gfix = wrap48(nnz * fix_of(1.0, 27))
    assert gfix == -(1 << 47)                              # the sum +2^20 reads back as -2^20
    assert fold_grad(gfix, 27, 16384) == F(-64.0)          # the step moves the weight the wrong way
    s = fix_shift(nnz)
    assert fold_grad(wrap48(nnz * fix_of(1.0, s)), s, 16384) == F(64.0)
    # just below the boundary the old unit still held
    assert fix_shift(nnz - 64) == 27 and wrap48((nnz - 64) * fix_of(1.0, 27)) == (nnz - 64) << 27


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_quantised_sums_match_eager_steps_within_the_bound(seed):
    rng = np.random.default_rng(seed)
    for _ in range(40):
        count = int(rng.integers(1, 5000))
        nnz = int(rng.choice([count, 1 << 20, 6_553_600, (1 << 32) - 1, int(rng.integers(count, 1 << 32))]))
        s = fix_shift(nnz)
        kind = rng.integers(0, 3)
        if kind == 0:
            r = rng.uniform(-1, 1, count)
        elif kind == 1:
            r = rng.choice([-1.0, 1.0, F(1e-6) - 1.0, 1.2e-4, 0.5], count)
        else:
            r = rng.uniform(-1, 1, count) * 10.0 ** rng.uniform(-8, 0, count)
        r = r.astype(np.float32)
        gfix = field_sum(r, s)
        exact = float(np.sum(r.astype(np.float64)))
        unit = 2.0 ** -s
        assert abs(gfix * unit - exact) <= count * unit / 2 * (1 + 1e-12), (count, s)
        rows = float(rng.integers(1, 70000))
        got = np.float64(fold_grad(gfix, s, rows))
        want = np.float64(F(np.float64(F(exact)) / rows))           # eager: float32(exact sum) / rows
        tol = (count * unit / 2) / rows + 2 * np.spacing(F(abs(want) + 1e-30)).astype(np.float64)
        assert abs(got - want) <= tol, (count, s, got, want)


def test_pending_steps_fold_with_their_own_unit():
    # two batches with steps pending at once (on different keys), e.g. batches of two trainers on one table, or the
    # steps a ring flush folds: each entry of rows_by_seq carries its own unit
    rows_by_seq = {}
    rows = {}
    batches = [(1, 3 << 20, "a", [0.75] * 9), (2, 1000, "b", [0.75] * 9)]   # units 2^-25 and 2^-27
    for seq, nnz, key, residuals in batches:
        s = fix_shift(nnz)
        rows_by_seq[seq] = (64, s)
        rows[key] = (seq, field_sum(residuals, s))
    for key, (seq, gfix) in rows.items():
        n_rows, s = rows_by_seq[seq]
        assert fold_grad(gfix, s, n_rows) == F(6.75 / 64)
    # folding with the other batch's unit would be off by a power of two
    assert fold_grad(rows["a"][1], 27, 64) != F(6.75 / 64)
