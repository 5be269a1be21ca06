"""The numpy restatement of the deterministic step's association (deterministic_model.py) on the CPU: -0.0 padding is
the identity, a one-term key equals a plain add, and the butterfly's order is the one written out by hand."""
import numpy as np

import deterministic_model as DM


def _bits(a):
    a = np.asarray(a)
    return a.view(np.uint32 if a.dtype == np.float32 else np.uint64)


def test_negative_zero_padding_is_the_identity():
    rng = np.random.default_rng(1)
    vals = np.concatenate([rng.normal(0, 1, 50), [0.0, -0.0, np.inf, -np.inf, 1e-45, -1e-45]]).astype(np.float32)
    for v in vals:
        assert _bits(v + np.float32(-0.0)) == _bits(v)
        assert _bits(DM.butterfly(np.array([v], np.float32))) == _bits(v)
    for v in vals.astype(np.float64):
        assert _bits(DM.butterfly(np.array([v]))) == _bits(v)


def test_one_term_key_is_a_plain_add():
    """A key with one token gets start + term, the bits of the default step's single atomic add."""
    rng = np.random.default_rng(2)
    for _ in range(200):
        t = rng.normal(0, 1, 4).astype(np.float32)
        s = rng.normal(0, 1, 4).astype(np.float32)
        assert (_bits(DM.key_sum(t[None, :], s)) == _bits(s + t)).all()
        g = rng.normal()
        assert _bits(DM.key_sum(np.array([g]), -0.0)) == _bits(np.float64(-0.0) + g)
    # signed zeros: g from -0.0 stays -0.0 for a term of -0.0 and becomes +0.0 for +0.0, as an atomic add does
    assert _bits(DM.key_sum(np.array([-0.0]), -0.0)) == _bits(np.float64(-0.0))
    assert _bits(DM.key_sum(np.array([0.0]), -0.0)) == _bits(np.float64(0.0))


def test_butterfly_order_by_hand():
    """Eight terms where the association shows: lane 0 ends with ((t0 + t4) + (t2 + t6)) + ((t1 + t5) + (t3 + t7)),
    the lanes past 8 adding -0.0 at o = 16 and 8."""
    t = np.array([1.0, 2.0 ** -24, -1.0, 2.0 ** -24, 3.0, -3.0, 2.0 ** -25, 2.0 ** -25], np.float32)
    f = np.float32
    want = (f(t[0] + t[4]) + f(t[2] + t[6])) + (f(t[1] + t[5]) + f(t[3] + t[7]))
    assert _bits(DM.butterfly(t)) == _bits(np.float32(want))
    # a left fold differs on these terms, so the test can tell the orders apart
    fold = np.float32(0.0)
    for v in t:
        fold = np.float32(fold + v)
    assert _bits(fold) != _bits(np.float32(want))


def test_runs_of_32_add_in_order():
    rng = np.random.default_rng(3)
    t = (rng.normal(0, 1, 100) * 2.0 ** rng.integers(-20, 20, 100)).astype(np.float32)
    want = np.float32(0.0)
    for i in range(0, 100, 32):
        want = np.float32(want + DM.butterfly(t[i:i + 32]))
    assert _bits(DM.key_sum(t, np.float32(0.0))) == _bits(want)
    # a full run: the tree whose level o adds a_i + a_(i+o) for i < o
    a = list(t[:32])
    for o in (16, 8, 4, 2, 1):
        a = [np.float32(a[i] + a[i + o]) for i in range(o)]
    assert _bits(DM.butterfly(t[:32])) == _bits(a[0])


def test_sgd_update_restatement():
    """The optimizer step from the accumulators: with L2 = 0 the latent gradient is A / rows exactly."""
    v = np.array([0.5, -0.25], np.float32)
    w, v2 = DM.sgd_update(0.0, v, (np.array([0.5, 1.0], np.float32), 0.25, 0.0), 4.0, 1.0)
    assert w == np.float32(-0.0625)
    assert (v2 == np.array([0.375, -0.5], np.float32)).all()
