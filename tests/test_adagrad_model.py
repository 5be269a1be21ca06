"""CPU checks of the AdaGrad statement (tests/adagrad_model.py): the zero-gradient identity, one rounding per
operation against exact rational arithmetic, the float64 bounds around the float32 step, and libffm's update."""
from fractions import Fraction

import numpy as np

import adagrad_model as A


def f32_round(x):
    """The float32 nearest to the rational x (ties to even), as a Fraction; x = 0 -> 0."""
    if x == 0:
        return Fraction(0)
    s = -1 if x < 0 else 1
    a = abs(x)
    e = a.numerator.bit_length() - a.denominator.bit_length()
    if Fraction(2) ** e > a:
        e -= 1
    e = max(e, -126)                      # subnormals share the smallest exponent's spacing
    ulp = Fraction(2) ** (e - 23)
    m = a / ulp
    r = m.numerator // m.denominator
    rem = m - r
    if rem > Fraction(1, 2) or (rem == Fraction(1, 2) and r % 2 == 1):
        r += 1
    return s * r * ulp


def sqrt_ok(x, r):
    """r (float32) is the nearest float32 to sqrt(x): sqrt(x) lies within half an ulp of r."""
    r = Fraction(float(r))
    e = r.numerator.bit_length() - r.denominator.bit_length()
    if Fraction(2) ** e > r:
        e -= 1
    half = Fraction(2) ** (e - 24)
    return (r - half) ** 2 <= x <= (r + half) ** 2


def values(seed, n):
    rng = np.random.default_rng(seed)
    g = (rng.standard_normal(n) * 10.0 ** rng.integers(-6, 3, n)).astype(np.float32)
    g[::7] = 0.0
    g[1::11] = np.float32(1e-40)          # subnormal
    g[2::13] = -np.float32(3e-39)
    w = (rng.standard_normal(n) * 0.3).astype(np.float32)
    nn = (rng.random(n) * 10.0 ** rng.integers(-8, 3, n)).astype(np.float32)
    nn[::5] = 0.0
    return g, w, nn


def test_zero_gradient_leaves_the_state():
    _, w, n = values(1, 4096)
    for z in (np.float32(0.0), np.float32(-0.0)):
        w2, n2 = A.step32(np.full_like(w, z), w, n)
        assert np.array_equal(w2.view(np.uint32), w.view(np.uint32))
        assert np.array_equal(n2.view(np.uint32), n.view(np.uint32))


def test_one_rounding_per_operation():
    g, w, n = values(2, 600)
    for lr, beta in ((A.LR, A.BETA), (1e-3, 0.5), (-0.05, 3e-7)):
        w2, n2 = A.step32(g, w, n, lr, beta)
        L, Bt = Fraction(float(np.float32(lr))), Fraction(float(np.float32(beta)))
        for i in range(g.size):
            G, W, N = Fraction(float(g[i])), Fraction(float(w[i])), Fraction(float(n[i]))
            gg = f32_round(G * G)
            nn = f32_round(N + gg)
            assert Fraction(float(n2[i])) == nn, i
            d = f32_round(Bt + nn)
            s = Fraction(float(np.sqrt(np.float32(float(d)))))
            assert sqrt_ok(d, np.float32(float(s))), i
            num = f32_round(L * G)
            quo = f32_round(num / s)
            assert Fraction(float(w2[i])) == f32_round(W - quo), i


def test_bounds_hold_the_float32_step():
    g, w, n = values(3, 20000)
    ok = np.abs(g) > 1e-30
    g, w, n = g[ok], w[ok], n[ok]
    rng = np.random.default_rng(4)
    eg = np.abs(g).astype(np.float64) * 1e-6 * rng.random(g.size)
    # a float32 gradient inside the interval: the bounds must hold the device's step from any of them
    gs = (g.astype(np.float64) + eg * (2 * rng.random(g.size) - 1)).astype(np.float32)
    inside = np.abs(gs.astype(np.float64) - g) <= eg
    w2, n2 = A.step32(gs, w, n)
    b = A.step64(g, eg, w, n)
    for name, got in (("w", w2), ("n", n2)):
        _, lo, hi = b[name]
        got = got.astype(np.float64)
        assert np.all(((got >= lo) & (got <= hi))[inside]), name
    # and they are tight: a step with twice the learning rate falls outside for most coordinates
    wbad, _ = A.step32(gs, w, n, lr=2 * A.LR)
    _, lo, hi = b["w"]
    moved = np.abs(g) > 1e-3
    assert np.mean(((wbad >= lo) & (wbad <= hi))[moved & inside]) < 0.01


def test_beta_one_is_libffm_in_exact_arithmetic():
    # a hand example: gradients 1/2, -3/4, 1/8 from w = 1/4, n = 0, eta = 1/5 (libffm: G = 1)
    gs = [Fraction(1, 2), Fraction(-3, 4), Fraction(1, 8)]
    eta = Fraction(1, 5)
    n, G = Fraction(0), Fraction(1)
    for g in gs:
        n += g * g
        G += g * g
        assert 1 + n == G  # the denominators agree exactly, so the steps eta g / sqrt(.) do too
    # and the float32 steps differ from libffm's float64 ones only by rounding
    w32, n32 = np.float32(0.25), np.float32(0.0)
    w64, G64 = 0.25, 1.0
    for g in gs:
        w32, n32 = A.step32(np.float32(float(g)), w32, n32, lr=float(eta), beta=1.0)
        w64, G64 = A.libffm_step(float(g), w64, G64, eta=float(eta))
    assert abs(float(w32) - w64) <= 8 * A.U * abs(w64)
    assert abs(float(n32) + 1.0 - G64) <= 4 * A.U * G64


def test_not_bitwise_libffm():
    # libffm rounds the running sum that starts at 1; here n starts at 0 and beta is added after: the float32 results
    # can differ in the last place
    rng = np.random.default_rng(5)
    g = (rng.standard_normal(4000) * 1e-3).astype(np.float32)
    w = np.zeros_like(g)
    n = np.zeros_like(g)
    G = np.ones_like(g)
    wl = np.zeros_like(g)
    for _ in range(3):
        w, n = A.step32(g, w, n, beta=1.0)
        G = (G + g * g).astype(np.float32)
        wl = (wl - (np.float32(A.LR) * g) / np.sqrt(G)).astype(np.float32)
    assert np.all(np.abs(w.astype(np.float64) - wl) <= 1e-5 * np.abs(wl) + 1e-12)
    assert not np.array_equal(w.view(np.uint32), wl.view(np.uint32))
