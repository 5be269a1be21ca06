"""AdaGrad, the table's third per-coordinate optimizer (include/xflow_b200.h, section 2), stated twice:

  * step32: the definition, operation by operation in numpy float32 (each numpy float32 operation is rounded to
    nearest on its own, and np.sqrt is correctly rounded), which the device must match bit for bit:
        n' = fl(n + fl(g * g))
        w' = fl(w - fl(fl(eta * g) / fl(sqrt(fl(beta + n')))))
  * step64: float64 with rounding bounds for a gradient known only to [g - eg, g + eg], in the style of
    fm_model.ftrl_step / sgd_step, for the training checks whose gradients the device sums in another order.

eta is the table's learning_rate and beta its beta, both float32 fields of the table's config.
"""
import numpy as np

U = 2.0 ** -24
SAFETY = 1.01
LR = float(np.float32(0.2))    # libffm's default eta
BETA = 1.0                     # libffm's accumulator start


def step32(g, w, n, lr=LR, beta=BETA):
    """One AdaGrad step per coordinate in float32: returns (w', n')."""
    g, w, n = (np.asarray(a, np.float32) for a in (g, w, n))
    lr, beta = np.float32(lr), np.float32(beta)
    with np.errstate(over="ignore", invalid="ignore", divide="ignore"):
        n2 = (n + g * g).astype(np.float32)
        w2 = (w - (lr * g) / np.sqrt(beta + n2)).astype(np.float32)
    return w2, n2


def step64(g, eg, w, n, lr=LR, beta=BETA):
    """The step for a gradient in [g - eg, g + eg] from the float state (w, n): {w, n: (centre, lo, hi)} in float64,
    with the float32 roundings of every operation inside the bounds."""
    g, eg, w, n = (np.asarray(a, np.float64) for a in (g, eg, w, n))
    lr, beta = float(np.float32(lr)), float(np.float32(beta))
    glo, ghi = g - eg, g + eg

    def q(x):  # eta g / sqrt(beta + n + g^2): increasing in g for eta > 0, decreasing for eta < 0
        return lr * x / np.sqrt(beta + n + x * x)

    g2lo = np.where((glo <= 0) & (ghi >= 0), 0.0, np.minimum(glo * glo, ghi * ghi))
    g2hi = np.maximum(glo * glo, ghi * ghi)
    G2 = g2hi
    e_n = SAFETY * U * (2 * G2 + n)               # g*g, then n + g*g
    n_c = n + g * g
    nlo, nhi = n + g2lo - e_n, n + g2hi + e_n
    qa, qb = q(glo), q(ghi)
    qlo, qhi = np.minimum(qa, qb), np.maximum(qa, qb)
    # relative error of the quotient: eta*g (U), the sqrt (U), the division (U), and half the relative error of
    # beta + n' (n' and the add: 3U, halved by the sqrt): 4.5U
    qmag = np.maximum(np.abs(qlo), np.abs(qhi))
    e_q = SAFETY * 4.5 * U * qmag
    w_c = w - q(g)
    wlo, whi = w - qhi - e_q, w - qlo + e_q
    e_w = SAFETY * U * np.maximum(np.abs(wlo), np.abs(whi))
    return dict(w=(w_c, wlo - e_w, whi + e_w), n=(n_c, nlo, nhi))


def libffm_step(g, w, G, eta=LR):
    """libffm's update for comparison: its accumulator G starts at 1 and holds the running sum; G' = G + g g,
    w' = w - eta g / sqrt(G')."""
    G2 = G + g * g
    return w - eta * g / np.sqrt(G2), G2

