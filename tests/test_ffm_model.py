"""The float64 statement of the field-aware FM (ffm_model.FFM64) against its definition: the pairwise sum, central
differences of the logloss, and the canonical FM when every token is in the one field."""
import numpy as np
import pytest

from common import CanonicalFM64
from ffm_model import FFM64, pairwise_y


def _batch(rng, B, n_keys, F, max_len, x_signed=True):
    """Ragged rows (some empty) with repeated keys inside rows, several tokens per field, absent fields."""
    lens = rng.integers(0, max_len + 1, B)
    lens[0] = 0
    rp = np.zeros(B + 1, np.int64); rp[1:] = np.cumsum(lens)
    n = int(rp[-1])
    idx = rng.integers(0, n_keys, n)
    if n > 3:
        idx[1] = idx[0]
    fields = rng.integers(0, max(F - 1, 1), n).astype(np.uint8)    # field F-1 mostly absent ...
    fields[rng.random(n) < 0.1] = F - 1                             # ... but sometimes there
    x = rng.uniform(0.2, 1.8, n)
    if x_signed:
        x[rng.random(n) < 0.3] *= -1.0
    lab = (rng.random(B) < 0.4).astype(np.uint8)
    return idx, rp, fields, x, lab


@pytest.mark.parametrize("L", [4, 8, 16, 32])
def test_field_sums_equal_the_pairwise_definition(L):
    rng = np.random.default_rng(L)
    F, n_keys = L // 4, 40
    W0, V0 = rng.normal(0, 0.5, n_keys), rng.normal(0, 0.5, (n_keys, L))
    m = FFM64(W0, V0, "ftrl")
    for vals in (True, False):
        idx, rp, fields, x, _ = _batch(rng, 30, n_keys, F, 9)
        xv = x if vals else None
        got = m.forward(idx, rp, fields, xv)
        want = pairwise_y(m.W, m.V, idx, rp, fields, xv)
        assert np.abs(got - want).max() <= 1e-12 * max(1.0, np.abs(want).max())
        assert got[0] == 0.0                                        # a row without tokens


def _logloss(y, lab):
    return np.where(lab == 1, np.logaddexp(0.0, -y), np.logaddexp(0.0, y)).sum()


@pytest.mark.parametrize("L", [4, 16])
def test_gradients_are_the_derivative_of_the_logloss(L):
    rng = np.random.default_rng(7 + L)
    F, n_keys = L // 4, 12
    W0, V0 = rng.normal(0, 0.4, n_keys), rng.normal(0, 0.4, (n_keys, L))
    idx, rp, fields, x, lab = _batch(rng, 10, n_keys, F, 8)
    m = FFM64(W0, V0, "sgd")
    y = m.forward(idx, rp, fields, x)
    res = 1.0 / (1.0 + np.exp(-y)) - lab
    gw, gv = m.gradients(idx, rp, fields, x, res)
    h = 1e-6
    num_w = np.zeros(n_keys)
    for k in range(n_keys):
        for s in (1, -1):
            mm = FFM64(W0, V0, "sgd"); mm.W[k] += s * h
            num_w[k] += s * _logloss(mm.forward(idx, rp, fields, x), lab) / (2 * h)
    assert np.abs(num_w - gw).max() <= 1e-7 * max(1.0, np.abs(gw).max())
    num_v = np.zeros((n_keys, L))
    for k in range(n_keys):
        for c in range(L):
            for s in (1, -1):
                mm = FFM64(W0, V0, "sgd"); mm.V[k, c] += s * h
                num_v[k, c] += s * _logloss(mm.forward(idx, rp, fields, x), lab) / (2 * h)
    assert np.abs(num_v - gv).max() <= 1e-7 * max(1.0, np.abs(gv).max())
    assert np.abs(gv).max() > 1e-3                                  # the check has something to see


@pytest.mark.parametrize("opt", ["ftrl", "sgd"])
def test_one_field_is_the_canonical_fm(opt):
    """F = 1 (L = 4), every field 0: the model is XF_MODEL_FM_CANONICAL at K = 4, step for step."""
    rng = np.random.default_rng(3)
    n_keys = 50
    keys = np.arange(1000, 1000 + n_keys, dtype=np.uint64)
    W0, V0 = rng.normal(0, 0.3, n_keys), rng.normal(0, 0.3, (n_keys, 4))
    pull = lambda ks: (W0[np.searchsorted(keys, ks)], V0[np.searchsorted(keys, ks)])
    fm = CanonicalFM64(4, opt, pull)
    ffm = FFM64(W0, V0, opt, lr=1e-3)
    for step in range(3):
        idx, rp, _, x, lab = _batch(rng, 40, n_keys, 1, 7)
        fields = np.zeros(idx.size, np.uint8)
        a = fm.step(rp, keys[idx], x.astype(np.float32), lab)
        b = ffm.step(idx, rp, fields, x.astype(np.float32), lab)
        assert np.abs(a - b).max() <= 1e-12
    ks = fm.keys()
    e = fm.export(ks)
    u = np.searchsorted(keys, ks)
    for name, arr in (("w", ffm.W), ("v", ffm.V)) + ((("nw", ffm.NW), ("zw", ffm.ZW), ("nv", ffm.NV), ("zv", ffm.ZV))
                                                      if opt == "ftrl" else ()):
        want = e[name].reshape(u.size, -1)
        got = arr[u].reshape(u.size, -1)
        assert np.abs(got - want).max() <= 1e-12 * max(1.0, np.abs(want).max()), name
