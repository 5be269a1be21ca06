"""float64 numpy statement of XF_MODEL_FFM (step_ffm.cu): the field-aware FM on canonical tables.

A key's latent row v[L] is F = L / 4 pieces of 4 coordinates; piece b is the key's vector for interacting with field b.
Row r has tokens i (key k_i, field f_i < F, value x_i):
    y = sum_i w_i x_i + sum_{i<j} <v_{i,f_j}, v_{j,f_i}> x_i x_j
computed through the field sums T[a][b] = sum_{i: f_i = a} x_i v_{i,b} and Q = sum_i x_i^2 |v_{i,f_i}|^2:
    y = sum_i w_i x_i + 1/2 (sum_{a,b} <T[a][b], T[b][a]> - Q)
    dL/dw_i = r x_i ,  dL/dv_{i,b} = r x_i (T[b][f_i] - [b = f_i] x_i v_{i,f_i})        r = sigmoid(y) - label
then gradients / rows and one FTRL or SGD step per touched key, on w and on all L coordinates.
"""
import numpy as np

from common import ftrl64

PIECE = 4  # coordinates per field vector (libffm's default k)


def sigmoid_ref(y):
    """Base::sigmoid as the device computes it: pow(2.718281828, y) with the clamps at -30 / 30."""
    with np.errstate(over="ignore"):
        e = np.power(2.718281828, np.clip(y, -30, 30))
    return np.where(y < -30, 1e-6, np.where(y > 30, 1.0, e / (1 + e)))


def pairwise_y(W, V, idx, rp, fields, x):
    """The definition itself: an explicit loop over the pairs i < j of each row's token positions."""
    L = V.shape[1]
    B = rp.size - 1
    x64 = np.ones(idx.size) if x is None else np.asarray(x, np.float64)
    y = np.zeros(B)
    for r in range(B):
        toks = range(int(rp[r]), int(rp[r + 1]))
        s = 0.0
        for i in toks:
            s += W[idx[i]] * x64[i]
        for i in toks:
            for j in toks:
                if j <= i:
                    continue
                fi, fj = int(fields[i]), int(fields[j])
                vi = V[idx[i], PIECE * fj: PIECE * fj + PIECE]
                vj = V[idx[j], PIECE * fi: PIECE * fi + PIECE]
                s += float(vi @ vj) * x64[i] * x64[j]
        y[r] = s
    assert L % PIECE == 0
    return y


class FFM64:
    """State W, NW, ZW [n] and V, NV, ZV [n, L] of the keys `idx` indexes; `lr` is the SGD learning rate."""

    def __init__(self, W0, V0, opt, lr=1e-3):
        self.V = np.asarray(V0, np.float64).copy()
        n, L = self.V.shape
        assert L % PIECE == 0
        self.F = L // PIECE
        self.W = np.zeros(n) if W0 is None else np.asarray(W0, np.float64).copy()
        self.NW, self.ZW = np.zeros(n), np.zeros(n)
        self.NV, self.ZV = np.zeros_like(self.V), np.zeros_like(self.V)
        self.opt, self.lr = opt, lr

    def _sums(self, idx, rp, fields, x):
        B, F = rp.size - 1, self.F
        row_of = np.repeat(np.arange(B), np.diff(rp).astype(np.int64))
        x64 = np.ones(idx.size) if x is None else np.asarray(x, np.float64)
        f = np.asarray(fields, np.int64)
        assert idx.size == 0 or f.max() < F
        Vt = self.V[idx].reshape(-1, F, PIECE)                        # [nnz, b, 4]: v_{i,b}
        T = np.zeros((B, F, F, PIECE)); np.add.at(T, (row_of, f), x64[:, None, None] * Vt)
        own = Vt[np.arange(idx.size), f]                               # v_{i,f_i}
        Q = np.zeros(B); np.add.at(Q, row_of, x64 ** 2 * (own ** 2).sum(1))
        wx = np.zeros(B); np.add.at(wx, row_of, self.W[idx] * x64)
        return row_of, x64, f, Vt, own, T, Q, wx

    @staticmethod
    def _blocks(rp, x, rows=1024):
        """The batch cut into blocks of rows (T takes B F^2 4 doubles): (row range, token range, x of the block)."""
        B = rp.size - 1
        for r0 in range(0, max(B, 1), rows):
            r1 = min(r0 + rows, B)
            a, b = int(rp[r0]), int(rp[r1])
            yield r0, r1, a, b, (None if x is None else x[a:b])

    def forward(self, idx, rp, fields, x):
        """y of every row."""
        y = np.zeros(rp.size - 1)
        for r0, r1, a, b, xb in self._blocks(rp, x):
            _, _, _, _, _, T, Q, wx = self._sums(idx[a:b], rp[r0:r1 + 1] - rp[r0], fields[a:b], xb)
            y[r0:r1] = wx + 0.5 * (np.einsum("rabk,rbak->r", T, T) - Q)
        return y

    def gradients(self, idx, rp, fields, x, res):
        """Per-key sums (not yet / rows) of dL/dw and dL/dv for row residuals `res`: gw [n], gv [n, L]."""
        gw = np.zeros(self.W.size)
        gv = np.zeros_like(self.V)
        res = np.asarray(res, np.float64)
        for r0, r1, a, b, xb in self._blocks(rp, x):
            ib = idx[a:b]
            row_of, x64, f, Vt, own, T, _, _ = self._sums(ib, rp[r0:r1 + 1] - rp[r0], fields[a:b], xb)
            rx = res[r0:r1][row_of] * x64
            d = T[row_of, :, f].copy()                                 # [nnz, b, 4]: T[b][f_i]
            d[np.arange(ib.size), f] -= x64[:, None] * own
            np.add.at(gw, ib, rx)
            np.add.at(gv, ib, (rx[:, None, None] * d).reshape(ib.size, -1))
        return gw, gv

    def step(self, idx, rp, fields, x, lab):
        """One training step on tokens whose keys are rows `idx` of the state; returns the rows' residuals."""
        B = rp.size - 1
        loss = sigmoid_ref(self.forward(idx, rp, fields, x)) - np.asarray(lab, np.float64)
        gw, gv = self.gradients(idx, rp, fields, x, loss)
        gw, gv = gw / B, gv / B
        u = np.unique(idx)
        if self.opt == "ftrl":
            self.W[u], self.NW[u], self.ZW[u] = ftrl64(gw[u], self.W[u], self.NW[u], self.ZW[u])
            self.V[u], self.NV[u], self.ZV[u] = ftrl64(gv[u], self.V[u], self.NV[u], self.ZV[u])
        else:
            self.W[u] -= self.lr * gw[u]
            self.V[u] = self.V[u] - self.lr * gv[u]
        return loss
