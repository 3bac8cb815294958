"""TEST INFRASTRUCTURE.  The causal-mask reference for tests/test_causal.py.

The mask is aligned bottom-right: with delta = C - R, query row i sees key j iff j <= i + delta.  Rows that see no key
(only when R > C, i < R - C) have O = 0, L = +inf, D = 0, dQ = 0 and add nothing to dK / dV.

`attention_f64` is a float64 matrix-form formulation (query rows in chunks, so the 4096 x 4096 shapes stay small in
memory); without the mask it is oracle/oracle_np.py's formulation.  `Network(..., causal=True)` exposes it with the
interface of oracle.Network (same seeded inputs, float32 results), so tests/attention_harness.py runs unchanged;
with causal=False it is oracle.Network itself.  tests/test_causal.py pins the masked formulation row by row against
the C oracle (every row of a causal problem is an unmasked problem over its visible keys), against PyTorch's
scaled_dot_product_attention with an explicit mask, and by finite differences of the masked loss."""
import numpy as np

import oracle


def causal_mask(R, C):
    """[R, C] boolean: True where query row i sees key j (j <= i + C - R)."""
    return np.arange(C)[None, :] <= np.arange(R)[:, None] + (C - R)


def attention_f64(Q, K, V, dO=None, causal=False, chunk=512):
    """O, L (natural-log units) and, with dO, D = rowsum(dO * O), dQ, dK, dV -- all float64."""
    Q, K, V = (np.asarray(x, np.float64) for x in (Q, K, V))
    R, D = Q.shape
    C = K.shape[0]
    scale = 1.0 / np.sqrt(D)
    out = {"O": np.zeros((R, D)), "L": np.zeros(R)}
    if dO is not None:
        dO = np.asarray(dO, np.float64)
        out.update(D=np.zeros(R), dQ=np.zeros((R, D)), dK=np.zeros((C, D)), dV=np.zeros((C, D)))
    for i0 in range(0, R, chunk):
        i1 = min(R, i0 + chunk)
        S = (Q[i0:i1] @ K.T) * scale
        if causal:
            S = np.where(np.arange(C)[None, :] <= np.arange(i0, i1)[:, None] + (C - R), S, -np.inf)
        m = S.max(axis=1, keepdims=True)
        empty = ~np.isfinite(m[:, 0])                 # every key masked
        m = np.where(np.isfinite(m), m, 0.0)
        E = np.exp(S - m)
        lsum = E.sum(axis=1, keepdims=True)
        P = E / np.where(lsum > 0, lsum, 1.0)
        O = P @ V
        out["O"][i0:i1] = O
        out["L"][i0:i1] = np.where(empty, np.inf, (m + np.log(np.where(lsum > 0, lsum, 1.0)))[:, 0])
        if dO is not None:
            g = dO[i0:i1]
            Dt = (g * O).sum(axis=1)
            dS = P * ((g @ V.T) - Dt[:, None]) * scale
            out["D"][i0:i1] = Dt
            out["dQ"][i0:i1] = dS @ K
            out["dK"] += dS.T @ Q[i0:i1]
            out["dV"] += P.T @ g
    return out


class Network(oracle.Network):
    """oracle.Network with an optional causal mask: Network(R, C, D, seed=..., threads=..., causal=False)."""

    def __init__(self, rowDimension, columnDimension, headDimension, seed=0, threads=1, causal=False):
        super().__init__(rowDimension, columnDimension, headDimension, seed=seed, threads=threads)
        self.causal = bool(causal)
        self._cache = None

    def _masked(self):
        key = (self.Q, self.K, self.V, self.dO)
        if self._cache is None or any(a is not b for a, b in zip(self._cache[0], key)):
            self._cache = (key, attention_f64(self.Q, self.K, self.V, self.dO, causal=True))
        return self._cache[1]

    def _f32(self, name):
        return np.ascontiguousarray(self._masked()[name], np.float32)

    def inferenceAttention(self, with_L=False):
        if not self.causal:
            return super().inferenceAttention(with_L)
        return (self._f32("O"), self._f32("L")) if with_L else self._f32("O")

    def createDTerms(self):
        return self._f32("D") if self.causal else super().createDTerms()

    def derivativeV(self):
        return self._f32("dV") if self.causal else super().derivativeV()

    def derivativeK(self):
        return self._f32("dK") if self.causal else super().derivativeK()

    def derivativeQ(self):
        return self._f32("dQ") if self.causal else super().derivativeQ()

    def loss(self):
        """sum(dO * O) (Network.swift's loss) under the mask, in float64."""
        if not self.causal:
            return super().loss()
        return float((np.asarray(self.dO, np.float64) * self._masked()["O"]).sum())
