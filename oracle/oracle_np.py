"""TEST INFRASTRUCTURE. Independent float64 numpy formulation of single-head attention and its
gradients (matrix form, not row-at-a-time) used ONLY to pin oracle/network_oracle.c
(tests/test_oracle.py). Math per the reference's README.md:41-46 and Network.swift:134-402."""
import numpy as np


def attention_f64(Q, K, V, dO=None):
    Q, K, V = (np.asarray(x, np.float64) for x in (Q, K, V))
    D = Q.shape[1]
    S = (Q @ K.T) / np.sqrt(D)
    m = S.max(axis=1, keepdims=True)
    E = np.exp(S - m)
    lsum = E.sum(axis=1, keepdims=True)
    P = E / lsum
    out = {"O": P @ V, "L": (m + np.log(lsum))[:, 0]}
    if dO is not None:
        dO = np.asarray(dO, np.float64)
        Dt = (dO * out["O"]).sum(axis=1)
        dP = dO @ V.T
        dS = P * (dP - Dt[:, None]) / np.sqrt(D)
        out.update(D=Dt, dV=P.T @ dO, dK=dS.T @ Q, dQ=dS @ K)
    return out
