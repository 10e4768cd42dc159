"""CPU restatement of sb_factor_append (stheno.jl_b200/csrc/append.cu, api.cu factor_splice): the Cholesky factor of
the stacked observations [x1; x2] from the factor L1 of the first ones, with the device's head / tail split.

    h = 128 floor(N1 / 128)      the head: L1's full block columns, kept verbatim
    r = N1 - h                   the tail: the old rows of L1's partial last block
    V = K21 L1^{-T}              over ALL old columns (N2 x N1)
    P = K22 + Sigma2 - V V'
    M = [L1[h:, h:]; V[:, h:]]   (r + N2) x r
    S = M M' + blockdiag(0_r, P) the Schur complement of the head in the joint matrix, order [tail; new]
    L = [[L1[:, :h], 0], [V[:, :h], chol(S)]]   with the rows of L1[:, :h] followed by those of V[:, :h]

Only tests/ import this module.
"""
from __future__ import annotations

import numpy as np
import scipy.linalg as sla

NB = 128


def noise_matrix(noise2, n2):
    """Sigma2 as a dense matrix: scalar, vector (diagonal) or matrix (its lower triangle is what the device reads)."""
    if np.ndim(noise2) == 0:
        return float(noise2) * np.eye(n2)
    if np.ndim(noise2) == 1:
        return np.diag(np.asarray(noise2, dtype=np.float64))
    A = np.tril(np.asarray(noise2, dtype=np.float64))
    return A + np.tril(A, -1).T


class AppendNotPosDef(np.linalg.LinAlgError):
    def __init__(self, info):
        super().__init__(f"not positive definite at pivot {info}")
        self.info = info


def append_factor(L1, K21, K22, noise2):
    """Joint lower Cholesky factor (N1 + N2 square).  On failure raises AppendNotPosDef with the 1-based pivot in
    the joint order (h + the pivot inside S), as sb_factor_append reports it."""
    L1 = np.asarray(L1, dtype=np.float64)
    K21 = np.asarray(K21, dtype=np.float64)
    n1, n2 = L1.shape[0], K21.shape[0]
    h = n1 // NB * NB
    r = n1 - h
    V = sla.solve_triangular(L1, K21.T, lower=True).T
    P = np.asarray(K22, dtype=np.float64) + noise_matrix(noise2, n2) - V @ V.T
    M = np.vstack([L1[h:, h:], V[:, h:]])
    S = M @ M.T
    S[r:, r:] += P
    LS, info = sla.lapack.dpotrf(S, lower=1, clean=1)
    if info != 0:
        raise AppendNotPosDef(h + info)
    L = np.zeros((n1 + n2, n1 + n2))
    L[:n1, :h] = L1[:, :h]
    L[n1:, :h] = V[:, :h]
    L[h:, h:] = LS
    return L
