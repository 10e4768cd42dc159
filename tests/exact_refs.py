"""Reference builders with exactly known answers, shared by test_exact_references.py (CPU checks of
the builders themselves) and test_gpu_exact.py (the device against them).

Exact factor.  `exact_factor(n)` is a lower triangle L* with 2^20 on the diagonal and random integers in
[-64, 64] on about a quarter of the sub-diagonal entries.  A = L* L*^T is formed EXACTLY in fp64: every
product L*[i,k] L*[j,k] is an integer of magnitude <= 2^40, and every partial sum of A[i,j] is an integer
of magnitude <= 2^40 + n 2^12 < 2^53 (n < 2^40), so any summation order, with or without FMA, gives the
same exact integer.  Positive-diagonal Cholesky factors are unique, so L* IS chol(A); and L* = 2^20 (I + E)
with |E| <= 2^-14 per entry, so L* and A have condition numbers close to 1 at the sizes used here.
  - logdet A = 2 n 20 ln 2.
  - Solves: X* has integer entries in [-16, 16] and Delta = A X*.  The row sums of |A| are below
    2^41 + n (2^27 + n 2^12) < 2^42 (n <= 4096), so every partial sum of A X* stays below 2^46 and Delta is
    exact; then A^{-1} Delta = X* exactly, and Delta^T A^{-1} Delta = sum(Delta * X*) is an exact integer.
  - rand: for an integer Z with |Z| <= 3, L* Z is exact (partial sums below 2^22 + n 2^8).

Exact low-rank model.  K = H C H^T + diag(d) with integer H (N x 8, entries in [-3, 3]), positive
integer C = diag(c) and d_i in {1, 2, 4}.  With integer y every quantity of logpdf's gradient and of the
posterior is a rational number, computed here exactly (fractions.Fraction) through Woodbury:
K^-1 = D^-1 - D^-1 H M^-1 H^T D^-1,  M = C^-1 + H^T D^-1 H  (8 x 8), O(N 64) work.
"""
from fractions import Fraction
import math

import numpy as np

DIAG_EXP = 20
DIAG = float(2 ** DIAG_EXP)


def exact_factor(n, seed, fill=0.25, amp=64):
    """L* (float64, integer valued): 2^20 on the diagonal, integers in [-amp, amp] on ~fill of the rest."""
    rng = np.random.default_rng(seed)
    L = np.tril(rng.integers(-amp, amp + 1, size=(n, n)), -1)
    L = L * (rng.random((n, n)) < fill)
    L = L.astype(np.float64)
    L[np.diag_indices(n)] = DIAG
    return L


def gram(L):
    """A = L L^T (exact for the integer factors above: see the module docstring)."""
    A = L @ L.T
    return np.tril(A) + np.tril(A, -1).T   # bit-symmetric whatever order the BLAS summed in


def exact_logdet(n):
    return 2.0 * n * DIAG_EXP * math.log(2.0)


def int_matrix(n, s, seed, amp):
    return np.random.default_rng(seed).integers(-amp, amp + 1, size=(n, s)).astype(np.float64)


def exact_quadratic(delta, x):
    """sum(delta * x) as an exact Python integer (delta, x integer valued)."""
    return sum(int(a) * int(b) for a, b in zip(np.ravel(delta), np.ravel(x)))


def exact_logpdf(n, quad):
    """-(n ln 2 pi + logdet + quad) / 2 to 30 digits (quad: exact integer)."""
    import mpmath
    with mpmath.workdps(40):
        v = -(n * mpmath.log(2 * mpmath.pi) + 2 * n * DIAG_EXP * mpmath.log(2) + mpmath.mpf(quad)) / 2
        return float(v)


def row_rel_error(L, Lref):
    """max_ij |L - Lref| / max_j |Lref[i, j]|."""
    return float(np.max(np.abs(L - Lref) / np.max(np.abs(Lref), axis=1, keepdims=True)))


def dpotf2_info(A):
    """LAPACK dpotf2 (lower, unblocked, left-looking), restated: the 1-based index of the first pivot
    that is not positive or is NaN (DISNAN), 0 if there is none."""
    A = np.array(A, dtype=np.float64)
    n = A.shape[0]
    with np.errstate(invalid="ignore", over="ignore"):
        for j in range(n):
            ajj = A[j, j] - A[j, :j] @ A[j, :j]
            if ajj <= 0.0 or np.isnan(ajj):
                return j + 1
            ajj = np.sqrt(ajj)
            A[j, j] = ajj
            if j + 1 < n:
                A[j + 1:, j] = (A[j + 1:, j] - A[j + 1:, :j] @ A[j, :j]) / ajj
    return 0


# -- exact low-rank model --------------------------------------------------------------------------

RANK = 8


def lowrank_model_data(n, seed):
    """H (n x 8, integers in [-3, 3]), c (8 positive integers), d (n values in {1, 2, 4}), y (integers)."""
    rng = np.random.default_rng(seed)
    H = rng.integers(-3, 4, size=(n, RANK))
    c = rng.integers(1, 4, size=RANK)
    d = 2 ** rng.integers(0, 3, size=n)
    y = rng.integers(-8, 9, size=n)
    return H, c, d, y


def _inv_exact(M):
    """Gauss-Jordan inverse of a small nonsingular matrix of Fractions."""
    m = len(M)
    a = [list(row) + [Fraction(int(i == j)) for j in range(m)] for i, row in enumerate(M)]
    for col in range(m):
        piv = next(r for r in range(col, m) if a[r][col] != 0)
        a[col], a[piv] = a[piv], a[col]
        p = a[col][col]
        a[col] = [v / p for v in a[col]]
        for r in range(m):
            if r != col and a[r][col] != 0:
                f = a[r][col]
                a[r] = [vr - f * vc for vr, vc in zip(a[r], a[col])]
    return [row[m:] for row in a]


class Woodbury:
    """Exact (rational) alpha, gradients and posterior of K = H diag(c) H^T + diag(d)."""

    def __init__(self, H, c, d, y):
        self.H = [[int(v) for v in row] for row in H]
        self.c = [int(v) for v in c]
        self.d = [int(v) for v in d]
        n, r = len(self.H), len(self.c)
        hd = [[Fraction(v, di) for v in row] for row, di in zip(self.H, self.d)]          # D^-1 H
        G = [[sum((hd[i][a] * self.H[i][b] for i in range(n)), Fraction(0)) for b in range(r)] for a in range(r)]
        M = [[G[a][b] + (Fraction(1, self.c[a]) if a == b else 0) for b in range(r)] for a in range(r)]
        self.Minv = _inv_exact(M)
        self.G = G
        # H^T K^-1 H = G - G M^-1 G
        GM = [[sum((G[a][k] * self.Minv[k][b] for k in range(r)), Fraction(0)) for b in range(r)] for a in range(r)]
        self.HKH = [[G[a][b] - sum((GM[a][k] * G[k][b] for k in range(r)), Fraction(0)) for b in range(r)]
                    for a in range(r)]
        self.hd = hd
        self.alpha, self.alpha_mag = self.solve([int(v) for v in y])

    def solve(self, v):
        """K^-1 v (v: integers), and the magnitudes |v_i| / d_i + sum_a |(D^-1 H)_ia w_a| of its terms."""
        n, r = len(self.H), len(self.c)
        u = [sum((self.hd[i][a] * v[i] for i in range(n)), Fraction(0)) for a in range(r)]
        w = [sum((self.Minv[a][b] * u[b] for b in range(r)), Fraction(0)) for a in range(r)]
        x = [Fraction(v[i], self.d[i]) - sum((self.hd[i][a] * w[a] for a in range(r)), Fraction(0))
             for i in range(n)]
        mag = [abs(Fraction(v[i], self.d[i])) + sum((abs(self.hd[i][a] * w[a]) for a in range(r)), Fraction(0))
               for i in range(n)]
        return x, mag

    def kinv_diag(self):
        r = len(self.c)
        out = []
        for i, hi in enumerate(self.hd):
            q = sum((hi[a] * self.Minv[a][b] * hi[b] for a in range(r) for b in range(r)), Fraction(0))
            out.append(Fraction(1, self.d[i]) - q)
        return out

    def grad_c(self):
        """d logpdf / d c_r = 1/2 ((h_r^T alpha)^2 - h_r^T K^-1 h_r)  and the magnitudes of its two terms."""
        n = len(self.H)
        ha = [sum((self.H[i][a] * self.alpha[i] for i in range(n)), Fraction(0)) for a in range(len(self.c))]
        g = [(ha[a] ** 2 - self.HKH[a][a]) / 2 for a in range(len(self.c))]
        mag = [(ha[a] ** 2 + abs(self.HKH[a][a])) / 2 for a in range(len(self.c))]
        return g, mag

    def grad_noise(self):
        """d logpdf / d d_i = 1/2 (alpha_i^2 - (K^-1)_ii)  and the magnitudes of its two terms."""
        kd = self.kinv_diag()
        return ([(a * a - k) / 2 for a, k in zip(self.alpha, kd)],
                [(a * a + abs(k)) / 2 for a, k in zip(self.alpha, kd)])

    def predict(self, Hs):
        """Posterior mean and variance at test rows Hs (rows of H), with the magnitudes of their terms."""
        n, r = len(self.H), len(self.c)
        ha = [sum((self.H[i][a] * self.alpha[i] for i in range(n)), Fraction(0)) for a in range(r)]
        absha = [sum((abs(self.H[i][a] * self.alpha[i]) for i in range(n)), Fraction(0)) for a in range(r)]
        m, v, mm, vm = [], [], [], []
        for hs in Hs:
            ch = [self.c[a] * int(hs[a]) for a in range(r)]
            m.append(sum((ch[a] * ha[a] for a in range(r)), Fraction(0)))
            mm.append(sum((abs(ch[a]) * absha[a] for a in range(r)), Fraction(0)))
            prior = sum(ch[a] * int(hs[a]) for a in range(r))
            q = sum((ch[a] * self.HKH[a][b] * ch[b] for a in range(r) for b in range(r)), Fraction(0))
            v.append(prior - q)
            vm.append(abs(prior) + abs(q))
        return m, v, mm, vm


def lowrank_dense(H, c, d):
    """K as a float64 matrix (exact: integer entries of magnitude <= 8 * 3 * 9 + 4)."""
    H = np.asarray(H, dtype=np.float64)
    return (H * np.asarray(c, dtype=np.float64)) @ H.T + np.diag(np.asarray(d, dtype=np.float64))


def lowrank_cond_bound(H, c, d):
    """Upper bound on cond(K): lambda_min >= min d, lambda_max <= max d + lambda_max(C^1/2 H^T H C^1/2)."""
    H = np.asarray(H, dtype=np.float64)
    s = np.sqrt(np.asarray(c, dtype=np.float64))
    inner = (H * s).T @ (H * s)
    return (float(np.max(d)) + float(np.linalg.eigvalsh(inner)[-1])) / float(np.min(d))
