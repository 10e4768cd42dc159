"""CPU checks of the exact references in exact_refs.py, so that test_gpu_exact.py compares the device with
references that are themselves verified: exact integer arithmetic, Woodbury against a dense
high-precision inverse, the expected `info` of non-finite input, and the power-of-two scaling identity."""
from fractions import Fraction

import numpy as np
import pytest
import scipy.linalg as sla

import exact_refs as er


@pytest.mark.parametrize("n", [1, 37, 200])
def test_gram_solve_and_quadratic_form_are_exact(n):
    L = er.exact_factor(n, seed=n)
    A = er.gram(L)
    Li = [[int(v) for v in row] for row in L]
    Ai = [[sum(Li[i][k] * Li[j][k] for k in range(n)) for j in range(n)] for i in range(n)]
    assert all(A[i, j] == Ai[i][j] for i in range(n) for j in range(n))
    X = er.int_matrix(n, 3, seed=7, amp=16)
    D = A @ X
    for s in range(3):
        col = [sum(Ai[i][j] * int(X[j, s]) for j in range(n)) for i in range(n)]
        assert all(D[i, s] == col[i] for i in range(n))
        q = er.exact_quadratic(D[:, s], X[:, s])
        assert q == sum(col[i] * int(X[i, s]) for i in range(n))
    Z = er.int_matrix(n, 2, seed=8, amp=3)
    LZ = L @ Z
    assert all(LZ[i, s] == sum(Li[i][k] * int(Z[k, s]) for k in range(n)) for i in range(n) for s in range(2))
    # the factor is the exact Cholesky factor: LAPACK recovers it to rounding
    assert er.row_rel_error(sla.cholesky(A, lower=True), L) <= 2.0 ** -50


def test_exact_logpdf_matches_scipy():
    n = 150
    L = er.exact_factor(n, seed=3)
    A = er.gram(L)
    X = er.int_matrix(n, 1, seed=4, amp=16)[:, 0]
    d = A @ X
    lp = er.exact_logpdf(n, er.exact_quadratic(d, X))
    c = sla.cho_factor(A, lower=True)
    ref = -(n * np.log(2 * np.pi) + 2 * np.sum(np.log(np.diag(c[0]))) + d @ sla.cho_solve(c, d)) / 2
    assert abs(lp - ref) <= 1e-14 * abs(lp)
    assert abs(er.exact_logdet(n) - 2 * np.sum(np.log(np.diag(c[0])))) <= 1e-14 * er.exact_logdet(n)


def _mp_dense_inverse(K):
    import mpmath
    with mpmath.workdps(50):
        return mpmath.inverse(mpmath.matrix([[int(v) for v in row] for row in K]))


def test_woodbury_against_dense_high_precision_inverse():
    import mpmath
    n = 60
    H, c, d, y = er.lowrank_model_data(n, seed=5)
    K = er.lowrank_dense(H, c, d)
    w = er.Woodbury(H, c, d, y)
    with mpmath.workdps(50):
        Ki = _mp_dense_inverse(K)
        alpha = Ki * mpmath.matrix([int(v) for v in y])
        tol = mpmath.mpf(10) ** -40
        for i in range(n):
            assert abs(mpmath.mpf(w.alpha[i].numerator) / w.alpha[i].denominator - alpha[i]) < tol
        kd = w.kinv_diag()
        for i in range(n):
            assert abs(mpmath.mpf(kd[i].numerator) / kd[i].denominator - Ki[i, i]) < tol
        g, _ = w.grad_c()
        for r in range(er.RANK):
            h = mpmath.matrix([int(v) for v in H[:, r]])
            ref = ((h.T * alpha)[0] ** 2 - (h.T * Ki * h)[0]) / 2
            assert abs(mpmath.mpf(g[r].numerator) / g[r].denominator - ref) < tol * (1 + abs(ref))
        # posterior at training rows 3 and 17: k*^T alpha and k** - k*^T K^-1 k*
        m, v, _, _ = w.predict([H[3], H[17]])
        Kp = (np.asarray(H, dtype=np.float64) * c) @ np.asarray(H, dtype=np.float64).T
        for j, i in enumerate((3, 17)):
            ks = mpmath.matrix([int(x) for x in Kp[i]])
            mref = (ks.T * alpha)[0]
            vref = int(Kp[i, i]) - (ks.T * Ki * ks)[0]
            assert abs(mpmath.mpf(m[j].numerator) / m[j].denominator - mref) < tol * (1 + abs(mref))
            assert abs(mpmath.mpf(v[j].numerator) / v[j].denominator - vref) < tol * (1 + abs(vref))


def test_lowrank_condition_bound():
    """The bound behind the rtol 1e-9 of the gradient / posterior tests: cond(K) <= 5e5 at N <= 2177,
    so an fp64 solve is good to cond * u ~ 6e-11."""
    for n in (1300, 2177):
        H, c, d, _ = er.lowrank_model_data(n, seed=n)
        b = er.lowrank_cond_bound(H, c, d)
        assert b <= 5e5, b
        if n == 1300:
            assert np.linalg.cond(er.lowrank_dense(H, c, d)) <= b * (1 + 1e-9)


@pytest.mark.parametrize("bad", [np.nan, np.inf, 1e300])
@pytest.mark.parametrize("i,j", [(150, 3), (299, 120), (40, 39), (200, 0)])
def test_nonfinite_info_is_row_plus_one(bad, i, j):
    """A NaN, +Inf or 1e300 at A[i, j] (i > j, both triangles) makes pivot i the first failure: pivots
    j+1 .. i-1 never read row i, and pivot i subtracts L[i, j]^2 (NaN, or Inf - Inf / -Inf; 1e300 / 2^20
    squared overflows)."""
    n = 300
    A = er.gram(er.exact_factor(n, seed=11))
    assert er.dpotf2_info(A) == 0
    A[i, j] = A[j, i] = bad
    assert er.dpotf2_info(A) == i + 1


def test_negative_pivot_info():
    n = 260
    L = er.exact_factor(n, seed=12)
    A = er.gram(L)
    for k in (0, 1, 127, 128, 259):
        B = A.copy()
        B[k, k] -= L[k, k] ** 2 + 2.0 ** 30
        assert er.dpotf2_info(B) == k + 1
    B = A.copy()
    for k in (200, 130):
        B[k, k] -= L[k, k] ** 2 + 2.0 ** 30
    assert er.dpotf2_info(B) == 131


def test_power_of_two_scaling_identity():
    """chol(D A D) = D chol(A) for D = diag(2^e): in IEEE arithmetic every rounding commutes with a
    power-of-two scale, so LAPACK's two factors agree bit for bit."""
    n = 300
    A = er.gram(er.exact_factor(n, seed=13))
    e = np.random.default_rng(14).integers(-30, 31, n)
    s = np.ldexp(1.0, e)
    L = sla.cholesky(A, lower=True)
    Ls = sla.cholesky(A * s[:, None] * s[None, :], lower=True)
    assert np.array_equal(Ls, L * s[:, None])
    # and the exact reference survives the scale: D L* is the factor of D A D
    np.testing.assert_array_equal(Ls, er.exact_factor(n, seed=13) * s[:, None])


def test_fraction_inverse():
    M = [[Fraction(4), Fraction(1)], [Fraction(2), Fraction(3)]]
    Mi = er._inv_exact(M)
    assert Mi == [[Fraction(3, 10), Fraction(-1, 10)], [Fraction(-1, 5), Fraction(2, 5)]]
