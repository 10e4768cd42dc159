"""The Cholesky factor, the triangular sweeps and the logpdf gradient against EXACT references
(exact_refs.py), at every remainder of the 4-block outer step, on both trailing-update paths.

Any SPD matrix A is factored through the public API as the DENSE OBSERVATION NOISE of a prior whose
covariance is exactly zero (GP(0 * ConstantKernel(1))): the assembly adds A to a packed matrix of zeros.
Every test runs under `trailing` = 0 (fp64 DMMA) and 1 (int8 Ozaki, which runs only for nblk > 8 block
columns) and asserts which path actually ran through the context's int8 op counter.
"""
import functools
import os

import numpy as np
import pytest
import scipy.linalg as sla

import exact_refs as er

pytestmark = pytest.mark.gpu

NB, OUTER_BLOCKS = 128, 4
# the context's trailing path when the tests start: fp64 DMMA unless SB_TRAILING=ozaki (read by sb_ctx_create)
INITIAL_TRAILING = 1 if os.environ.get("SB_TRAILING") == "ozaki" else 0
SIZES = [1, 127, 128, 129, 511, 513, 640, 1000, 1025, 1153, 1300, 1536, 1665, 2049, 2177]


@pytest.fixture(params=[0, 1], ids=["dmma", "ozaki"])
def trailing(request, sb):
    """Route the default context's trailing updates through the DMMA (0) or the int8 Ozaki (1) kernel."""
    ctx = sb.default_context()
    ctx.set_option("trailing", request.param)
    try:
        yield request.param
    finally:
        ctx.set_option("trailing", INITIAL_TRAILING)


def nblk(n):
    return (n + NB - 1) // NB


def check_path(sb, trailing, n):
    """The int8 Ozaki driver runs only with trailing = 1 and more than 2 outer steps of block columns."""
    ops = sb.default_context().timings()["trailing_int8_ops"]
    ozaki = trailing == 1 and nblk(n) > 2 * OUTER_BLOCKS
    assert (ops > 0) if ozaki else (ops == 0), (trailing, n, ops)
    print(f"N={n} nblk={nblk(n)} trailing={trailing}: {'int8 Ozaki' if ozaki else 'serial DMMA'} path")


def zero_prior(sb):
    return sb.gppp(lambda GP: dict(f=GP(0.0 * sb.ConstantKernel(1.0))))


def dense_fx(sb, A):
    n = A.shape[0]
    return zero_prior(sb)(sb.GPPPInput("f", np.arange(n, dtype=np.float64)), A)


def factor(sb, A, trailing):
    """Device factor of A (dense noise of the zero prior) and the FiniteGP that owns it."""
    fx = dense_fx(sb, A)
    sb.default_context().timings(reset=True)
    L = fx.factor().to_dense_L()
    check_path(sb, trailing, A.shape[0])
    return fx, L


@functools.lru_cache(maxsize=None)
def problem(n):
    L = er.exact_factor(n, seed=1000 + n)
    return L, er.gram(L)


def calibrated_tol(A, Lref):
    """Forward-error bound of a correct fp64 Cholesky on this matrix: 8x SciPy's error against the exact
    factor, floored at 2^-50 relative to the row's max (SciPy is usually exact on these integer matrices:
    every intermediate is an integer or an exact division by a power of two)."""
    return max(8.0 * er.row_rel_error(sla.cholesky(A, lower=True), Lref), 2.0 ** -50)


# -- 1. the exact factor, its solves and its samples ---------------------------------------------

@pytest.mark.parametrize("n", SIZES)
def test_exact_factor_solves_and_samples(sb, trailing, n):
    """L, logdet, alpha, logpdf (S = 1, 7, 8, 9, 17 columns: the vector sweeps run in groups of 8) and
    rand (S = 1, 9) against exact values.  The factor tolerance is calibrated: on these matrices SciPy's
    cholesky is exact (error 0), so the bound is the 2^-50 floor relative to the row's max."""
    Ls, A = problem(n)
    x = np.arange(min(n, 64), dtype=np.float64)
    assert np.all(sb.cov(zero_prior(sb), sb.GPPPInput("f", x)) == 0.0)
    fx, L = factor(sb, A, trailing)
    tol = calibrated_tol(A, Ls)
    err = er.row_rel_error(L, Ls)
    assert err <= tol, (err, tol)
    assert np.all(np.triu(L, 1) == 0.0)
    ld = fx.factor().logdet()
    assert abs(ld - er.exact_logdet(n)) <= 1e-14 * er.exact_logdet(n), (ld, er.exact_logdet(n))

    X = er.int_matrix(n, 17, seed=n, amp=16)
    D = A @ X
    alpha = sb.posterior(fx, D[:, 0]).alpha
    assert np.max(np.abs(alpha - X[:, 0])) <= 1e-12 * np.max(np.abs(X[:, 0])), np.max(np.abs(alpha - X[:, 0]))
    exact = np.array([er.exact_logpdf(n, er.exact_quadratic(D[:, s], X[:, s])) for s in range(17)])
    for S in (1, 7, 8, 9, 17):
        lp = sb.logpdf(fx, D[:, 0] if S == 1 else D[:, :S])
        np.testing.assert_allclose(lp, exact[0] if S == 1 else exact[:S], rtol=1e-13, atol=0, err_msg=f"S={S}")

    # rand = L Z with the device's own L: its distance from the exact L* Z is the factor's error times |Z|
    # plus the rounding of the product
    Z = er.int_matrix(n, 9, seed=n + 1, amp=3)
    LZ = Ls @ Z
    for S in (1, 9):
        got = sb.rand(fx, Z[:, 0] if S == 1 else Z[:, :S]).reshape(n, S)
        bound = (np.abs(L - Ls) + 2.0 ** -50 * np.abs(Ls)) @ np.abs(Z[:, :S])
        assert np.all(np.abs(got - LZ[:, :S]) <= bound), (S, np.max(np.abs(got - LZ[:, :S]) - bound))


# -- 2. metamorphic and structural checks ---------------------------------------------------------

@pytest.mark.parametrize("n", [640, 1300, 2177])
def test_power_of_two_scaling_commutes(sb, trailing, n):
    """chol(D A D) = D chol(A) for D = diag(2^e), e in [-30, 30] (a 2^120 range of row scales): every fp64
    rounding commutes with a power-of-two scale, and so do the Ozaki digit planes -- per-row scales in the
    trailing updates, and in the panel solve per-row scales of the column-equilibrated operands A21 E^-1 and
    inv(L_512) E, E = diag(2^ilogb(L_kk)), which D leaves unchanged.  At most 2 ulp per entry on both paths;
    prints whether the two factors were bit-identical."""
    Ls, A = problem(n)
    e = np.random.default_rng(n + 2).integers(-30, 31, n)
    s = np.ldexp(1.0, e)
    _, L = factor(sb, A, trailing)
    _, Ld = factor(sb, A * s[:, None] * s[None, :], trailing)
    ref = L * s[:, None]                                   # exact: a power-of-two scale
    nz = ref != 0.0
    ulps = np.abs(Ld[nz] - ref[nz]) / np.spacing(np.abs(ref[nz]))
    print(f"N={n} trailing={trailing}: max {ulps.max():.3g} ulp, bit-identical: {bool(np.array_equal(Ld, ref))}")
    assert np.array_equal(Ld == 0.0, ref == 0.0)
    assert ulps.max() <= 2.0


@pytest.mark.parametrize("n", [1300, 2177])
def test_dynamic_range_inside_rows(sb, trailing, n):
    """The sub-diagonal parts of a few columns of L* scaled by 2^-40: the rows under them span 2^40 in
    magnitude, which the Ozaki digit planes (per-row scale, 56 bits) cut short.  DESIGN.md bounds the
    truncation at ~5e-15 of max|row_i| max|row_j|, which is below the forward error of LAPACK on the same
    matrix.  (The diagonal is left alone: a 2^-20 pivot under integer entries would make A singular in fp64.)"""
    Ls, _ = problem(n)
    Ls = Ls.copy()
    for c in (3, 200, 515, 700, n - 200):
        Ls[c + 1:, c] *= 2.0 ** -40
    A = er.gram(Ls)   # no longer exact in fp64: the calibration measures LAPACK on the rounded matrix
    _, L = factor(sb, A, trailing)
    tol = calibrated_tol(A, Ls)
    err = er.row_rel_error(L, Ls)
    assert err <= tol, (err, tol)


@pytest.mark.parametrize("n,cut", [(1300, 700), (2177, 1100)])
def test_block_diagonal_gives_exact_zeros(sb, trailing, n, cut):
    """A block diagonal with the boundary off the 128 grid: the factor's off-block entries are exactly 0.0
    (on the Ozaki path the all-zero rows of a panel take the zero-row sentinel of the digit planes)."""
    Ls, _ = problem(n)
    Ls = Ls.copy()
    Ls[cut:, :cut] = 0.0
    A = er.gram(Ls)
    _, L = factor(sb, A, trailing)
    assert np.all(L[cut:, :cut] == 0.0), np.count_nonzero(L[cut:, :cut])
    assert er.row_rel_error(L, Ls) <= calibrated_tol(A, Ls)


# -- 3. info of a failed factorisation ------------------------------------------------------------

def bad_pivots(n):
    last = (nblk(n) - 1) // OUTER_BLOCKS * OUTER_BLOCKS * NB   # first row of the last outer step
    return sorted({k for k in (0, 1, 127, 128, 511, 512, 513, last, n - 1) if k < n})


@pytest.mark.parametrize("n", [640, 1300])
def test_info_is_first_failing_pivot(sb, trailing, n):
    """A[k, k] -> A[k, k] - L*[k, k]^2 - 2^30 makes pivot k exactly -2^30: info must be k + 1 (LAPACK's
    1-based first failing pivot); with two bad pivots the smaller one.  Then the unmodified matrix on the
    same context factors and matches the exact factor: no per-factor state leaks between factorisations."""
    Ls, A = problem(n)
    for k in bad_pivots(n):
        B = A.copy()
        B[k, k] -= Ls[k, k] ** 2 + 2.0 ** 30
        with pytest.raises(sb.PosDefException) as ei:
            dense_fx(sb, B).factor()
        assert ei.value.info == k + 1, (k, ei.value.info)
    B = A.copy()
    for k in (n - 1, 130):
        B[k, k] -= Ls[k, k] ** 2 + 2.0 ** 30
    with pytest.raises(sb.PosDefException) as ei:
        dense_fx(sb, B).factor()
    assert ei.value.info == 131
    _, L = factor(sb, A, trailing)
    assert er.row_rel_error(L, Ls) <= calibrated_tol(A, Ls)


# -- 4. non-finite input ----------------------------------------------------------------------------

@pytest.mark.parametrize("bad", [np.nan, np.inf, 1e300], ids=["nan", "inf", "huge"])
def test_nonfinite_entry_is_reported_at_its_row(sb, trailing, bad):
    """A NaN, +Inf or a finite 1e300 at A[i, j], i > j: pivot i is the first to become NaN or -Inf (pivots
    j+1 .. i-1 never read row i), so info = i + 1 on both paths.  Rows i lie under the 512-wide diagonal
    block of their outer step (the Ozaki panel solve and trailing update) and inside it (DMMA products)."""
    n = 1300
    Ls, A = problem(n)
    for i, j in [(900, 100), (1299, 511), (1200, 600), (300, 100), (1023, 700)]:
        B = A.copy()
        B[i, j] = B[j, i] = bad
        with pytest.raises(sb.PosDefException) as ei:
            dense_fx(sb, B).factor()
        assert ei.value.info == i + 1, (i, j, ei.value.info)
    _, L = factor(sb, A, trailing)
    assert er.row_rel_error(L, Ls) <= calibrated_tol(A, Ls)


def test_posterior_at_nan_input(sb, trailing):
    """Posterior mean and variance at a NaN test input are NaN; the other test points are unaffected."""
    rng = np.random.default_rng(5)
    n = 1300
    x = rng.uniform(0, 40, n)
    y = np.sin(x) + 0.3 * rng.standard_normal(n)
    xs = rng.uniform(0, 40, 300)
    f = sb.gppp(lambda GP: dict(f=GP(sb.SEKernel())))
    fx = f(sb.GPPPInput("f", x), 0.1)
    sb.default_context().timings(reset=True)
    post = sb.posterior(fx, y)
    check_path(sb, trailing, n)
    m0, v0 = sb.mean_and_var(post, sb.GPPPInput("f", xs))
    xn = xs.copy()
    xn[[0, 131, 299]] = np.nan
    m, v = sb.mean_and_var(post, sb.GPPPInput("f", xn))
    ok = ~np.isnan(xn)
    assert np.all(np.isnan(m[~ok])) and np.all(np.isnan(v[~ok])), (m[~ok], v[~ok])
    np.testing.assert_allclose(m[ok], m0[ok], rtol=1e-13, atol=1e-15)
    np.testing.assert_allclose(v[ok], v0[ok], rtol=1e-12, atol=1e-15)


# -- 5. gradients and posterior against an exact low-rank model -------------------------------------

@functools.lru_cache(maxsize=None)
def lowrank(n):
    H, c, d, y = er.lowrank_model_data(n, seed=n)
    return H, c, d, y, er.Woodbury(H, c, d, y)


def lowrank_gppp(sb, H, c):
    """f = sum_r h_r * GP(c_r * ConstantKernel(1)) over inputs x = 0 .. N-1 (function scaling)."""
    def build(GP):
        atoms = [GP(float(cr) * sb.ConstantKernel(1.0)) for cr in c]
        f = None
        for r, a in enumerate(atoms):
            col = H[:, r].astype(np.float64)
            term = (lambda x, col=col: col[int(x)]) * a
            f = term if f is None else f + term
        return dict(f=f, **{f"a{r}": a for r, a in enumerate(atoms)})
    return sb.gppp(build)


def _close(got, exact, mag, rtol, what):
    exact = np.array([float(v) for v in exact])
    mag = np.array([float(v) for v in mag])
    err = np.abs(np.asarray(got) - exact)
    assert np.all(err <= rtol * mag), (what, float(np.max(err / mag)))


@pytest.mark.parametrize("n", [1300, 2177])
def test_lowrank_gradients_and_posterior(sb, trailing, n):
    """K = sum_{r<8} c_r h_r h_r^T + diag(d): 8 terms per block (> MAX_TERMS, so assembly and gradient
    reduction take their accumulate pass), against exact rational Woodbury references.  lambda_min(K) >= 1
    and lambda_max(K) <= 5e5 (test_exact_references checks the bound), so fp64 solves are good to
    cond(K) u ~ 6e-11 of the magnitudes of each formula's terms; rtol 1e-9 leaves a 16x margin."""
    H, c, d, y, wb = lowrank(n)
    fs = lowrank_gppp(sb, H, c)
    x = np.arange(n, dtype=np.float64)
    fx = fs(sb.GPPPInput("f", x), d.astype(np.float64))
    yf = y.astype(np.float64)
    sb.default_context().timings(reset=True)
    gr = sb.grad_logpdf(fx, yf)
    check_path(sb, trailing, n)
    post = sb.posterior(fx, yf)
    _close(post.alpha, wb.alpha, wb.alpha_mag, 1e-9, "alpha")
    g, mag = wb.grad_c()
    got = [gr.for_atom(fs.fs[f"a{r}"], 0)["dcoeff"] for r in range(er.RANK)]
    _close(got, g, mag, 1e-9, "dc")
    gn, magn = wb.grad_noise()
    _close(gr.noise, gn, magn, 1e-9, "dnoise")
    for ns in (1, 129, 300):
        idx = (np.arange(ns) * 7 + 3) % n
        m, v = sb.mean_and_var(post, sb.GPPPInput("f", idx.astype(np.float64)))
        me, ve, mm, vm = wb.predict(H[idx])
        _close(m, me, mm, 1e-9, f"mean N*={ns}")
        _close(v, ve, vm, 1e-9, f"var N*={ns}")


# -- 5b. a real kernel: SE + Matern-5/2 + White, closed-form derivatives -----------------------------

def _se_m52_white(x, th, dtype):
    """K, and dK / d(multiplier) and dK / d(log input scale) of each component (kappa_and_dlogs restated)."""
    v1, l1, v2, l2, w, s2 = th
    x = np.asarray(x, dtype=dtype)
    r = np.abs(x[:, None] - x[None, :])
    d2 = (r / dtype(l1)) ** 2
    k1 = np.exp(-d2 / 2)
    s = np.sqrt(dtype(5)) * r / dtype(l2)
    e = np.exp(-s)
    k2 = (1 + s + s * s / 3) * e
    dk2 = -(s * s / 3) * (1 + s) * e
    kw = (x[:, None] == x[None, :]).astype(dtype)
    K = dtype(v1) * k1 + dtype(v2) * k2 + dtype(w) * kw + dtype(s2) * np.eye(len(x), dtype=dtype)
    return K, dict(c1=k1, s1=dtype(v1) * (-d2 * k1), c2=k2, s2=dtype(v2) * dk2, cw=kw)


def _grad_terms(Kinv, alpha, dK):
    """1/2 (alpha' dK alpha - sum(K^-1 * dK)) and the magnitudes of its two terms."""
    a = float(alpha @ dK @ alpha)
    t = float(np.sum(Kinv * dK))
    return (a - t) / 2, (abs(a) + abs(t)) / 2


def test_real_kernel_gradients(sb, trailing):
    """d logpdf / d (variances, log input scales, white multiplier, noise) of SE + Matern-5/2 + White at
    N = 2177 against 1/2 (alpha' dK alpha - tr(K^-1 dK)) with closed-form dK and SciPy's cho_solve.
    cond(K) is ~1e3 (lambda_min >= w + s2 = 0.15), so fp64 is good to ~1e-13 of each formula's terms; the
    reference is recomputed in np.longdouble (kernel matrix, derivatives and the alpha-dependent term, alpha
    refined once with a longdouble residual) and must agree with the fp64 one to 1e-12, 100x inside the
    rtol 1e-10 the device is held to."""
    rng = np.random.default_rng(2177)
    n = 2177
    x = np.sort(rng.uniform(0, n / 32, n))
    y = np.sin(x) + 0.3 * rng.standard_normal(n)
    th = (1.3, 0.8, 0.6, 1.7, 0.05, 0.1)
    fs = sb.gppp(lambda GP: dict(f=GP(th[0] * sb.with_lengthscale(sb.SEKernel(), th[1])
                                      + th[2] * sb.with_lengthscale(sb.Matern52Kernel(), th[3])
                                      + th[4] * sb.WhiteKernel())))
    sb.default_context().timings(reset=True)
    gr = sb.grad_logpdf(fs(sb.GPPPInput("f", x), th[5]), y)
    check_path(sb, trailing, n)
    atom = fs.fs["f"]
    got = dict(c1=gr.for_atom(atom, 0)["dcoeff"], s1=gr.for_atom(atom, 0)["dlogscale"],
               c2=gr.for_atom(atom, 1)["dcoeff"], s2=gr.for_atom(atom, 1)["dlogscale"],
               cw=gr.for_atom(atom, 2)["dcoeff"], noise=gr.noise)

    K, dK = _se_m52_white(x, th, np.float64)
    dK["noise"] = np.eye(n)
    cf = sla.cho_factor(K, lower=True)
    alpha = sla.cho_solve(cf, y)
    Kinv = sla.cho_solve(cf, np.eye(n))
    Kl, dKl = _se_m52_white(x, th, np.longdouble)
    dKl["noise"] = np.eye(n, dtype=np.longdouble)
    al = alpha.astype(np.longdouble)
    al = al + sla.cho_solve(cf, np.asarray(y.astype(np.longdouble) - Kl @ al, dtype=np.float64))
    for key, D in dK.items():
        ref, mag = _grad_terms(Kinv, alpha, D)
        refl = (float(al @ dKl[key] @ al) - float(np.sum(Kinv.astype(np.longdouble) * dKl[key]))) / 2
        assert abs(ref - refl) <= 1e-12 * mag, (key, ref, refl)
        assert abs(got[key] - ref) <= 1e-10 * mag, (key, got[key], ref, abs(got[key] - ref) / mag)
