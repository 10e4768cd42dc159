"""CPU pins for the numerical schemes the CUDA library uses in place of LAPACK's dpotrf / dtrsm (the reference's
`cholesky(Symmetric(cov(fx)))`, SURVEY.md App. A): the int8 digit-plane product, the wide panel phase and the
peer-to-peer exchange protocol -- restated in NumPy in oracle/device_algorithms.py and checked here against
exact integer arithmetic, LAPACK and randomised interleavings.  The device kernels are compared with the
oracle and with LAPACK on the GPU (tests/test_gpu_parity.py), which checks their end results, not the raw
int32 digit products."""
from fractions import Fraction

import numpy as np
import pytest

from oracle import device_algorithms as da


def _rows(rng, m, K, spread):
    """rows with very different magnitudes and a few exact zeros"""
    P = rng.standard_normal((m, K)) * np.exp(rng.uniform(-spread, spread, (m, 1)))
    P[rng.random((m, K)) < 0.02] = 0.0
    return P


def test_digit_planes_reconstruct_to_56_bits():
    rng = np.random.default_rng(1)
    P = _rows(rng, 64, 96, 30.0)
    P[5] = 0.0                                     # an all-zero row has scale 0 and zero digits
    d, s = da.oz_slice(P)
    assert d.dtype == np.int8 and d.shape == (7, 64, 96)
    R = da.oz_reconstruct(d, s)
    mx = np.max(np.abs(P), axis=1, keepdims=True)
    assert np.all(np.abs(R - P) <= mx * 2.0 ** -53)  # half an ulp of the 56-bit grid is 2^-56 * 2^(e) <= mx 2^-54
    assert s[5] == 0.0 and not d[:, 5].any()
    # balanced digits: the six low planes really use the signed range
    assert d[1:].min() == -128 and d[1:].max() == 127


def test_digit_planes_are_an_exact_integer_identity():
    """Z = sum_p d_p 256^(6-p) holds exactly (checked with Python integers), including negative values and carries."""
    rng = np.random.default_rng(2)
    P = _rows(rng, 8, 40, 5.0)
    d, s = da.oz_slice(P)
    e = np.round(np.log2(s)).astype(int) + 31
    for i in range(P.shape[0]):
        for k in range(P.shape[1]):
            Z = int(np.rint(np.ldexp(P[i, k], 55 - e[i])))
            assert Z == sum(int(d[p, i, k]) * 256 ** (6 - p) for p in range(7))


def test_digit_plane_product_matches_exact_arithmetic():
    rng = np.random.default_rng(3)
    m, n, K = 24, 16, 512
    A, B = _rows(rng, m, K, 8.0), _rows(rng, n, K, 8.0)
    dA, sA = da.oz_slice(A)
    dB, sB = da.oz_slice(B)
    C, gmax = da.oz_product(dA, sA, dB, sB)
    assert gmax < 2 ** 31                           # int32 accumulators: 7 pairs x 512 x 2^14 < 2^31
    assert 7 * K * 128 * 128 < 2 ** 31
    exact = np.array([[float(sum(Fraction(a) * Fraction(b) for a, b in zip(A[i], B[j]))) for j in range(n)] for i in range(m)])
    bound = np.max(np.abs(A), axis=1)[:, None] * np.max(np.abs(B), axis=1)[None, :]
    err = np.abs(C - exact) / bound
    # dropped pairs (p + q > 6) + 56-bit rounding: a few 1e-15 of max|row_i| max|row_j| per unit of sqrt(K)
    assert err.max() < 2e-13, err.max()
    # and it is not worse than plain fp64 accumulation by more than that
    assert np.abs(A @ B.T - exact).max() / bound.max() < 1e-13


def test_dropping_low_digit_pairs_is_what_limits_the_accuracy():
    rng = np.random.default_rng(4)
    A, B = rng.standard_normal((8, 256)), rng.standard_normal((8, 256))
    dA, sA = da.oz_slice(A)
    dB, sB = da.oz_slice(B)
    full, _ = da.oz_product(dA, sA, dB, sB, max_group=12)     # all 49 pairs: exact up to the 56-bit rounding
    kept, _ = da.oz_product(dA, sA, dB, sB)                   # the kernel's 28 pairs
    exact = np.array([[float(sum(Fraction(a) * Fraction(b) for a, b in zip(A[i], B[j]))) for j in range(8)] for i in range(8)])
    assert np.abs(full - exact).max() < 1e-14
    assert np.abs(kept - exact).max() < 5e-13
    assert np.abs(kept - exact).max() >= np.abs(full - exact).max()


@pytest.mark.parametrize("m_below", [0, 128, 640])
def test_wide_panel_phase_equals_lapack(m_below):
    rng = np.random.default_rng(5)
    w, n = 512, 512 + m_below
    G = rng.standard_normal((n, n + 8))
    S = G @ G.T / n + 0.5 * np.eye(n)
    L = np.linalg.cholesky(S)
    out, W = da.wide_panel_factor(S[:, :w].copy())
    np.testing.assert_allclose(np.tril(out[:w]), L[:w, :w], rtol=0, atol=2e-13)
    np.testing.assert_allclose(out[w:], L[w:, :w], rtol=0, atol=2e-13)
    # the identity rows hold inv(L_512): block lower triangular, and W L = I
    np.testing.assert_allclose(W @ L[:w, :w], np.eye(w), atol=1e-12)
    assert np.all(W[:128, 128:] == 0.0) and np.all(W[128:256, 256:] == 0.0)


def test_wide_panel_phase_with_the_digit_plane_product():
    """the device's panel solve: X = A inv(L_512)^T through int8 digit planes of both operands"""
    rng = np.random.default_rng(6)
    w, n = 512, 512 + 256
    G = rng.standard_normal((n, n + 8))
    S = G @ G.T / n + 0.1 * np.eye(n)
    d = np.exp(rng.uniform(-4, 4, n))
    S = S * d[:, None] * d[None, :]                 # badly scaled rows / columns, still SPD
    L = np.linalg.cholesky(S)

    def product(A, Wm):
        dA, sA = da.oz_slice(A)
        dW, sW = da.oz_slice(Wm)
        return da.oz_product(dA, sA, dW, sW)[0]

    out, _ = da.wide_panel_factor(S[:, :w].copy(), product=product)
    scale = np.sqrt(np.diag(S))[w:, None]           # |L_ij| <= sqrt(S_ii): the natural error unit of a Cholesky row
    assert np.max(np.abs(out[w:] - L[w:, :w]) / scale) < 1e-11


@pytest.mark.parametrize("world", [2, 3, 4, 5, 8])
def test_p2p_exchange_protocol_is_safe_and_live(world):
    rng = np.random.default_rng(100 + world)
    for trial in range(30):
        ncols = int(rng.integers(5, 90))
        base = [int(b) for b in rng.integers(0, 50, world)] if trial % 2 else None   # counters survive across factorisations
        mdl = da.P2PExchangeModel(world, ncols, slots=8, base=base)
        bias = None if trial % 3 else [1e-3 if r == trial % world else 1.0 for r in range(world)]   # one very slow rank
        mdl.run(rng, bias)
        for r in range(world):
            assert sorted(mdl.got[r]) == [k for k in range(ncols) if k % world != r]


def test_p2p_exchange_without_the_slot_guard_is_caught():
    """Sanity of the model, and why the guard exists: with 8 ranks only half of them own a column in a given
    outer step, so a slow rank is not implicitly waited for; without the ack guard a fast owner overwrites the
    slot the slow rank still has to pull."""
    rng = np.random.default_rng(7)
    hit = 0
    for trial in range(40):
        mdl = da.P2PExchangeModel(8, 64, slots=8, guard=False)
        try:
            mdl.run(rng, [1e-3 if r == trial % 8 else 1.0 for r in range(8)])
        except AssertionError as e:
            assert "overwrites slot" in str(e) or "expected column" in str(e)
            hit += 1
    assert hit > 0
