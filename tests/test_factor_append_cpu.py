"""The append restatement (tests/append_ref.py) against LAPACK's Cholesky of the joint matrix: the head / tail split
sb_factor_append uses gives the joint factor at every tail size, for every noise form, and chains."""
import numpy as np
import pytest
import scipy.linalg as sla

from append_ref import NB, AppendNotPosDef, append_factor, noise_matrix


def se(a, b, ell=1.0):
    return np.exp(-0.5 * ((a[:, None] - b[None, :]) / ell) ** 2)


def problem(n1, n2, seed, noise1=0.1, noise2=0.2, span=None):
    rng = np.random.default_rng(seed)
    span = span or max(4.0, (n1 + n2) / 16)
    x1, x2 = rng.uniform(0, span, n1), rng.uniform(0, span, n2)
    S1 = noise_matrix(noise1, n1)
    K11 = se(x1, x1) + S1
    return x1, x2, K11, se(x2, x1), se(x2, x2)


def joint(K11, K21, K22, noise2):
    return np.block([[K11, K21.T], [K21, K22 + noise_matrix(noise2, K22.shape[0])]])


@pytest.mark.parametrize("n1", [5, 127, 128, 129, 255, 256, 257, 383])
@pytest.mark.parametrize("n2", [1, 127, 128, 129, 700])
def test_append_matches_joint_cholesky(n1, n2):
    _, _, K11, K21, K22 = problem(n1, n2, seed=n1 * 1000 + n2)
    L1 = np.linalg.cholesky(K11)
    L = append_factor(L1, K21, K22, 0.2)
    Lref = sla.cholesky(joint(K11, K21, K22, 0.2), lower=True)
    np.testing.assert_allclose(L, Lref, rtol=0, atol=1e-13 * np.abs(Lref).max())


@pytest.mark.parametrize("n1", [130, 255, 384])
def test_head_block_columns_are_the_old_ones_bit_for_bit(n1):
    _, _, K11, K21, K22 = problem(n1, 200, seed=7)
    L1 = np.linalg.cholesky(K11)
    L = append_factor(L1, K21, K22, 0.2)
    h = n1 // NB * NB
    assert np.array_equal(L[:n1, :h], L1[:, :h])
    assert np.array_equal(L[:h, h:], np.zeros((h, L.shape[0] - h)))


@pytest.mark.parametrize("kind", ["scalar", "diag", "dense"])
@pytest.mark.parametrize("n1", [129, 256])
def test_noise_forms_of_the_new_observations(kind, n1):
    n2 = 150
    rng = np.random.default_rng(11)
    _, _, K11, K21, K22 = problem(n1, n2, seed=3)
    if kind == "scalar":
        s2 = 0.3
    elif kind == "diag":
        s2 = rng.uniform(0.05, 0.5, n2)
    else:
        B = rng.standard_normal((n2, 5))
        s2 = 0.05 * B @ B.T + 0.1 * np.eye(n2)
    L = append_factor(np.linalg.cholesky(K11), K21, K22, s2)
    Lref = sla.cholesky(joint(K11, K21, K22, s2), lower=True)
    np.testing.assert_allclose(L, Lref, rtol=0, atol=1e-13)


def test_dense_noise_of_the_old_observations():
    """The append never needs Sigma1: it lives in L1 only."""
    n1, n2 = 300, 140
    rng = np.random.default_rng(5)
    B = rng.standard_normal((n1, 7))
    S1 = 0.02 * B @ B.T + 0.1 * np.eye(n1)
    _, _, K11, K21, K22 = problem(n1, n2, seed=9, noise1=S1)
    L = append_factor(np.linalg.cholesky(K11), K21, K22, 0.2)
    Lref = sla.cholesky(joint(K11, K21, K22, 0.2), lower=True)
    np.testing.assert_allclose(L, Lref, rtol=0, atol=1e-13)


def test_chained_appends_equal_one_joint_factorisation():
    rng = np.random.default_rng(2)
    sizes = [200, 57, 130, 300]
    xs = [rng.uniform(0, 40, n) for n in sizes]
    noises = [0.1, 0.2, rng.uniform(0.05, 0.3, sizes[2]), 0.15]
    x = xs[0]
    L = np.linalg.cholesky(se(x, x) + noise_matrix(noises[0], sizes[0]))
    for xn, sn in zip(xs[1:], noises[1:]):
        L = append_factor(L, se(xn, x), se(xn, xn), sn)
        x = np.concatenate([x, xn])
    K = se(x, x) + sla.block_diag(*[noise_matrix(s, n) for s, n in zip(noises, sizes)])
    np.testing.assert_allclose(L, sla.cholesky(K, lower=True), rtol=0, atol=1e-13)


@pytest.mark.parametrize("n1", [100, 128, 200])
def test_failing_append_reports_the_joint_pivot(n1):
    _, _, K11, K21, K22 = problem(n1, 40, seed=4)
    with pytest.raises(AppendNotPosDef) as e:
        append_factor(np.linalg.cholesky(K11), K21, K22, -2.0)
    assert e.value.info == n1 + 1
