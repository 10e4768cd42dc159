"""Posterior mean and variance and the logpdf gradient of the exact low-rank model (exact_refs.py, Woodbury
references) at the outer-step remainders of the posterior sweep that test_gpu_exact.py's low-rank test
does not reach: N = 640 (5 block columns, nblk = 1 mod 4: a one-column last outer step) and N = 1536
(12 block columns, nblk = 0 mod 4: full steps only).  The sweep solves 4 block columns per outer step and
applies them to the rest of W in one K = 512 update; both trailing-update paths run.
"""
import numpy as np
import pytest

import exact_refs as er
from test_gpu_exact import _close, check_path, lowrank, lowrank_gppp, trailing  # noqa: F401 (trailing: fixture)

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("n", [640, 1536])
def test_lowrank_posterior_and_gradients_at_sweep_remainders(sb, trailing, n):
    """Same model, references and rtol 1e-9 as test_gpu_exact.test_lowrank_gradients_and_posterior
    (lambda_min(K) >= 1, lambda_max(K) <= 5e5); test points cover every block column of W."""
    H, c, d, y, wb = lowrank(n)
    fs = lowrank_gppp(sb, H, c)
    fx = fs(sb.GPPPInput("f", np.arange(n, dtype=np.float64)), d.astype(np.float64))
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
