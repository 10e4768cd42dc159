"""The dense restatement of the elbo gradient (vfe_grad_ref.py) against central differences of the oracle's
elbo, through the same lowered specs and the same (leaf, component) aggregation the device path uses.  No GPU:
the specs are lowered on the host and evaluated with plan_eval."""
import numpy as np
import pytest

import vfe_grad_ref as ref

TH = np.array([1.3, 0.8, 0.6, 1.7, 0.05])   # v1, l1, v2, l2, white multiplier


def build(m, th):
    v1, l1, v2, l2, wv = th

    def mk(GP):
        f1 = GP(v1 * m.with_lengthscale(m.SEKernel(), l1))
        f2 = GP(v2 * m.with_lengthscale(m.Matern52Kernel(), l2) + wv * m.WhiteKernel())
        return dict(f1=f1, f2=f2, f3=f1 + 0.5 * f2)
    return m.gppp(mk)


def data():
    rng = np.random.default_rng(8)
    x3, x1 = rng.uniform(0, 10, 60), rng.uniform(0, 10, 40)
    z1, z2 = np.linspace(0.3, 9.7, 7), np.linspace(0.1, 9.9, 6)
    y = rng.standard_normal(100)
    return x3, x1, z1, z2, y


def obs(m, x3, x1):
    return m.BlockData(m.GPPPInput("f3", x3), m.GPPPInput("f1", x1))


def pseudo(m, z1, z2):
    return m.BlockData(m.GPPPInput("f1", z1), m.GPPPInput("f2", z2))


def host_gradient(sb, th, noise, jitter):
    """Dense elbo and gradient through the lowered specs: (elbo, per-(leaf, component) entries, d/d noise,
    d/d jitter) with the same conventions as grad_elbo."""
    x3, x1, z1, z2, y = data()
    fs = build(sb, th)
    fx, fz = fs(obs(sb, x3, x1), noise), fs(pseudo(sb, z1, z2), jitter)
    a = sb.finite._VfeInputs(sb.VFE(fz), fx, y)
    raw = ref.raw_gradient(a, jitter, noise)
    agg = {}
    for spec, key in ((a.uu, "uu"), (a.xu, "xu"), (a.ffd, "ff")):
        sb.finite._aggregate_terms(agg, spec, raw[key][0])
    kern = sb.finite.LogpdfGradient(None, list(agg.values()))
    gn = raw["noise_f"][0].sum() if np.ndim(noise) == 0 else raw["noise_f"][0]
    gj = raw["noise_u"][0].sum() if np.ndim(jitter) == 0 else raw["noise_u"][0]
    return raw["elbo"], kern, gn, gj, fs


def oracle_elbo(orc, th, noise, jitter):
    x3, x1, z1, z2, y = data()
    fo = build(orc, th)
    return orc.elbo(orc.VFE(fo(pseudo(orc, z1, z2), jitter)), fo(obs(orc, x3, x1), noise), y)


def central(f, x, h):
    return (f(x + h) - f(x - h)) / (2 * h)


@pytest.mark.parametrize("vector_noise", [False, True], ids=["scalar_noise", "vector_noise"])
def test_dense_elbo_gradient_vs_finite_differences(sb, orc, vector_noise):
    rng = np.random.default_rng(9)
    noise = rng.uniform(0.1, 0.3, 100) if vector_noise else 0.15
    jitter = rng.uniform(1e-3, 2e-3, 13) if vector_noise else 1e-3
    e, kern, gn, gj, fs = host_gradient(sb, TH, noise, jitter)
    np.testing.assert_allclose(e, oracle_elbo(orc, TH, noise, jitter), rtol=1e-12)
    k1, k2, kw = kern.for_atom(fs.fs["f1"], 0), kern.for_atom(fs.fs["f2"], 0), kern.for_atom(fs.fs["f2"], 1)
    got = np.array([k1["dcoeff"], -k1["dlogscale"] / TH[1], k2["dcoeff"], -k2["dlogscale"] / TH[3], kw["dcoeff"]])
    fd = np.zeros(5)
    for i in range(5):
        def fth(v, i=i):
            t = TH.copy()
            t[i] = v
            return oracle_elbo(orc, t, noise, jitter)
        fd[i] = central(fth, TH[i], 1e-5 * TH[i])
    np.testing.assert_allclose(got, fd, rtol=1e-6)
    i0, j0 = 17, 4
    if vector_noise:
        def fn(v):
            nv = noise.copy()
            nv[i0] = v
            return oracle_elbo(orc, TH, nv, jitter)

        def fj(v):
            jv = jitter.copy()
            jv[j0] = v
            return oracle_elbo(orc, TH, noise, jv)
        np.testing.assert_allclose(gn[i0], central(fn, noise[i0], 1e-5 * noise[i0]), rtol=1e-6)
        np.testing.assert_allclose(gj[j0], central(fj, jitter[j0], 1e-4 * jitter[j0]), rtol=1e-6)
    else:
        np.testing.assert_allclose(gn, central(lambda v: oracle_elbo(orc, TH, v, jitter), noise, 1e-5 * noise),
                                   rtol=1e-6)
        np.testing.assert_allclose(gj, central(lambda v: oracle_elbo(orc, TH, noise, v), jitter, 1e-4 * jitter),
                                   rtol=1e-6)

