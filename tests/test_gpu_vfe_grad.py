"""Device gradient of the VFE elbo (sb_vfe_grad / grad_elbo) against finite differences of the oracle, against
the dense restatement (vfe_grad_ref.py) at the scale of the K_fu stream, against grad_logpdf when the
pseudo-points are the observations, and at the config-4 shape.  Every case runs with `trailing` = 0 (fp64
DMMA) and 1 (int8 Ozaki, which the M x M factors take only above 8 block columns) and asserts which path ran."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

import vfe_grad_ref as ref

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NB, OUTER_BLOCKS = 128, 4
INITIAL_TRAILING = 1 if os.environ.get("SB_TRAILING") == "ozaki" else 0


@pytest.fixture(params=[0, 1], ids=["dmma", "ozaki"])
def trailing(request, sb):
    ctx = sb.default_context()
    ctx.set_option("trailing", request.param)
    try:
        yield request.param
    finally:
        ctx.set_option("trailing", INITIAL_TRAILING)


def check_path(sb, trailing, m):
    """The M x M factors run the int8 Ozaki driver only with trailing = 1 and more than 8 block columns."""
    ops = sb.default_context().timings()["trailing_int8_ops"]
    ozaki = trailing == 1 and (m + NB - 1) // NB > 2 * OUTER_BLOCKS
    assert (ops > 0) if ozaki else (ops == 0), (trailing, m, ops)


def device_raw(sb, v, fx, y):
    """The raw arrays of sb_vfe_grad and the elbo of the same handle."""
    a = sb.finite._VfeInputs(v, fx, y)
    handle, e, _ = sb.finite._vfe_create(v, fx, y, a)
    out = dict(uu=np.zeros(2 * max(1, a.uu.nterms)), xu=np.zeros(2 * max(1, a.xu.nterms)),
               ff=np.zeros(2 * max(1, a.ffd.nterms)), noise_u=np.empty(a.m), noise_f=np.empty(a.n))
    lib = sb.lib.load()
    sb.lib.check(lib.sb_vfe_grad(handle.ctx.h, handle.h, C.byref(a.uu), C.byref(a.xu), C.byref(a.ffd), C.byref(a.nf),
                                 a.delta.ctypes.data, *[out[k].ctypes.data for k in ("uu", "xu", "ff", "noise_u", "noise_f")]))
    return a, e, out


# -- 1. finite differences of the oracle's elbo ------------------------------------------------------

def _model(m, th):
    v1, l1, v2, l2, wv = th

    def mk(GP):
        f1 = GP(v1 * m.with_lengthscale(m.SEKernel(), l1))
        f2 = GP(v2 * m.with_lengthscale(m.Matern52Kernel(), l2) + wv * m.WhiteKernel())
        return dict(f1=f1, f2=f2, f3=f1 + 0.5 * f2)
    return m.gppp(mk)


def test_elbo_gradient_vs_finite_differences(sb, orc, trailing):
    rng = np.random.default_rng(61)
    x3, x1 = rng.uniform(0, 10, 300), rng.uniform(0, 10, 220)
    z1, z2 = np.linspace(0.2, 9.8, 40), np.linspace(0.1, 9.9, 33)
    y = rng.standard_normal(520)
    th = np.array([1.3, 0.8, 0.6, 1.7, 0.05])
    noise, jitter = 0.15, 1e-3

    def obs(m):
        return m.BlockData(m.GPPPInput("f3", x3), m.GPPPInput("f1", x1))

    def pseudo(m):
        return m.BlockData(m.GPPPInput("f1", z1), m.GPPPInput("f2", z2))

    def elbo_o(t, nz=noise, jt=jitter):
        fo = _model(orc, t)
        return orc.elbo(orc.VFE(fo(pseudo(orc), jt)), fo(obs(orc), nz), y)

    fs = _model(sb, th)
    sb.default_context().timings(reset=True)
    gr = sb.grad_elbo(sb.VFE(fs(pseudo(sb), jitter)), fs(obs(sb), noise), y)
    check_path(sb, trailing, 73)
    np.testing.assert_allclose(gr.elbo, elbo_o(th), rtol=1e-10)
    k1, k2, kw = gr.for_atom(fs.fs["f1"], 0), gr.for_atom(fs.fs["f2"], 0), gr.for_atom(fs.fs["f2"], 1)
    got = np.array([k1["dcoeff"], -k1["dlogscale"] / th[1], k2["dcoeff"], -k2["dlogscale"] / th[3], kw["dcoeff"],
                    gr.noise, gr.inducing_noise])
    fd = np.zeros(7)
    for i in range(5):
        h = 1e-5 * th[i]
        tp, tm = th.copy(), th.copy()
        tp[i] += h
        tm[i] -= h
        fd[i] = (elbo_o(tp) - elbo_o(tm)) / (2 * h)
    fd[5] = (elbo_o(th, nz=noise * (1 + 1e-5)) - elbo_o(th, nz=noise * (1 - 1e-5))) / (2e-5 * noise)
    fd[6] = (elbo_o(th, jt=jitter * (1 + 1e-4)) - elbo_o(th, jt=jitter * (1 - 1e-4))) / (2e-4 * jitter)
    np.testing.assert_allclose(got, fd, rtol=1e-5, atol=1e-6)
    # one element of vector observation noise
    nv = rng.uniform(0.1, 0.3, 520)
    gv = sb.grad_elbo(sb.SparseFiniteGP(fs(obs(sb), nv), fs(pseudo(sb), jitter)), y)
    i0 = 17
    nvp, nvm = nv.copy(), nv.copy()
    nvp[i0] += 1e-6
    nvm[i0] -= 1e-6
    np.testing.assert_allclose(gv.noise[i0], (elbo_o(th, nz=nvp) - elbo_o(th, nz=nvm)) / 2e-6, rtol=1e-5, atol=1e-6)


# -- 2. dense reference at the scale of the stream -------------------------------------------------------

def test_raw_gradient_vs_dense_reference(sb, trailing):
    """N = 2 * 16384 + 1001 (three chunks, the last ragged), M = 1000 (not a multiple of 128, two outer steps)
    and one block of 7 terms (more than the 6 a device block holds): every raw array within 1e-9 of the sum of
    the absolute values of its elementwise contributions."""
    rng = np.random.default_rng(33769)
    n, m = 2 * 16384 + 1001, 1000
    x = rng.uniform(0, 300, n)
    z = np.linspace(0, 300, m)
    y = np.sin(x) + 0.3 * rng.standard_normal(n)
    noise = rng.uniform(0.05, 0.15, n)
    jitter = 1e-2
    parts = [(1.0, "SEKernel", 1.2), (0.5, "Matern12Kernel", 2.0), (0.4, "Matern32Kernel", 0.7),
             (0.3, "Matern52Kernel", 1.5), (0.2, "SEKernel", 0.4), (0.2, "Matern52Kernel", 3.0)]

    def mk(GP):
        k = 0.05 * sb.WhiteKernel()
        for v, name, ell in parts:
            k = k + v * sb.with_lengthscale(getattr(sb, name)(), ell)
        return dict(f=GP(k))
    fs = sb.gppp(mk)
    fx, fz = fs(sb.GPPPInput("f", x), noise), fs(sb.GPPPInput("f", z), jitter)
    sb.default_context().timings(reset=True)
    a, e, got = device_raw(sb, sb.VFE(fz), fx, y)
    check_path(sb, trailing, m)
    assert a.xu.nterms == 7 and a.uu.nterms == 7
    want = ref.raw_gradient(a, jitter, noise)
    np.testing.assert_allclose(e, want["elbo"], rtol=1e-11)
    for key in ("uu", "xu", "ff", "noise_u", "noise_f"):
        g, mag = want[key]
        err = np.abs(got[key] - g)
        assert np.all(err <= 1e-9 * mag), (key, float(np.max(err / np.maximum(mag, 1e-300))))


# -- 3. pseudo-points at the observations: elbo == logpdf, and so are their gradients ---------------------

def test_inducing_at_observations_matches_logpdf_gradient(sb, trailing):
    """README.md:75-78: Z = X with a vanishing jitter makes the elbo the exact logpdf; then the kernel and noise
    gradients of the two agree too (in exact fp64 on the host: 1e-10 for the kernel, 7e-9 for the noise;
    cond(K_uu) ~ 2e5)."""
    rng = np.random.default_rng(1500)
    x = rng.uniform(0, 300, 1500)
    y = np.sin(x) + 0.3 * rng.standard_normal(1500)
    f = sb.gppp(lambda GP: dict(f=GP(sb.Matern12Kernel())))
    fx = f(sb.GPPPInput("f", x), 0.1)
    sb.default_context().timings(reset=True)
    ge = sb.grad_elbo(sb.VFE(f(sb.GPPPInput("f", x), 1e-10)), fx, y)
    check_path(sb, trailing, 1500)
    gl = sb.grad_logpdf(fx, y)
    ke, kl = ge.for_atom(f.fs["f"], 0), gl.for_atom(f.fs["f"], 0)
    np.testing.assert_allclose([ke["dcoeff"], ke["dlogscale"]], [kl["dcoeff"], kl["dlogscale"]], rtol=1e-7)
    np.testing.assert_allclose(ge.noise, gl.noise, rtol=1e-7)
    np.testing.assert_allclose(ge.elbo, sb.logpdf(fx, y), rtol=1e-7)


# -- 4. config-4 shape ------------------------------------------------------------------------------------

def test_config4_shape(sb, trailing):
    """N = 131072, M = 4096: the value from the gradient's handle is the elbo; the variance and lengthscale
    gradients match central differences of the device elbo."""
    rng = np.random.default_rng(4)
    n, m = 131072, 4096
    x = rng.uniform(0, m, n)
    z = np.arange(m) + 0.5
    y = np.sin(x) + 0.3 * rng.standard_normal(n)
    th = np.array([1.1, 1.3])

    def parts(t):
        fs = sb.gppp(lambda GP: dict(f=GP(t[0] * sb.with_lengthscale(sb.SEKernel(), t[1]))))
        return fs, fs(sb.GPPPInput("f", x), 0.1), fs(sb.GPPPInput("f", z), 1e-9)

    fs, fx, fz = parts(th)
    sb.default_context().timings(reset=True)
    gr = sb.grad_elbo(sb.VFE(fz), fx, y)
    check_path(sb, trailing, m)
    np.testing.assert_allclose(gr.elbo, sb.elbo(sb.VFE(fz), fx, y), rtol=1e-13)
    k = gr.for_atom(fs.fs["f"], 0)
    got = np.array([k["dcoeff"], -k["dlogscale"] / th[1]])
    fd = np.zeros(2)
    for i in range(2):
        h = 1e-4 * th[i]
        tp, tm = th.copy(), th.copy()
        tp[i] += h
        tm[i] -= h
        _, fxp, fzp = parts(tp)
        _, fxm, fzm = parts(tm)
        fd[i] = (sb.elbo(sb.VFE(fzp), fxp, y) - sb.elbo(sb.VFE(fzm), fxm, y)) / (2 * h)
    np.testing.assert_allclose(got, fd, rtol=1e-4)


# -- 5. invalid arguments -----------------------------------------------------------------------------------

def test_invalid_arguments_are_refused(sb):
    rng = np.random.default_rng(5)
    f = sb.gppp(lambda GP: dict(f=GP(sb.SEKernel())))

    def problem(n, m):
        x, z = rng.uniform(0, 10, n), np.linspace(0, 10, m)
        return sb.VFE(f(sb.GPPPInput("f", z), 1e-6)), f(sb.GPPPInput("f", x), 0.1), rng.standard_normal(n)

    v, fx, y = problem(300, 20)
    a = sb.finite._VfeInputs(v, fx, y)
    handle, _, _ = sb.finite._vfe_create(v, fx, y, a)
    lib = sb.lib.load()
    g = [np.zeros(max(2 * a.uu.nterms, 2)), np.zeros(max(2 * a.xu.nterms, 2)), np.zeros(max(2 * a.ffd.nterms, 2)),
         np.zeros(a.m), np.zeros(a.n)]

    def call(uu, xu, ffd, nf):
        return lib.sb_vfe_grad(handle.ctx.h, handle.h, C.byref(uu), C.byref(xu), C.byref(ffd), C.byref(nf),
                               a.delta.ctypes.data, *[b.ctypes.data for b in g])

    assert call(a.uu, a.xu, a.ffd, a.nf) == sb.lib.SB_OK
    dense = sb.finite._noise_struct(0.1 * np.eye(a.n), a.n)
    assert call(a.uu, a.xu, a.ffd, dense) == sb.lib.SB_ERR_INVALID
    b_n = sb.finite._VfeInputs(*problem(301, 20))      # N differs from the handle's
    b_m = sb.finite._VfeInputs(*problem(300, 21))      # M differs
    assert call(a.uu, b_n.xu, b_n.ffd, a.nf) == sb.lib.SB_ERR_INVALID
    assert call(a.uu, a.xu, b_n.ffd, a.nf) == sb.lib.SB_ERR_INVALID
    assert call(b_m.uu, a.xu, a.ffd, a.nf) == sb.lib.SB_ERR_INVALID
    assert call(a.uu, b_m.xu, a.ffd, a.nf) == sb.lib.SB_ERR_INVALID
    with pytest.raises(ValueError):
        sb.grad_elbo(v, fx, y[:-1])
    with pytest.raises(NotImplementedError):
        sb.grad_elbo(v, f(sb.GPPPInput("f", rng.uniform(0, 10, 300)), 0.1 * np.eye(300)), y)
    # the context is still usable
    gr = sb.grad_elbo(v, fx, y)
    np.testing.assert_allclose(gr.elbo, sb.elbo(v, fx, y), rtol=1e-13)
    np.testing.assert_allclose(gr.noise, g[4].sum(), rtol=1e-10)


# -- 6. two GPUs --------------------------------------------------------------------------------------------

def test_elbo_gradient_sharded_over_two_gpus():
    """The chunks sharded over 2 ranks with one all-reduce of the partial sums: the same gradient as 1 GPU."""
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2",
           "--master-addr", "127.0.0.1", "--master-port", "29563", os.path.join(ROOT, "tests", "dist_vfe_grad_worker.py")]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=300)
    assert "VFE_GRAD_DIST_OK" in r.stdout, r.stdout[-2000:] + r.stderr[-3000:]
