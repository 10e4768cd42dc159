"""sb_factor_append on the GPU: posterior(f_post(x2, s2), y2) extends the old factor instead of refactorising the
stacked problem.  Checked against the CPU oracle on the stacked data, against the device's own fresh joint
factorisation, through export / import, chained, on the int8 Ozaki path, at the config-2 size and on two GPUs."""
import ctypes as C
import gc
import os
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RTOL = 1e-10
NB = 128


def se_model(m):
    return m.gppp(lambda GP: dict(f=GP(m.SEKernel())))


def matern_model(m):
    return m.gppp(lambda GP: dict(f=GP(m.with_lengthscale(m.Matern52Kernel(), 2.0))))


def f3_white_model(m):
    """f3 = f1 + f2 (examples/process_decomposition) with a White term in f1: an f3 input equal to an f1 input
    picks it up in the cross-covariance."""
    return m.gppp(lambda GP: (lambda f1, f2: dict(f1=f1, f2=f2, f3=f1 + f2))(
        GP(m.SEKernel() + 0.1 * m.WhiteKernel()), GP(m.Matern52Kernel())))


def handle_logpdf(sb, fac, delta):
    out = (C.c_double * 1)()
    d = np.ascontiguousarray(delta, dtype=np.float64)
    sb.lib.check(sb.lib.load().sb_logpdf(fac.ctx.h, fac.h, d.ctypes.data, 1, out))
    return out[0]


def two_step(sb, orc, builder, n1, n2, seed, s1=0.1, s2=0.2, proc1="f", proc2="f", shared=0):
    """p12 = posterior(posterior(fx1, y1)(x2, s2), y2) on the device and the oracle's posterior of the stacked
    observations.  shared: the first `shared` new inputs repeat old ones."""
    rng = np.random.default_rng(seed)
    span = max(10.0, (n1 + n2) / 32)
    x1, x2 = rng.uniform(0, span, n1), rng.uniform(0, span, n2)
    x2[:shared] = x1[:shared]
    fs, fo = builder(sb), builder(orc)
    bo = orc.BlockData(orc.GPPPInput(proc1, x1), orc.GPPPInput(proc2, x2))
    noise = np.concatenate([np.broadcast_to(s1, n1), np.broadcast_to(s2, n2)]).astype(np.float64)
    y = orc.rand(fo(bo, noise), rng.standard_normal(n1 + n2))
    p1 = sb.posterior(fs(sb.GPPPInput(proc1, x1), s1), y[:n1])
    p12 = sb.posterior(p1(sb.GPPPInput(proc2, x2), s2), y[n1:])
    po = orc.posterior(fo(bo, noise), y)
    return fs, fo, p1, p12, po, (x1, x2, y, noise), span


CASES = [  # (model, N1, N2): the Schur factor S has r + N2 rows, r = N1 mod 128
    ("se", 1000, 700),          # r = 104, S = 804: one full 4-block outer step and a remainder of 3
    ("matern52", 4097, 1500),   # r = 1, S = 1501: 12 blocks
    ("se", 4223, 2048),         # r = 127, S = 2175: 17 blocks, remainder 1
    ("se", 16384, 2048),        # r = 0, S = P
]


@pytest.mark.parametrize("name,n1,n2", CASES)
def test_appended_posterior_matches_oracle(sb, orc, name, n1, n2):
    builder = {"se": se_model, "matern52": matern_model}[name]
    fs, fo, p1, p12, po, (x1, x2, y, noise), span = two_step(sb, orc, builder, n1, n2, seed=n1 + n2)
    rng = np.random.default_rng(1)
    xs = rng.uniform(0, span, 300)
    m, v = sb.mean_and_var(p12, sb.GPPPInput("f", xs))
    mo, vo = orc.mean_and_var(po, orc.GPPPInput("f", xs))
    np.testing.assert_allclose(m, mo, rtol=RTOL, atol=1e-11)
    np.testing.assert_allclose(v, vo, rtol=1e-9, atol=1e-11)
    xc = xs[:120]
    np.testing.assert_allclose(sb.cov(p12, sb.GPPPInput("f", xc)), orc.cov(po, orc.GPPPInput("f", xc)),
                               rtol=RTOL, atol=1e-11)
    z = rng.standard_normal((120, 2))
    np.testing.assert_allclose(sb.rand(p12(sb.GPPPInput("f", xc), 0.05), z),
                               orc.rand(po(orc.GPPPInput("f", xc), 0.05), z), rtol=RTOL, atol=1e-10)


def test_gppp_old_on_f1_new_on_f3_with_white_at_shared_inputs(sb, orc):
    fs, fo, p1, p12, po, (x1, x2, y, noise), span = two_step(sb, orc, f3_white_model, 700, 450, seed=3,
                                                              proc1="f1", proc2="f3", shared=40)
    rng = np.random.default_rng(2)
    xa, xb = rng.uniform(0, span, 90), rng.uniform(0, span, 70)
    xa[:10] = x1[:10]
    qs = sb.BlockData(sb.GPPPInput("f1", xa), sb.GPPPInput("f2", xb), sb.GPPPInput("f3", xa))
    qo = orc.BlockData(orc.GPPPInput("f1", xa), orc.GPPPInput("f2", xb), orc.GPPPInput("f3", xa))
    m, v = sb.mean_and_var(p12, qs)
    mo, vo = orc.mean_and_var(po, qo)
    np.testing.assert_allclose(m, mo, rtol=RTOL, atol=1e-11)
    np.testing.assert_allclose(v, vo, rtol=1e-9, atol=1e-11)
    np.testing.assert_allclose(sb.cov(p12, qs), orc.cov(po, qo), rtol=RTOL, atol=1e-11)


def fresh_joint(sb, fs, x1, x2, noise):
    return fs(sb.BlockData(sb.GPPPInput("f", x1), sb.GPPPInput("f", x2)), noise)


@pytest.mark.parametrize("n1,n2,kind", [(1000, 300, "scalar"), (4096, 300, "diag"), (700, 260, "dense"),
                                        (100, 90, "scalar")])
def test_appended_factor_equals_fresh_joint_factorisation(sb, n1, n2, kind):
    rng = np.random.default_rng(n1)
    span = (n1 + n2) / 32
    x1, x2 = rng.uniform(0, span, n1), rng.uniform(0, span, n2)
    if kind == "scalar":
        s2, s2full = 0.2, np.full(n2, 0.2)
    elif kind == "diag":
        s2 = rng.uniform(0.05, 0.3, n2)
        s2full = s2
    else:
        B = rng.standard_normal((n2, 6))
        s2 = 0.02 * B @ B.T + 0.1 * np.eye(n2)
        s2full = s2
    fs = se_model(sb)
    y = np.sin(np.concatenate([x1, x2])) + 0.1 * rng.standard_normal(n1 + n2)
    p1 = sb.posterior(fs(sb.GPPPInput("f", x1), 0.1), y[:n1])
    p12 = sb.posterior(p1(sb.GPPPInput("f", x2), s2), y[n1:])
    if kind == "dense":
        noise = np.zeros((n1 + n2, n1 + n2))
        noise[:n1, :n1] = 0.1 * np.eye(n1)
        noise[n1:, n1:] = s2full
    else:
        noise = np.concatenate([np.full(n1, 0.1), s2full])
    fj = fresh_joint(sb, fs, x1, x2, noise)
    L, Lj = p12.fac.to_dense_L(), fj.factor().to_dense_L()
    h = n1 // NB * NB
    np.testing.assert_array_equal(L[:n1, :h], p1.fac.to_dense_L()[:, :h])   # the head is the old factor, verbatim
    np.testing.assert_allclose(L, Lj, rtol=0, atol=1e-12)
    assert abs(p12.fac.logdet() - fj.factor().logdet()) <= 1e-12 * abs(fj.factor().logdet())
    lp = handle_logpdf(sb, p12.fac, p12.delta)
    assert abs(lp - sb.logpdf(fj, y)) <= 1e-12 * abs(lp)
    # export -> import of the appended handle: bit-identical logpdf and predictions
    xs = rng.uniform(0, span, 200)
    m, v = sb.mean_and_var(p12, sb.GPPPInput("f", xs))
    blob = p12.fac.export()
    fx2 = sb.load_factor(fresh_joint(sb, fs, x1, x2, noise), blob.copy())
    assert sb.logpdf(fx2, y) == lp
    m2, v2 = sb.mean_and_var(sb.posterior(fx2, y), sb.GPPPInput("f", xs))
    np.testing.assert_array_equal(m2, m)
    np.testing.assert_array_equal(v2, v)


def test_chained_appends_equal_one_stacked_posterior_and_leave_p1_unchanged(sb, orc):
    rng = np.random.default_rng(9)
    sizes, noises = [300, 200, 130, 129], [0.1, 0.2, 0.05, 0.15]
    xs_in = [rng.uniform(0, 30, n) for n in sizes]
    fs, fo = se_model(sb), se_model(orc)
    ys = [np.sin(x) + 0.2 * rng.standard_normal(x.size) for x in xs_in]
    xq = rng.uniform(0, 30, 150)
    p1 = sb.posterior(fs(sb.GPPPInput("f", xs_in[0]), noises[0]), ys[0])
    m1, v1 = sb.mean_and_var(p1, sb.GPPPInput("f", xq))
    p = p1
    for x, s, y in zip(xs_in[1:], noises[1:], ys[1:]):
        p = sb.posterior(p(sb.GPPPInput("f", x), s), y)
    bo = orc.BlockData(*[orc.GPPPInput("f", x) for x in xs_in])
    noise = np.concatenate([np.full(n, s) for n, s in zip(sizes, noises)])
    po = orc.posterior(fo(bo, noise), np.concatenate(ys))
    m, v = sb.mean_and_var(p, sb.GPPPInput("f", xq))
    mo, vo = orc.mean_and_var(po, orc.GPPPInput("f", xq))
    np.testing.assert_allclose(m, mo, rtol=RTOL, atol=1e-11)
    np.testing.assert_allclose(v, vo, rtol=1e-9, atol=1e-11)
    fj = fs(sb.BlockData(*[sb.GPPPInput("f", x) for x in xs_in]), noise)
    np.testing.assert_allclose(p.fac.to_dense_L(), fj.factor().to_dense_L(), rtol=0, atol=1e-12)
    m1b, v1b = sb.mean_and_var(p1, sb.GPPPInput("f", xq))   # posterior is pure: p1 predicts as before
    np.testing.assert_array_equal(m1b, m1)
    np.testing.assert_array_equal(v1b, v1)


@pytest.mark.parametrize("n1", [1000, 4096, 100])
def test_negative_new_noise_reports_the_joint_pivot(sb, n1):
    rng = np.random.default_rng(4)
    x1, x2 = rng.uniform(0, 30, n1), rng.uniform(0, 30, 64)
    fs = se_model(sb)
    p1 = sb.posterior(fs(sb.GPPPInput("f", x1), 0.1), np.sin(x1))
    with pytest.raises(sb.PosDefException) as e:
        sb.posterior(p1(sb.GPPPInput("f", x2), -2.0), np.sin(x2))
    assert e.value.info == n1 + 1
    m = sb.mean(p1, sb.GPPPInput("f", x2))   # the old posterior still works
    assert np.all(np.isfinite(m))


def test_int8_ozaki_append(sb, orc):
    ctx = sb.default_context()
    ctx.set_option("trailing", 1)
    try:
        rng = np.random.default_rng(12)
        n1, n2 = 4096, 1500
        x1, x2 = rng.uniform(0, 170, n1), rng.uniform(0, 170, n2)
        fs, fo = se_model(sb), se_model(orc)
        bo = orc.BlockData(orc.GPPPInput("f", x1), orc.GPPPInput("f", x2))
        noise = np.concatenate([np.full(n1, 0.1), np.full(n2, 0.2)])
        y = orc.rand(fo(bo, noise), rng.standard_normal(n1 + n2))
        p1 = sb.posterior(fs(sb.GPPPInput("f", x1), 0.1), y[:n1])
        ctx.timings(reset=True)
        p12 = sb.posterior(p1(sb.GPPPInput("f", x2), 0.2), y[n1:])
        assert ctx.timings()["trailing_int8_ops"] > 0, "the int8 Ozaki path did not run on S (12 blocks)"
        po = orc.posterior(fo(bo, noise), y)
        xs = rng.uniform(0, 170, 300)
        m, v = sb.mean_and_var(p12, sb.GPPPInput("f", xs))
        mo, vo = orc.mean_and_var(po, orc.GPPPInput("f", xs))
        np.testing.assert_allclose(m, mo, rtol=RTOL, atol=1e-11)
        np.testing.assert_allclose(v, vo, rtol=1e-9, atol=1e-11)
    finally:
        ctx.set_option("trailing", 0)


def test_config2_full_size_append_matches_fresh_joint(sb):
    """N1 = 65536 (bench.make_inputs), N2 = 4096: logpdf, posterior mean and variance from the appended handle
    against a fresh joint factorisation.  The appended handle is released before the joint one is built."""
    sys.path.insert(0, ROOT)
    from bench import make_inputs
    n1, n2 = 65536, 4096
    x, y, xs = make_inputs(n1 + n2, 4096)
    x1, x2, y1, y2 = x[:n1], x[n1:], y[:n1], y[n1:]
    fs = se_model(sb)
    p1 = sb.posterior(fs(sb.GPPPInput("f", x1), 0.1), y1)
    p12 = sb.posterior(p1(sb.GPPPInput("f", x2), 0.1), y2)
    lp = handle_logpdf(sb, p12.fac, p12.delta)
    m, v = sb.mean_and_var(p12, sb.GPPPInput("f", xs))
    del p12, p1
    gc.collect()
    fj = fs(sb.BlockData(sb.GPPPInput("f", x1), sb.GPPPInput("f", x2)), 0.1)
    lpj = sb.logpdf(fj, y)
    mj, vj = sb.mean_and_var(sb.posterior(fj, y), sb.GPPPInput("f", xs))
    assert abs(lp - lpj) <= RTOL * abs(lpj), (lp, lpj)
    np.testing.assert_allclose(m, mj, rtol=RTOL, atol=1e-11)
    np.testing.assert_allclose(v, vj, rtol=RTOL, atol=1e-11)


def test_append_then_sharded_predict_on_two_gpus():
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2",
           "--master-addr", "127.0.0.1", "--master-port", "29571", os.path.join(ROOT, "tests", "dist_append_worker.py")]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=300)
    assert "APPEND_DIST_OK" in r.stdout, r.stdout[-2000:] + r.stderr[-3000:]
