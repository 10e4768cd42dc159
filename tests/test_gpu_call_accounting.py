"""sb_timings.kernel_launches counts every kernel an ABI call launches exactly once: for each single-GPU entry point
the delta a call adds must equal the CUDA kernels torch.profiler records for it, on both trailing paths.  Factors
and VFE handles the calls under test need but do not build themselves are made outside the profiled region; the
ones built under it stay at or below 8 block columns, where the (uncounted) wide-panel kernels of the int8 Ozaki
driver do not run."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


@pytest.fixture(params=[0, 1], ids=["dmma", "ozaki"])
def trailing(request, sb):
    ctx = sb.default_context()
    ctx.set_option("trailing", request.param)
    try:
        yield request.param
    finally:
        ctx.set_option("trailing", 0)


def launches(sb, fn):
    """(kernel_launches added by fn(), CUDA kernels the profiler records while fn runs)"""
    import torch
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile
    ctx = sb.default_context()
    torch.cuda.synchronize()
    before = ctx.timings()["kernel_launches"]
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    counted = ctx.timings()["kernel_launches"] - before
    kernels = [e for e in prof.events()
               if e.device_type == DeviceType.CUDA and not e.name.startswith(("Memcpy", "Memset"))]
    return counted, len(kernels)


def test_kernel_launches_match_profiler(sb, trailing):
    rng = np.random.default_rng(2)
    f = sb.gppp(lambda GP: dict(f=GP(sb.SEKernel())))
    x, xs, x2 = rng.uniform(0, 48, 1536), rng.uniform(0, 48, 300), rng.uniform(0, 48, 200)
    y, y2 = np.sin(x) + 0.3 * rng.standard_normal(1536), np.cos(x2)
    fx = f(sb.GPPPInput("f", x), 0.1)
    fx.factor()   # 12 block columns: the posterior sweeps below take the int8 path when trailing = 1
    post = sb.posterior(fx, y)
    xo, zo = rng.uniform(0, 200, 20000), np.linspace(0, 200, 1200)
    yo = np.sin(xo / 7)
    vfe, fxo = sb.VFE(f(sb.GPPPInput("f", zo), 1e-6)), f(sb.GPPPInput("f", xo), 0.1)
    ap = sb.ApproxPosteriorGP(vfe, fxo, yo)   # 10 block columns: int8 sweeps when trailing = 1
    vin = sb.finite._VfeInputs(vfe, fxo, yo)
    g = [np.zeros(2 * max(1, s.nterms)) for s in (vin.uu, vin.xu, vin.ffd)] + [np.empty(vin.m), np.empty(vin.n)]
    lib = sb.lib.load()

    def vfe_grad():
        h = ap.handle
        sb.lib.check(lib.sb_vfe_grad(h.ctx.h, h.h, C.byref(vin.uu), C.byref(vin.xu), C.byref(vin.ffd),
                                     C.byref(vin.nf), vin.delta.ctypes.data, *[a.ctypes.data for a in g]))

    calls = {
        "sb_cov_dense": lambda: sb.cov(f, sb.GPPPInput("f", xs)),
        "sb_cov_diag": lambda: sb.var(f, sb.GPPPInput("f", xs)),
        "sb_factor_create": lambda: f(sb.GPPPInput("f", x[:1000]), 0.1).factor(),
        "sb_logpdf": lambda: sb.logpdf(fx, y),
        "sb_factor_set_data": lambda: sb.posterior(fx, y),
        "sb_predict mean": lambda: post.mean(sb.GPPPInput("f", xs)),
        "sb_predict var": lambda: post.var(sb.GPPPInput("f", xs)),
        "sb_predict mean+var": lambda: post.mean_and_var(sb.GPPPInput("f", xs)),
        "sb_predict_cov": lambda: post.cov(sb.GPPPInput("f", xs)),
        "sb_predict_factor": lambda: post(sb.GPPPInput("f", xs), 0.2).factor(),
        "sb_factor_append + set_data": lambda: sb.posterior(post(sb.GPPPInput("f", x2), 0.2), y2),
        "sb_rand": lambda: sb.rand(fx, rng.standard_normal(1536)),
        "sb_logpdf_grad": lambda: sb.grad_logpdf(fx, y),
        "sb_vfe_create": lambda: sb.elbo(sb.VFE(f(sb.GPPPInput("f", zo[:1000]), 1e-6)), fxo, yo),
        "sb_vfe_grad": vfe_grad,
        "sb_vfe_predict": lambda: ap.mean_and_var(sb.GPPPInput("f", xs)),
        "sb_vfe_predict_cov": lambda: ap.cov(sb.GPPPInput("f", xs)),
    }
    launches(sb, calls["sb_cov_dense"])   # the profiler's first session starts CUPTI
    seen = {name: launches(sb, fn) for name, fn in calls.items()}
    assert all(k > 0 for _, k in seen.values()), seen
    assert {n: v for n, v in seen.items() if v[0] != v[1]} == {}, seen
