"""stheno.jl_b200 -- H100-native dense-GP inference hot path behind the Stheno/AbstractGPs API.

Only what the path needs: `csrc/` (CUDA kernels + C ABI -> libstheno_b200.so), `lib.py` (ctypes
binding == what the Julia shim `ccall`s), `inputs.py` / `gp.py` / `finite.py` (host-side mirror
of the reference's operator surface: gppp, GPPPInput, BlockData, f(X, s2), logpdf, posterior,
elbo, split ...).  Import name: `stheno_jl_b200` (see /stheno_jl_b200.py at the repo root; the
directory keeps the reference's spelling and therefore is not itself a valid Python identifier).
"""
from .inputs import BlockData, ColVecs, GPPPInput, blocks, split, vcat  # noqa: F401
from .gp import (  # noqa: F401
    GP, GPC, GPPP, AtomicGP, ConstantKernel, DerivedGP, ExponentialKernel, Kernel, Matern12Kernel,
    Matern32Kernel, Matern52Kernel, Periodic, SEKernel, Select, Shift, SqExponentialKernel, Stretch,
    WhiteKernel, additive_gp, atomic, compose, cross, gppp, periodic, select, shift, stretch,
    with_lengthscale,
)
from .finite import (  # noqa: F401
    ApproxPosteriorGP, FiniteGP, PosteriorGP, SparseFiniteGP, VFE, approx_posterior, cov, dtc, elbo,
    ElboGradient, LogpdfGradient, grad_elbo, grad_logpdf, load_factor, logpdf, marginals, mean, mean_and_cov, mean_and_var, posterior, rand, save_factor, var,
)
from .lib import Context, PosDefException, SthenoB200Error, default_context, set_default_context  # noqa: F401
