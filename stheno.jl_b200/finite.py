"""FiniteGP-level API on the CUDA path: logpdf / posterior / marginals / rand / elbo.

Mirror of the AbstractGPs entry points the reference reaches through Stheno
(`logpdf(f(x, s), y)`, `posterior`, `mean/cov/var/marginals`, `rand`, `elbo(VFE(fz), fx, y)`;
call sites Stheno.jl README.md:61-96, src/gp/sparse_finite_gp.jl:52-62,
test/gp/util.jl:9-88).  The interception is one level above the reference's seam
(docs/src/internals.md:8-24): the covariance matrix is assembled, factorised and solved on the
device through the C ABI (include/stheno_b200.h) and never exists on the host.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import lib as _lib
from .gp import GPPP, Lowered, SthenoAbstractGP, spec_dense, spec_diag, spec_symmetric
from .inputs import BlockData, ColVecs, npoints


def _ctx():
    return _lib.default_context()


def _out(n, like=None, shape=None):
    return np.empty(shape if shape is not None else n, dtype=np.float64)


class _Factor:
    """Owner of an `sb_factor*` (device-resident Cholesky factor)."""

    def __init__(self, h, ctx, n):
        self.h, self.ctx, self.n = h, ctx, n
        self.alpha_owner = None  # the PosteriorGP whose alpha currently sits in the device handle

    def __del__(self):
        try:
            if self.h and self.ctx.h:  # the ctx owns the pool the factor returns its memory to
                _lib.load().sb_factor_destroy(self.h)
            self.h = None
        except Exception:
            pass

    def logdet(self):
        v = C.c_double()
        _lib.check(_lib.load().sb_factor_logdet(self.ctx.h, self.h, C.byref(v)))
        return v.value

    def export(self) -> np.ndarray:
        """Checkpoint: header | packed L | diagonal-block inverses | alpha as one uint8 array."""
        n = C.c_int64(0)
        lib = _lib.load()
        _lib.check(lib.sb_factor_export_size(self.ctx.h, self.h, C.byref(n)))
        blob = np.empty(n.value, dtype=np.uint8)
        _lib.check(lib.sb_factor_export(self.ctx.h, self.h, blob.ctypes.data, n.value))
        return blob

    @staticmethod
    def load(blob: np.ndarray, n: int, ctx=None) -> "_Factor":
        ctx = ctx or _ctx()
        blob = np.ascontiguousarray(blob, dtype=np.uint8)
        h = C.c_void_p()
        _lib.check(_lib.load().sb_factor_import(ctx.h, blob.ctypes.data, blob.size, C.byref(h)))
        return _Factor(h, ctx, n)

    def to_dense_L(self):
        L = np.empty((self.n, self.n), dtype=np.float64, order="F")
        _lib.check(_lib.load().sb_factor_get_L(self.ctx.h, self.h, L.ctypes.data))
        return L


def _noise_struct(noise, n):
    ns = _lib.sb_noise()
    keep = None
    if np.ndim(noise) == 0:
        ns.sigma2 = float(noise)
        ns.diag = None
        ns.dense = None
    elif np.ndim(noise) == 1:
        keep = np.ascontiguousarray(noise, dtype=np.float64)
        if keep.shape[0] != n:
            raise ValueError("noise vector length mismatch")
        ns.sigma2 = 0.0
        ns.diag = keep.ctypes.data
        ns.dense = None
    else:
        keep = np.asfortranarray(noise, dtype=np.float64)
        if keep.shape != (n, n):
            raise ValueError("noise matrix shape mismatch")
        ns.sigma2 = 0.0
        ns.diag = None
        ns.dense = keep.ctypes.data
    ns._keep = keep
    return ns


class FiniteGP:
    """`f(x, noise)`: a GPPP / Stheno process (or a posterior) at a finite input collection."""

    def __init__(self, f, x, noise=1e-18):
        self.f, self.x, self.noise = f, x, noise
        self._factor = None
        self._lowered = None
        if isinstance(f, (GPPP, SthenoAbstractGP)):
            self.prior, self.post = f, None
        elif isinstance(f, _Posterior):
            self.prior, self.post = f.prior, f
        else:
            raise TypeError(f"cannot index a {type(f).__name__}")

    def __len__(self):
        return npoints(self.x)

    @property
    def lowered(self) -> Lowered:
        if self._lowered is None:
            self._lowered = Lowered(self.prior, self.x)
        return self._lowered

    def noise_diag(self):
        n = len(self)
        if np.ndim(self.noise) == 0:
            return np.full(n, float(self.noise))
        if np.ndim(self.noise) == 1:
            return np.asarray(self.noise, dtype=np.float64)
        return np.diag(self.noise)

    # -- exact factorisation of cov(fx) = cov(f, x) + Sigma_y (device) ----------------------
    def factor(self) -> _Factor:
        if self.post is not None:
            if not isinstance(self.post, PosteriorGP):
                raise NotImplementedError("joint sampling from an approximate (VFE) posterior is not on the CUDA path yet")
            if self._factor is None:
                # cholesky(cov(f_post(x*, noise))): posterior covariance formed and factorised on device
                post = self.post
                ls = Lowered(post.prior, self.x)
                cross, full = spec_dense(ls, post.lx), spec_dense(ls, ls)
                ns = _noise_struct(self.noise, ls.n)
                h, info = C.c_void_p(), C.c_int64(0)
                st = _lib.load().sb_predict_factor(post.fac.ctx.h, post.fac.h, C.byref(cross), C.byref(full),
                                                   C.byref(ns), C.byref(h), C.byref(info))
                _lib.check(st, info)
                self._factor = _Factor(h, post.fac.ctx, ls.n)
            return self._factor
        if self._factor is None:
            lx = self.lowered
            spec = spec_symmetric(lx)
            ns = _noise_struct(self.noise, lx.n)
            h = C.c_void_p()
            info = C.c_int64(0)
            ctx = _ctx()
            st = _lib.load().sb_factor_create(ctx.h, C.byref(spec), C.byref(ns), C.byref(h), C.byref(info))
            _lib.check(st, info)
            self._factor = _Factor(h, ctx, lx.n)
        return self._factor


class LogpdfGradient:
    """Gradient of logpdf(fx, y) w.r.t. the parameters the lowered plan exposes (SURVEY 8f.1).

    noise:    d/d sigma^2 (scalar noise) or d/d diag(Sigma_y) (vector noise).
    kernels:  list of dicts, one per (atomic leaf, kernel component): `atom`, `component` (index into
              the leaf kernel's lowered sum), `kernel_id`, `coeff` / `input_scale` (current values),
              `dcoeff` = d/d(component multiplier, i.e. the kernel variance),
              `dlogscale` = d/d log(input scale)  (= -d/d log(lengthscale)).
    The caller applies its own chain rule, exactly as Zygote does through user code in the reference."""

    def __init__(self, noise, kernels):
        self.noise, self.kernels = noise, kernels

    def for_atom(self, atom, component=0):
        for k in self.kernels:
            if k["atom"] is atom and k["component"] == component:
                return k
        raise KeyError("no such leaf / component in this gradient")


def grad_logpdf(fx: "FiniteGP", y) -> LogpdfGradient:
    """d logpdf(fx, y) / d theta = 1/2 tr((alpha alpha' - K^-1) dK/dtheta) on the device."""
    if fx.post is not None or isinstance(fx, SparseFiniteGP):
        raise NotImplementedError("grad_logpdf: prior FiniteGPs only")
    if np.ndim(fx.noise) == 2:
        raise NotImplementedError("grad_logpdf: scalar or diagonal observation noise")
    post = posterior(fx, y)
    post._install_alpha()
    lx = fx.lowered
    spec = spec_symmetric(lx)
    g = np.zeros(2 * max(1, spec.nterms), dtype=np.float64)
    qd = np.empty(lx.n, dtype=np.float64)
    fac = post.fac
    _lib.check(_lib.load().sb_logpdf_grad(fac.ctx.h, fac.h, C.byref(spec), g.ctypes.data, qd.ctypes.data))
    agg = {}
    _aggregate_terms(agg, spec, g)
    noise = float(qd.sum()) if np.ndim(fx.noise) == 0 else qd
    return LogpdfGradient(noise, list(agg.values()))


def _aggregate_terms(agg, spec, g):
    """Add the per-term gradient g (g[2t] = d/d coeff_t, g[2t+1] = d/d log input scale_t) of `spec` into the
    per-(leaf, kernel component) entries of `agg`."""
    for t, (atom, key, ci, kid, pair_coeff, kc, iscale) in enumerate(spec._meta):
        e = agg.setdefault((id(atom), key, ci), dict(atom=atom, component=ci, kernel_id=kid, coeff=kc,
                                                    input_scale=iscale, dcoeff=0.0, dlogscale=0.0))
        e["dcoeff"] += g[2 * t] * pair_coeff       # term coefficient = pair_coeff * kc
        e["dlogscale"] += g[2 * t + 1]


def save_factor(fx: "FiniteGP") -> np.ndarray:
    """Checkpoint the device-resident Cholesky factor of `fx` (SURVEY 8f.4)."""
    return fx.factor().export()


def load_factor(fx: "FiniteGP", blob: np.ndarray) -> "FiniteGP":
    """Resume: install a checkpointed factor into `fx` (same prior, inputs and noise as when saved)
    instead of re-assembling and re-factorising."""
    if fx.post is not None:
        raise NotImplementedError("load_factor: prior FiniteGPs only")
    fx._factor = _Factor.load(blob, len(fx))
    return fx


# -- statistics --------------------------------------------------------------------------------


def _prior_mean(prior, x):
    return Lowered(prior, x).mean()


def mean(f, x=None):
    if isinstance(f, FiniteGP):
        return mean(f.f, f.x)
    if isinstance(f, SparseFiniteGP):
        return mean(f.fobs)
    if isinstance(f, _Posterior):
        return f.mean(x)
    return _prior_mean(f, x)


def cov(f, x=None, y=None):
    """cov(fx) | cov(fx, gx) | cov(f, x) | cov(f, x, x')  -> host matrix (parity / small N)."""
    if isinstance(f, SparseFiniteGP):
        raise RuntimeError(COVARIANCE_ERROR)
    if isinstance(f, FiniteGP):
        if isinstance(x, FiniteGP):
            if f.post is not None or x.post is not None or f.prior is not x.prior:
                raise NotImplementedError("cov(fx, gx) needs two FiniteGPs of the same prior")
            return cov(f.prior, f.x, x.x)
        K = cov(f.f, f.x)
        if np.ndim(f.noise) == 2:
            return K + np.asarray(f.noise)
        K[np.diag_indices_from(K)] += f.noise_diag()
        return K
    if isinstance(f, _Posterior):
        return f.cov(x, y)
    lx = Lowered(f, x)
    ly = lx if y is None else Lowered(f, y)
    spec = spec_dense(lx, ly)
    K = np.empty((lx.n, ly.n), dtype=np.float64, order="F")
    if K.size:
        _lib.check(_lib.load().sb_cov_dense(_ctx().h, C.byref(spec), K.ctypes.data))
    return K


def var(f, x=None, y=None):
    if isinstance(f, FiniteGP):
        return var(f.f, f.x) + f.noise_diag()
    if isinstance(f, _Posterior):
        return f.var(x)
    lx = Lowered(f, x)
    ly = None if y is None else Lowered(f, y)
    spec = spec_diag(lx, ly)
    v = np.empty(lx.n, dtype=np.float64)
    if v.size:
        _lib.check(_lib.load().sb_cov_diag(_ctx().h, C.byref(spec), v.ctypes.data))
    return v


def mean_and_var(f, x=None):
    if isinstance(f, FiniteGP):
        if f.post is not None:
            m, v = f.post.mean_and_var(f.x)
            return m, v + f.noise_diag()
        return mean(f), var(f)
    if isinstance(f, _Posterior):
        return f.mean_and_var(x)
    return mean(f, x), var(f, x)


def mean_and_cov(f, x=None):
    if isinstance(f, FiniteGP):
        return mean(f), cov(f)
    return mean(f, x), cov(f, x)


def marginals(fx):
    """`marginals(fx)` = Normal.(mean, sqrt.(var)) -> (mean, std) arrays."""
    if isinstance(fx, SparseFiniteGP):
        return marginals(fx.fobs)
    m, v = mean_and_var(fx)
    return m, np.sqrt(v)


def _finite_mean(fx):
    return fx.post.mean(fx.x) if fx.post is not None else fx.lowered.mean()


def logpdf(fx, y):
    """logpdf(fx, y) / logpdf(fx, Y) (columns of Y)."""
    if isinstance(fx, SparseFiniteGP):
        Y = np.asarray(y, dtype=np.float64)
        if Y.ndim == 2:
            return np.array([elbo(VFE(fx.finducing), fx.fobs, Y[:, j]) for j in range(Y.shape[1])])
        return elbo(VFE(fx.finducing), fx.fobs, Y)
    Y = np.asarray(y, dtype=np.float64)
    if Y.shape[0] != len(fx):
        raise ValueError("length(y) != length(fx)")
    m = _finite_mean(fx)
    delta = np.asfortranarray(Y - (m if Y.ndim == 1 else m[:, None]))
    S = 1 if Y.ndim == 1 else Y.shape[1]
    fac = fx.factor()
    out = (C.c_double * S)()
    _lib.check(_lib.load().sb_logpdf(fac.ctx.h, fac.h, delta.ctypes.data, S, out))
    return out[0] if Y.ndim == 1 else np.array(out[:])


def rand(fx, z):
    """rand(rng, fx[, S]) with the standard normals `z` (N or N x S) drawn by the caller:
    m .+ cholesky(cov(fx)).U' * z."""
    if isinstance(fx, SparseFiniteGP):
        return rand(fx.fobs, z)
    z = np.asarray(z, dtype=np.float64)
    S = 1 if z.ndim == 1 else z.shape[1]
    zz = np.asfortranarray(z.reshape(len(fx), S))
    out = np.empty((len(fx), S), dtype=np.float64, order="F")
    fac = fx.factor()
    _lib.check(_lib.load().sb_rand(fac.ctx.h, fac.h, zz.ctypes.data, S, out.ctypes.data))
    m = _finite_mean(fx)
    return out[:, 0] + m if z.ndim == 1 else out + m[:, None]


class _Posterior:
    """Predictions of a posterior process on the device.  A subclass supplies its ABI calls (`_PREDICT`: mean / var,
    `_COV`: dense covariance), its device handle (`_handle`) and the lowered inputs of its training side (`_train`)."""

    def __call__(self, x, noise=1e-18):
        return FiniteGP(self, x, noise)

    def _install_alpha(self):
        """Make the device handle hold this posterior's weights before a mean is predicted from it."""

    def _predict(self, x, want_mean, want_var):
        ls = Lowered(self.prior, x)
        cross = spec_dense(ls, self._train)
        pd = spec_diag(ls) if want_var else None
        m = np.empty(ls.n) if want_mean else None
        v = np.empty(ls.n) if want_var else None
        if want_mean:
            self._install_alpha()
        _lib.check(getattr(_lib.load(), self._PREDICT)(
            self._handle.ctx.h, self._handle.h, C.byref(cross), C.byref(pd) if pd is not None else None,
            m.ctypes.data if m is not None else None, v.ctypes.data if v is not None else None))
        if m is not None:
            m += ls.mean()
        return m, v

    def mean(self, x):
        return self._predict(x, True, False)[0]

    def var(self, x):
        return self._predict(x, False, True)[1]

    def mean_and_var(self, x):
        return self._predict(x, True, True)

    def cov(self, x, y=None):
        """cov(f_post, x) and cov(f_post, x, z).  The cross form evaluates the joint posterior covariance of the
        stacked inputs [x; z] on the device and returns its off-diagonal block."""
        if y is not None:
            nx = npoints(x)
            K = self.cov(_stack_inputs(self.prior, x, y))
            return np.asfortranarray(K[:nx, nx:])
        ls = Lowered(self.prior, x)
        cross = spec_dense(ls, self._train)
        full = spec_dense(ls, ls)
        K = np.empty((ls.n, ls.n), dtype=np.float64, order="F")
        _lib.check(getattr(_lib.load(), self._COV)(self._handle.ctx.h, self._handle.h, C.byref(cross), C.byref(full),
                                                   K.ctypes.data))
        return K


class PosteriorGP(_Posterior):
    """`posterior(fx, y)`: shares the device factor of `fx` and keeps ITS OWN alpha = C \\ (y - m)
    (AbstractGPs PosteriorGP stores (alpha, C, x, delta); `posterior` is a pure function, so two
    posteriors built from one fx must not see each other's data).
    cov(f_post, x, z) = K(x,z) - (C.U'\\K_{X,x})'(C.U'\\K_{X,z}) (AbstractGPs, SURVEY App. A)."""

    _PREDICT, _COV = "sb_predict", "sb_predict_cov"

    def __init__(self, fx: FiniteGP, y):
        y = np.asarray(y, dtype=np.float64)
        if y.shape != (len(fx),):
            raise ValueError("length(y) != length(fx)")
        self.prior, self.x = fx.prior, fx.x
        self.lx = fx.lowered
        self.fac = fx.factor()
        self.noise = fx.noise
        self.y = y
        self.delta = np.ascontiguousarray(y - self.lx.mean())
        lib = _lib.load()
        _lib.check(lib.sb_factor_set_data(self.fac.ctx.h, self.fac.h, self.delta.ctypes.data))
        self._alpha = np.empty(self.lx.n, dtype=np.float64)
        _lib.check(lib.sb_factor_alpha(self.fac.ctx.h, self.fac.h, self._alpha.ctypes.data))
        self.fac.alpha_owner = self

    @property
    def _handle(self):
        return self.fac

    @property
    def _train(self):
        return self.lx

    @property
    def alpha(self):
        return self._alpha.copy()

    def _install_alpha(self):
        if self.fac.alpha_owner is not self:
            _lib.check(_lib.load().sb_factor_set_alpha(self.fac.ctx.h, self.fac.h, self._alpha.ctypes.data))
            self.fac.alpha_owner = self


def _stack_inputs(prior, x, z):
    """[x; z] as one input collection of `prior` (BlockData for a GPPP, concatenation otherwise)."""
    if isinstance(prior, GPPP):
        return BlockData([x, z])
    if isinstance(x, ColVecs) and isinstance(z, ColVecs):
        return ColVecs(np.concatenate([x.X, z.X], axis=1))
    return np.concatenate([np.asarray(x, dtype=np.float64), np.asarray(z, dtype=np.float64)])


def _stack_noise(n1, s1, n2, s2):
    """Sigma_y of the stacked observations [x1; x2]: scalar / vector / matrix noises combined."""
    if np.ndim(s1) <= 1 and np.ndim(s2) <= 1:
        d1 = np.full(n1, float(s1)) if np.ndim(s1) == 0 else np.asarray(s1, dtype=np.float64)
        d2 = np.full(n2, float(s2)) if np.ndim(s2) == 0 else np.asarray(s2, dtype=np.float64)
        return np.concatenate([d1, d2])
    S = np.zeros((n1 + n2, n1 + n2))
    S[:n1, :n1] = np.diag(np.full(n1, float(s1))) if np.ndim(s1) == 0 else (np.diag(s1) if np.ndim(s1) == 1 else s1)
    S[n1:, n1:] = np.diag(np.full(n2, float(s2))) if np.ndim(s2) == 0 else (np.diag(s2) if np.ndim(s2) == 1 else s2)
    return S


def posterior(fx, y):
    if isinstance(fx, SparseFiniteGP):
        return approx_posterior(VFE(fx.finducing), fx.fobs, y)
    if isinstance(fx, VFE):
        raise TypeError("use posterior(VFE(fz), fx, y)")
    if fx.post is not None:
        # posterior(f_post(x2, s2), y2): sequential conditioning == conditioning the prior on the
        # stacked observations [x1; x2] with block-diagonal noise.  As AbstractGPs' update_chol, p1's
        # factor is extended on the device (sb_factor_append), not refactorised; p1 itself is unchanged.
        p1 = fx.post
        if not isinstance(p1, PosteriorGP):
            raise NotImplementedError("posterior of an approximate (VFE) posterior is not on the CUDA path")
        y2 = np.asarray(y, dtype=np.float64)
        if y2.shape != (len(fx),):
            raise ValueError("length(y) != length(fx)")
        n1, n2 = npoints(p1.x), len(fx)
        joint = FiniteGP(p1.prior, _stack_inputs(p1.prior, p1.x, fx.x), _stack_noise(n1, p1.noise, n2, fx.noise))
        l2 = fx.lowered
        cross, full = spec_dense(l2, p1.lx), spec_dense(l2, l2)
        ns = _noise_struct(fx.noise, l2.n)
        h, info = C.c_void_p(), C.c_int64(0)
        st = _lib.load().sb_factor_append(p1.fac.ctx.h, p1.fac.h, C.byref(cross), C.byref(full), C.byref(ns),
                                          C.byref(h), C.byref(info))
        _lib.check(st, info)
        joint._factor = _Factor(h, p1.fac.ctx, n1 + n2)
        return PosteriorGP(joint, np.concatenate([p1.y, y2]))
    return PosteriorGP(fx, y)


# -- VFE / elbo ----------------------------------------------------------------------------------

COVARIANCE_ERROR = (
    "The covariance matrix of a sparse GP can often be dense and can cause the computer to "
    "run out of memory. If you are sure you have enough memory, you can use `cov(f.fobs)`."
)


class VFE:
    def __init__(self, fz: FiniteGP):
        self.fz = fz


class SparseFiniteGP:
    """src/gp/sparse_finite_gp.jl:30-62."""

    def __init__(self, fobs: FiniteGP, finducing: FiniteGP):
        self.fobs, self.finducing = fobs, finducing

    def __len__(self):
        return len(self.fobs)


class _VfeHandle:
    def __init__(self, h, ctx):
        self.h, self.ctx = h, ctx

    def __del__(self):
        try:
            if self.h and self.ctx.h:
                _lib.load().sb_vfe_destroy(self.h)
            self.h = None
        except Exception:
            pass


class _VfeInputs:
    """The specs, noises and residual of elbo(VFE(fz), fx, y), built once for sb_vfe_create and sb_vfe_grad."""

    def __init__(self, v: VFE, fx: FiniteGP, y):
        fz = v.fz
        if fz.prior is not fx.prior:
            raise ValueError("VFE: inducing and observed FiniteGPs must share the prior")
        if np.ndim(fx.noise) > 1:
            raise NotImplementedError("VFE needs diagonal observation noise")
        y = np.asarray(y, dtype=np.float64)
        if y.shape != (len(fx),):
            raise ValueError("DimensionMismatch: length(y) != length(fx)")
        lz, lx = fz.lowered, fx.lowered
        self.uu = spec_symmetric(lz)
        self.xu = spec_dense(lx, lz)
        self.ffd = spec_diag(lx)
        self.nu, self.nf = _noise_struct(fz.noise, lz.n), _noise_struct(fx.noise, lx.n)
        self.delta = np.ascontiguousarray(y - lx.mean())
        self.n, self.m = lx.n, lz.n


def _vfe_create(v: VFE, fx: FiniteGP, y, inputs: _VfeInputs | None = None):
    a = inputs if inputs is not None else _VfeInputs(v, fx, y)
    h = C.c_void_p()
    out2 = (C.c_double * 2)()
    info = C.c_int64(0)
    ctx = _ctx()
    st = _lib.load().sb_vfe_create(ctx.h, C.byref(a.uu), C.byref(a.nu), C.byref(a.xu), C.byref(a.ffd),
                                   C.byref(a.nf), a.delta.ctypes.data, C.byref(h), out2, C.byref(info))
    _lib.check(st, info)
    return _VfeHandle(h, ctx), out2[0], out2[1]


def elbo(v, fx=None, y=None):
    if isinstance(v, SparseFiniteGP):
        return elbo(VFE(v.finducing), v.fobs, fx)
    return _vfe_create(v, fx, y)[1]


def dtc(v: VFE, fx: FiniteGP, y):
    return _vfe_create(v, fx, y)[2]


class ElboGradient(LogpdfGradient):
    """Gradient of elbo(VFE(fz), fx, y) w.r.t. the parameters the lowered plan exposes, with the elbo itself.

    elbo:            the value from the same device pass (one handle build gives value and gradient).
    noise:           d/d sigma^2 (scalar observation noise) or d/d diag(Sigma_y) (vector noise).
    inducing_noise:  d/d jitter (scalar fz.noise) or d/d its diagonal (vector fz.noise).
    kernels / for_atom(): as in LogpdfGradient, summed over cov(fz), cov(f, x, z) and var(f, x)."""

    def __init__(self, elbo, noise, inducing_noise, kernels):
        super().__init__(noise, kernels)
        self.elbo, self.inducing_noise = elbo, inducing_noise


def grad_elbo(v, fx=None, y=None) -> ElboGradient:
    """d elbo(VFE(fz), fx, y) / d theta on the device (also grad_elbo(sparse::SparseFiniteGP, y)): the reverse
    pass of sb_vfe_create streams K_fu in the same chunks (DESIGN.md §4)."""
    if isinstance(v, SparseFiniteGP):
        return grad_elbo(VFE(v.finducing), v.fobs, fx)
    if np.ndim(v.fz.noise) > 1:
        raise NotImplementedError("grad_elbo: scalar or diagonal inducing-point noise")
    a = _VfeInputs(v, fx, y)
    handle, e, _ = _vfe_create(v, fx, y, a)
    g_uu = np.zeros(2 * max(1, a.uu.nterms))
    g_xu = np.zeros(2 * max(1, a.xu.nterms))
    g_ff = np.zeros(2 * max(1, a.ffd.nterms))
    g_nu, g_nf = np.empty(a.m), np.empty(a.n)
    _lib.check(_lib.load().sb_vfe_grad(
        handle.ctx.h, handle.h, C.byref(a.uu), C.byref(a.xu), C.byref(a.ffd), C.byref(a.nf), a.delta.ctypes.data,
        g_uu.ctypes.data, g_xu.ctypes.data, g_ff.ctypes.data, g_nu.ctypes.data, g_nf.ctypes.data))
    agg = {}
    for spec, g in ((a.uu, g_uu), (a.xu, g_xu), (a.ffd, g_ff)):
        _aggregate_terms(agg, spec, g)
    noise = float(g_nf.sum()) if np.ndim(fx.noise) == 0 else g_nf
    inducing = float(g_nu.sum()) if np.ndim(v.fz.noise) == 0 else g_nu
    return ElboGradient(e, noise, inducing, list(agg.values()))


class ApproxPosteriorGP(_Posterior):
    """`posterior(VFE(fz), fx, y)`: the VFE handle holds its own weights.  cov(f_approx_post, x) =
    K** - B'B + (Lambda.U'\\B)'(Lambda.U'\\B) with B = U' \\ K_{z*} (AbstractGPs approx posterior)."""

    _PREDICT, _COV = "sb_vfe_predict", "sb_vfe_predict_cov"

    def __init__(self, v: VFE, fx: FiniteGP, y):
        self.prior = fx.prior
        self.lz = v.fz.lowered
        self.handle, self.elbo, self.dtc = _vfe_create(v, fx, y)

    @property
    def _handle(self):
        return self.handle

    @property
    def _train(self):
        return self.lz


def approx_posterior(v: VFE, fx: FiniteGP, y):
    return ApproxPosteriorGP(v, fx, y)
