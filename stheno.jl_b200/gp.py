"""GP nodes, affine transformations and *plan lowering* for the CUDA hot path.

Host-side mirror of the reference's node types and operator surface
(Stheno.jl src/gp/{util,atomic_gp,derived_gp}.jl, src/affine_transformations/*.jl,
src/gaussian_process_probabilistic_programme.jl) -- same names, argument meaning and errors --
but NOT its evaluation strategy.  The reference evaluates `cov(f_p, f_q, x, x')` by an id-ordered
recursion that materialises an N x N' matrix per node (src/gp/derived_gp.jl:31-59).  Here every
process is lowered ONCE to the closed form (SURVEY.md Appendix B.3)

    f_p(x) = m_p(x) + sum_r  c_r * s_r(x) * a_r(g_r(x))         a_r: atomic leaf GP

and a covariance block becomes a flat term list for the device
(sum over pairs of terms that share the *same* atomic leaf, object identity as in
src/gp/atomic_gp.jl:36-38; no shared leaf => no term => the block is zeros).  User closures
(scale functions, input maps, means) are evaluated on the host, O(N); O(N^2)/O(N^3) work never
runs on the host.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Callable

import numpy as np

from . import lib as _lib
from .inputs import BlockData, ColVecs, GPPPInput, iter_points, npoints

# --------------------------------------------------------------------------------------
# KernelFunctions-like kernel objects (only what lowers to the device's fixed kernel family)
# --------------------------------------------------------------------------------------


class Kernel:
    def __add__(self, other):
        if not isinstance(other, Kernel):
            return NotImplemented
        return KernelSum(self, other)

    def __rmul__(self, c):
        return ScaledKernel(self, float(c))

    def __mul__(self, c):
        if isinstance(c, Kernel):
            raise NotImplementedError("kernel products are outside the CUDA hot-path scope")
        return ScaledKernel(self, float(c))

    def lowered(self):
        """-> list of (coeff, kernel_id, param, input_scale)."""
        raise NotImplementedError


class _Base(Kernel):
    kid = -1

    def lowered(self):
        return [(1.0, self.kid, 0.0, 1.0)]


class SEKernel(_Base):
    kid = _lib.K_SE


SqExponentialKernel = SEKernel


class Matern12Kernel(_Base):
    kid = _lib.K_MATERN12


ExponentialKernel = Matern12Kernel


class Matern32Kernel(_Base):
    kid = _lib.K_MATERN32


class Matern52Kernel(_Base):
    kid = _lib.K_MATERN52


class WhiteKernel(_Base):
    kid = _lib.K_WHITE


class ConstantKernel(Kernel):
    def __init__(self, c=1.0):
        self.c = float(c)

    def lowered(self):
        return [(1.0, _lib.K_CONST, self.c, 1.0)]


class ScaledKernel(Kernel):
    def __init__(self, k, s2):
        self.k, self.s2 = k, s2

    def lowered(self):
        return [(c * self.s2, kid, p, s) for (c, kid, p, s) in self.k.lowered()]


class KernelSum(Kernel):
    def __init__(self, a, b):
        self.a, self.b = a, b

    def lowered(self):
        return self.a.lowered() + self.b.lowered()


class TransformedKernel(Kernel):
    """k o ScaleTransform(s)."""

    def __init__(self, k, s):
        self.k, self.s = k, float(s)

    def lowered(self):
        return [(c, kid, p, s * self.s) for (c, kid, p, s) in self.k.lowered()]


def with_lengthscale(k: Kernel, ell: float) -> Kernel:
    return TransformedKernel(k, 1.0 / ell)


class GP:
    """AbstractGPs.GP: GP(kernel) zero mean, GP(c, kernel) constant mean, GP(fn, kernel)."""

    def __init__(self, *args):
        if len(args) == 1:
            self.mean_fn, self.kernel = 0.0, args[0]
        elif len(args) == 2:
            self.mean_fn, self.kernel = args
        else:
            raise TypeError("GP(kernel) or GP(mean, kernel)")
        if not isinstance(self.kernel, Kernel):
            raise TypeError("GP needs a Kernel")

    def mean_vector(self, x):
        if callable(self.mean_fn):
            return np.array([self.mean_fn(v) for v in iter_points(x)], dtype=np.float64)
        return np.full(npoints(x), float(self.mean_fn), dtype=np.float64)


# --------------------------------------------------------------------------------------
# Nodes (src/gp/util.jl:18-25, atomic_gp.jl:11-22, derived_gp.jl:7-17)
# --------------------------------------------------------------------------------------


class GPC:
    """GP collection counter."""

    def __init__(self):
        self.n = 0


class SthenoAbstractGP:
    n: int
    gpc: GPC

    # operator surface (addition.jl:8-12,62-65; product.jl:11-13,73; compose.jl:8)
    def __add__(self, other):
        return _add(self, other)

    def __radd__(self, other):
        return _add(other, self)

    def __sub__(self, other):
        if isinstance(other, SthenoAbstractGP):
            return _add(self, -other)
        return _add(self, -other)

    def __rsub__(self, other):
        return _add(other, -self)

    def __mul__(self, other):
        return _mul(other, self)

    def __rmul__(self, other):
        return _mul(other, self)

    def __neg__(self):
        return _mul(-1, self)

    def __matmul__(self, g):
        """`f @ g` stands for the reference's `f ∘ g`."""
        return compose(self, g)

    def __call__(self, x, noise=1e-18):
        from .finite import FiniteGP
        return FiniteGP(self, x, noise)


class AtomicGP(SthenoAbstractGP):
    def __init__(self, gp, gpc: GPC):
        self.gp = gp
        self.n = gpc.n + 1
        self.gpc = gpc
        gpc.n += 1


def atomic(gp, gpc: GPC) -> AtomicGP:
    return AtomicGP(gp, gpc)


class DerivedGP(SthenoAbstractGP):
    def __init__(self, args, gpc: GPC):
        self.args = args
        self.n = gpc.n + 1
        self.gpc = gpc
        gpc.n += 1


def _add(a, b):
    if isinstance(a, SthenoAbstractGP) and isinstance(b, SthenoAbstractGP):
        assert a.gpc is b.gpc, "processes belong to different GPCs"  # addition.jl:9
        return DerivedGP(("+", a, b), a.gpc)
    if isinstance(b, SthenoAbstractGP):
        return DerivedGP(("+known", a, b), b.gpc)
    return DerivedGP(("+known", b, a), a.gpc)


def _mul(f, g):
    if isinstance(f, SthenoAbstractGP) and isinstance(g, SthenoAbstractGP):
        raise ValueError("Cannot multiply two GPs together.")  # ArgumentError, product.jl:13
    if isinstance(g, SthenoAbstractGP):
        return DerivedGP(("*", f, g), g.gpc)
    return DerivedGP(("*", g, f), f.gpc)


def compose(f: SthenoAbstractGP, g) -> DerivedGP:
    return DerivedGP(("o", f, g), f.gpc)


def cross(fs):
    """src/affine_transformations/cross.jl:37-45 (kept for API parity; allocates an id)."""
    assert len(fs) >= 1
    assert all(f.gpc is fs[0].gpc for f in fs)
    return DerivedGP(("cross", list(fs)), fs[0].gpc)


# -- input maps (compose.jl:36-127) ------------------------------------------------------


def map_input(g, x):
    if hasattr(g, "broadcast"):
        return g.broadcast(x)
    pts = [g(v) for v in iter_points(x)]
    if len(pts) and np.ndim(pts[0]) == 1:
        return ColVecs(np.stack(pts, axis=1))
    return np.asarray(pts, dtype=np.float64)


class Stretch:
    def __init__(self, l):
        self.l = l

    def __call__(self, x):
        return self.l * x if np.ndim(self.l) == 0 else np.asarray(self.l) @ x

    def broadcast(self, x):
        if isinstance(x, ColVecs):
            return ColVecs(self.l * x.X if np.ndim(self.l) == 0 else np.asarray(self.l) @ x.X)
        return self.l * np.asarray(x)


def stretch(f, l):
    if np.ndim(l) == 1:
        l = np.diag(np.asarray(l, dtype=np.float64))
    return compose(f, Stretch(l))


class Select:
    def __init__(self, idx):
        self.idx = idx

    def __call__(self, x):
        return x[self.idx]

    def broadcast(self, x):
        if not isinstance(x, ColVecs):
            raise TypeError("select needs ColVecs inputs")
        if isinstance(self.idx, (int, np.integer)):
            return x.X[self.idx, :]
        return ColVecs(x.X[np.asarray(self.idx), :])


def select(f, idx):
    return compose(f, Select(idx))


class Periodic:
    def __init__(self, f):
        self.f = f

    def __call__(self, t):
        w = (2 * math.pi * self.f) * t
        return np.array([math.cos(w), math.sin(w)])

    def broadcast(self, x):
        w = (2 * math.pi * self.f) * np.asarray(x)
        return ColVecs(np.vstack([np.cos(w), np.sin(w)]))


def periodic(g, f):
    return compose(g, Periodic(f))


class Shift:
    def __init__(self, a):
        self.a = a

    def __call__(self, x):
        return x - self.a

    def broadcast(self, x):
        if isinstance(x, ColVecs):
            a = np.asarray(self.a)
            return ColVecs(x.X - (a.reshape(-1, 1) if a.ndim == 1 else a))
        return np.asarray(x) - self.a


def shift(f, a):
    return compose(f, Shift(a))


def additive_gp(fs, indices=None):
    """additive_gp.jl:10,26-29: sum_i fs[i] o Select(indices[i])."""
    if indices is None:
        indices = list(range(len(fs)))
    proj = [compose(f, Select(idx)) for f, idx in zip(fs, indices)]
    out = proj[0]
    for p in proj[1:]:
        out = out + p
    return out


# --------------------------------------------------------------------------------------
# GPPP (gaussian_process_probabilistic_programme.jl:13-43, :166-201)
# --------------------------------------------------------------------------------------


class GPPP:
    def __init__(self, fs: dict, gpc: GPC):
        self.fs = dict(fs)
        self.gpc = gpc

    def __call__(self, x, noise=1e-18):
        from .finite import FiniteGP
        return FiniteGP(self, x, noise)


GaussianProcessProbabilisticProgramme = GPPP


def gppp(build: Callable) -> GPPP:
    """Python spelling of `@gppp let ... end`: `build(GP)` is called with a `GP` constructor
    that wraps every `GP(...)` into `atomic(GP(...), gpc)` (what the macro's postwalk does,
    gppp.jl:194-197) and must return the dict of named processes.

        f = gppp(lambda GP: (lambda f1, f2: dict(f1=f1, f2=f2, f3=f1 + f2))(
                     GP(SEKernel()), GP(Matern52Kernel())))
    """
    gpc = GPC()
    fs = build(lambda *a: atomic(GP(*a), gpc))
    if not isinstance(fs, dict):
        raise RuntimeError("gppp needs a let block.")  # gppp.jl:170
    return GPPP(fs, gpc)


def extract_components(f: GPPP, x):
    """gppp.jl:25,27-30,32-43 -> (list of processes, list of raw input vectors, BlockData|None).
    Unlike the reference no `cross` node is allocated (cross.jl:39 bumps the GPC on every call)."""
    if isinstance(x, GPPPInput):
        return [f.fs[x.p]], [x.x]
    if isinstance(x, BlockData):
        ps, vs = [], []
        for b in x.X:
            p, v = extract_components(f, b)
            ps += p
            vs += v
        return ps, vs
    x = list(x)  # vector of (symbol, feature) tuples: regroup by first occurrence
    symbols = [t[0] for t in x]
    feats = [t[1] for t in x]
    uniq = []
    for s in symbols:
        if s not in uniq:
            uniq.append(s)
    blocks = []
    for s in uniq:
        sel = [feats[i] for i, t in enumerate(symbols) if t == s]
        if len(sel) and np.ndim(sel[0]) == 1:
            blocks.append(GPPPInput(s, ColVecs(np.stack(sel, axis=1))))
        else:
            blocks.append(GPPPInput(s, np.asarray(sel)))
    return extract_components(f, BlockData(blocks))


# --------------------------------------------------------------------------------------
# Lowering
# --------------------------------------------------------------------------------------


@dataclass
class LTerm:
    atom: AtomicGP            # the leaf whose GP supplies the kernel
    coeff: float
    scale: np.ndarray | None  # per-point scale vector or None (== ones)
    z: object                 # inputs seen by the atom's kernel (1-D array or ColVecs)
    key: tuple = ()           # identity of the leaf: ids of the chain of wrapping atomics (nested GPPPs)

    def same_leaf(self, other) -> bool:
        """Object identity as in src/gp/atomic_gp.jl:36-38; for a GPPP used as an atomic inside
        another GPPP the whole chain of wrappers must coincide (two different outer atomics
        wrapping the same inner programme are independent)."""
        return self.atom is other.atom and self.key == other.key


def lower(p: SthenoAbstractGP, x):
    """-> (mean vector, [LTerm]) of process p at inputs x (SURVEY.md App. B.3)."""
    if isinstance(p, AtomicGP):
        if isinstance(p.gp, GPPP):
            # a whole programme used as one atomic (test/gaussian_process_probabilistic_programme.jl:
            # 107-120): its inputs are themselves GPPPInputs naming the inner process
            if not isinstance(x, GPPPInput):
                raise NotImplementedError("nested GPPP: only GPPPInput inner inputs are lowered (no BlockData / tuple vectors)")
            m, terms = lower(p.gp.fs[x.p], x.x)
            return m, [LTerm(t.atom, t.coeff, t.scale, t.z, (id(p),) + t.key) for t in terms]
        return p.gp.mean_vector(x), [LTerm(p, 1.0, None, x)]
    op = p.args[0]
    if op == "+":
        ma, ta = lower(p.args[1], x)
        mb, tb = lower(p.args[2], x)
        return ma + mb, ta + tb
    if op == "+known":
        b = p.args[1]
        m, t = lower(p.args[2], x)
        bx = np.array([b(v) for v in iter_points(x)], dtype=np.float64) if callable(b) else float(b)
        return bx + m, t
    if op == "*":
        s = p.args[1]
        m, t = lower(p.args[2], x)
        if callable(s):
            sx = np.array([s(v) for v in iter_points(x)], dtype=np.float64)
            out = [LTerm(u.atom, u.coeff, sx if u.scale is None else sx * u.scale, u.z, u.key) for u in t]
            return sx * m, out
        s = float(s)
        return s * m, [LTerm(u.atom, s * u.coeff, u.scale, u.z, u.key) for u in t]
    if op == "o":
        return lower(p.args[1], map_input(p.args[2], x))
    if op == "cross":
        raise TypeError("cross nodes are lowered at the block level")
    raise AssertionError(op)


def _as_point_major(z, scale: float):
    """(n, dim) C-contiguous float64 array of kernel inputs, times the kernel's input scale."""
    if hasattr(z, "data_ptr"):  # torch CUDA tensor already resident in HBM: (n,) or (n, dim)
        import torch
        if z.dtype != torch.float64:
            raise NotImplementedError("device inputs must be float64")
        a = z.contiguous().reshape(z.shape[0], -1)
        return a if scale == 1.0 else a * scale
    if isinstance(z, ColVecs):
        a = np.ascontiguousarray(z.X.T, dtype=np.float64)
    else:
        a = np.asarray(z)
        if a.dtype == np.float32:
            raise NotImplementedError("Float32 inputs: SB_F32 path is reserved, not built")
        a = np.ascontiguousarray(a, dtype=np.float64).reshape(-1, 1)
    if scale != 1.0:
        a = a * scale
    return a


class SpecBuilder:
    """Accumulates arrays / terms / blocks and emits the ctypes `sb_covspec`."""

    def __init__(self, nrows, ncols, symmetric):
        self.nrows, self.ncols, self.symmetric = int(nrows), int(ncols), int(symmetric)
        self.arrays: list[np.ndarray] = []
        self.dims: list[int] = []
        self._cache: dict = {}
        self.terms: list[tuple] = []
        self.term_meta: list[tuple] = []
        self.blocks: list[tuple] = []

    def _input(self, z, scale):
        key = ("z", id(z.X) if isinstance(z, ColVecs) else id(z), scale)
        if key not in self._cache:
            a = _as_point_major(z, scale)
            self._cache[key] = len(self.arrays)
            self.arrays.append(a)
            self.dims.append(a.shape[1])
            self._keep = getattr(self, "_keep", []) + [z]  # keep ids alive
        return self._cache[key]

    def _scale(self, s):
        if s is None:
            return -1
        key = ("s", id(s))
        if key not in self._cache:
            self._cache[key] = len(self.arrays)
            self.arrays.append(np.ascontiguousarray(s, dtype=np.float64))
            self.dims.append(0)
            self._keep = getattr(self, "_keep", []) + [s]
        return self._cache[key]

    def add_block(self, row0, nrows, col0, ncols, lt_rows, lt_cols):
        term0 = len(self.terms)
        for a in lt_rows:
            for b in lt_cols:
                if not a.same_leaf(b):
                    continue  # independent leaves: zeros (atomic_gp.jl:36-38)
                for ci, (kc, kid, param, iscale) in enumerate(a.atom.gp.kernel.lowered()):
                    # gradient bookkeeping: which leaf / kernel component this term belongs to and the
                    # factor its coefficient carries besides the component's own multiplier kc
                    self.term_meta.append((a.atom, a.key, ci, kid, a.coeff * b.coeff, kc, iscale))
                    zl = self._input(a.z, iscale)
                    zr = self._input(b.z, iscale)
                    if self.dims[zl] != self.dims[zr]:
                        raise ValueError("input dimension mismatch between the two sides of a kernel")
                    self.terms.append((kid, zl, zr, self._scale(a.scale), self._scale(b.scale),
                                       a.coeff * b.coeff * kc, param))
        self.blocks.append((int(row0), int(nrows), int(col0), int(ncols), term0, len(self.terms) - term0))

    def finish(self):
        C = _lib.C
        arrs = (_lib.sb_array * max(1, len(self.arrays)))()
        for i, a in enumerate(self.arrays):
            arrs[i].data = _lib.ptr(a)
            arrs[i].n = a.shape[0]
            arrs[i].dim = self.dims[i]
        terms = (_lib.sb_term * max(1, len(self.terms)))()
        for i, (kid, zl, zr, sl, sr, coeff, param) in enumerate(self.terms):
            t = terms[i]
            t.kernel, t.zl, t.zr, t.sl, t.sr, t.coeff, t.param = kid, zl, zr, sl, sr, coeff, param
        blocks = (_lib.sb_block * max(1, len(self.blocks)))()
        for i, (r0, nr, c0, nc, t0, nt) in enumerate(self.blocks):
            b = blocks[i]
            b.row0, b.nrows, b.col0, b.ncols, b.term0, b.nterms = r0, nr, c0, nc, t0, nt
        spec = _lib.sb_covspec()
        spec.nrows, spec.ncols, spec.symmetric = self.nrows, self.ncols, self.symmetric
        spec.narrays, spec.arrays = len(self.arrays), arrs
        spec.nterms, spec.terms = len(self.terms), terms
        spec.nblocks, spec.blocks = len(self.blocks), blocks
        spec._keep = (arrs, terms, blocks, self.arrays, getattr(self, "_keep", None))
        spec._meta = self.term_meta
        return spec


class Lowered:
    """A GPPP (or bare Stheno process) indexed at an input collection, lowered once:
    per block the mean vector and the term list."""

    def __init__(self, f, x):
        if isinstance(f, GPPP):
            procs, xs = extract_components(f, x)
        elif isinstance(f, SthenoAbstractGP):
            if isinstance(x, BlockData) and isinstance(f, DerivedGP) and f.args[0] == "cross":
                procs, xs = list(f.args[1]), list(x.X)
            else:
                procs, xs = [f], [x]
        else:
            raise TypeError(f"cannot index a {type(f).__name__}")
        self.procs, self.xs = procs, xs
        self.lengths = [npoints(v) for v in xs]
        self.offsets = np.concatenate([[0], np.cumsum(self.lengths)]).astype(np.int64)
        self.n = int(self.offsets[-1])
        self.means, self.terms = [], []
        for p, v in zip(procs, xs):
            m, t = lower(p, v)
            self.means.append(np.asarray(m, dtype=np.float64) * np.ones(npoints(v)))
            self.terms.append(t)

    def mean(self):
        return np.concatenate(self.means) if self.means else np.zeros(0)


def spec_symmetric(lx: Lowered):
    """cov(f, x) for the factor path: blocks on/below the block diagonal only."""
    sb = SpecBuilder(lx.n, lx.n, 1)
    for i in range(len(lx.procs)):
        for j in range(i + 1):
            sb.add_block(lx.offsets[i], lx.lengths[i], lx.offsets[j], lx.lengths[j], lx.terms[i], lx.terms[j])
    return sb.finish()


def spec_dense(lx: Lowered, ly: Lowered):
    """cov(f, x, x'): all blocks."""
    sb = SpecBuilder(lx.n, ly.n, 0)
    for i in range(len(lx.procs)):
        for j in range(len(ly.procs)):
            sb.add_block(lx.offsets[i], lx.lengths[i], ly.offsets[j], ly.lengths[j], lx.terms[i], ly.terms[j])
    return sb.finish()


def spec_diag(lx: Lowered, ly: Lowered | None = None):
    """var(f, x) / var(f, x, x'): paired points, block by block (cross.jl:64-67,74-77)."""
    ly = lx if ly is None else ly
    if lx.lengths != ly.lengths:
        raise ValueError("var(f, x, x') needs inputs of identical block lengths")
    sb = SpecBuilder(lx.n, lx.n, 0)
    for i in range(len(lx.procs)):
        sb.add_block(lx.offsets[i], lx.lengths[i], lx.offsets[i], lx.lengths[i], lx.terms[i], ly.terms[i])
    return sb.finish()
