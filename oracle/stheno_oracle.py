"""CPU ORACLE -- TEST INFRASTRUCTURE ONLY.  NOT A PRODUCT PATH.

A NumPy/SciPy(OpenBLAS) restatement of the reference algorithm for the dense-GP hot path
of Stheno.jl (commit 905f995, v0.8.2).  Only `tests/`,
`__graft_entry__.smoke()` and `bench.py`'s cpu_baseline / `--impl reference` leg may import
this module, and only as the checker / reported baseline.

PARITY STATUS: **parity unpinned numerically**.  The reference is Julia; no `julia` binary
exists in this image or on the GPU box, and the arithmetic (KernelFunctions.jl,
AbstractGPs.jl, Distances.jl, LAPACK) is un-vendored (Project.toml:6-22, no Manifest).  The
reference's own tests hold NO golden numbers for this path (SURVEY.md section 4) -- they pin
*relations* (cov(f,x)==kernelmatrix, independent atomics => zeros, elbo<=logpdf, elbo==logpdf
when Z==X, var==diag(cov), split row ranges ...).  Every one of those relations is ported to
tests/test_oracle_relations.py and pins this oracle; integer paths (BlockData indexing, split)
are pinned bit-exact.

Structure mirrors the reference so each function can cite the file:line it restates:
  * routing:  AtomicGP / DerivedGP / cross / + / * / compose  -> the *recursive* id-ordered
    algorithm of src/gp/derived_gp.jl:31-59 (NOT the flattened term plan the product uses, so
    the product's plan lowering is checked against the reference algorithm, not itself).
  * arithmetic: KernelFunctions `kernelmatrix` (Distances GEMM-trick pairwise, SURVEY App. A),
    AbstractGPs FiniteGP/logpdf/posterior/rand/VFE-elbo (SURVEY App. A).
"""
from __future__ import annotations

import math
from typing import Callable, Sequence

import numpy as np
import scipy.linalg as sla

# --------------------------------------------------------------------------------------
# Inputs: Vector{<:Real}  == 1-D numpy array;  ColVecs(X) with X of shape (D, N).
# --------------------------------------------------------------------------------------


class ColVecs:
    """KernelFunctions.ColVecs: a D x N matrix viewed as N vectors of length D."""

    def __init__(self, X):
        self.X = np.asarray(X)
        assert self.X.ndim == 2

    def __len__(self):
        return self.X.shape[1]

    def __getitem__(self, idx):
        if isinstance(idx, (int, np.integer)):
            return self.X[:, idx]
        return ColVecs(self.X[:, idx])

    def __eq__(self, other):
        return isinstance(other, ColVecs) and np.array_equal(self.X, other.X)


def _as_matrix(x):
    """(D, N) matrix of an input collection (1-D real vector -> 1 x N)."""
    if isinstance(x, ColVecs):
        return x.X
    x = np.asarray(x)
    if x.ndim == 1:
        return x.reshape(1, -1)
    raise TypeError("inputs must be a 1-D real vector or ColVecs")


def _length(x):
    if isinstance(x, (ColVecs, GPPPInput, BlockData)):
        return len(x)
    return len(x)


# --------------------------------------------------------------------------------------
# src/input_collection_types.jl
# --------------------------------------------------------------------------------------


class GPPPInput:
    """src/input_collection_types.jl:24-33: vector `x` tagged with process key `p`."""

    def __init__(self, p, x):
        self.p = p
        self.x = x

    def __len__(self):  # :29
        return _length(self.x)

    def __getitem__(self, idx):  # :31-33 (0-based here)
        if isinstance(idx, (int, np.integer)):
            return (self.p, self.x[idx])
        return [(self.p, v) for v in _iter_points(self.x[idx])]

    def __iter__(self):
        for v in _iter_points(self.x):
            yield (self.p, v)

    def __eq__(self, other):
        if isinstance(other, GPPPInput):
            return self.p == other.p and _points_equal(self.x, other.x)
        return NotImplemented


def _iter_points(x):
    if isinstance(x, ColVecs):
        for i in range(len(x)):
            yield x.X[:, i]
    elif isinstance(x, (GPPPInput, BlockData)):
        yield from x
    else:
        yield from x


def _points_equal(a, b):
    if isinstance(a, ColVecs) or isinstance(b, ColVecs):
        return isinstance(a, ColVecs) and a == b
    if isinstance(a, (GPPPInput, BlockData)):
        return a == b
    return np.array_equal(np.asarray(a), np.asarray(b))


class BlockData:
    """src/input_collection_types.jl:61-95: ordered ragged collection of input vectors that
    behaves as one flat vector (integer semantics are bit-exact requirements)."""

    def __init__(self, *xs):
        if len(xs) == 1 and isinstance(xs[0], list):
            xs = xs[0]
        self.X = list(xs)

    def __len__(self):  # :69
        return sum(_length(b) for b in self.X)

    def locate(self, n):
        """0-based linear index -> (block, offset); restates the while loop of :71-78."""
        b = 0
        while n >= _length(self.X[b]):
            n -= _length(self.X[b])
            b += 1
        return b, n

    def __getitem__(self, n):
        b, off = self.locate(int(n))
        return self.X[b][off]

    def __iter__(self):
        for b in self.X:
            yield from _iter_points(b)

    def __eq__(self, other):  # :80
        return (isinstance(other, BlockData) and len(self.X) == len(other.X)
                and all(_points_equal(a, b) for a, b in zip(self.X, other.X)))

    def blocks(self):  # :82
        return self.X

    def view(self, b, n):  # :84
        return self.X[b][n]

    def eachindex(self):  # :88-91  (1-based, as BlockArray(1:sum, lengths))
        lengths = [_length(b) for b in self.X]
        out, start = [], 1
        for L in lengths:
            out.append(np.arange(start, start + L))
            start += L
        return out


def vcat(*xs):  # :93-95
    return BlockData(list(xs))


def get_indices(x: BlockData):
    """gppp.jl:131-134  (1-based inclusive ranges, as in the reference)."""
    lengths = [_length(b) for b in x.X]
    sz = np.cumsum(lengths)
    return [(int(sz[n] - lengths[n] + 1), int(sz[n])) for n in range(len(lengths))]


def split(x: BlockData, Y):
    """gppp.jl:121-129."""
    Y = np.asarray(Y)
    if Y.ndim == 2:
        if len(x) != Y.shape[0]:
            raise RuntimeError("Expected length(x) == size(Y, 1)")
        return [Y[a - 1:b, :] for a, b in get_indices(x)]
    if len(x) != len(Y):
        raise RuntimeError("Expected length(x) == length(y)")
    return [Y[a - 1:b] for a, b in get_indices(x)]


# --------------------------------------------------------------------------------------
# KernelFunctions.jl / Distances.jl  (un-vendored; SURVEY.md Appendix A)
# --------------------------------------------------------------------------------------


def pairwise_sqeuclidean(X, Y=None):
    """Distances.pairwise(SqEuclidean(), X, Y; dims=2): max(|x|^2 + |y|^2 - 2 x'y, 0) with the
    cross term from a BLAS GEMM; the one-argument form zeroes the diagonal exactly."""
    if Y is None:
        sa = np.einsum("dn,dn->n", X, X) if X.shape[0] > 1 else (X[0] * X[0])
        R = X.T @ X if X.shape[0] > 1 else np.multiply.outer(X[0], X[0])
        R = (sa[:, None] + sa[None, :]) - 2.0 * R
        np.maximum(R, 0.0, out=R)
        np.fill_diagonal(R, 0.0)
        return R
    if X.shape[0] > 1:
        sa = np.einsum("dn,dn->n", X, X)
        sb = np.einsum("dn,dn->n", Y, Y)
        R = X.T @ Y
    else:
        sa, sb = X[0] * X[0], Y[0] * Y[0]
        R = np.multiply.outer(X[0], Y[0])
    R = (sa[:, None] + sb[None, :]) - 2.0 * R
    np.maximum(R, 0.0, out=R)
    return R


def colwise_sqeuclidean(X, Y):
    """Distances.colwise(SqEuclidean(), X, Y): sum_d (x_d - y_d)^2 (direct, used by
    kernelmatrix_diag)."""
    d = X - Y
    return np.einsum("dn,dn->n", d, d)


class Kernel:
    def __add__(self, other):
        return KernelSum(self, other)

    def __rmul__(self, c):
        return ScaledKernel(self, float(c))

    def __mul__(self, c):
        if isinstance(c, Kernel):
            raise NotImplementedError("kernel products are outside the hot-path scope")
        return ScaledKernel(self, float(c))

    # -- interface ----------------------------------------------------------------------
    def matrix(self, x, y=None):
        raise NotImplementedError

    def diag(self, x, y=None):
        raise NotImplementedError


class _SimpleKernel(Kernel):
    """SimpleKernel: kappa(metric(x, y)).  metric is SqEuclidean (SE) or Euclidean (Matern)."""
    sq = True

    def kappa(self, d):
        raise NotImplementedError

    def matrix(self, x, y=None):
        X = _as_matrix(x)
        D2 = pairwise_sqeuclidean(X, None if y is None else _as_matrix(y))
        return self.kappa(D2 if self.sq else np.sqrt(D2))

    def diag(self, x, y=None):
        X = _as_matrix(x)
        if y is None:
            D2 = np.zeros(X.shape[1], dtype=X.dtype)
        else:
            D2 = colwise_sqeuclidean(X, _as_matrix(y))
        return self.kappa(D2 if self.sq else np.sqrt(D2))


class SEKernel(_SimpleKernel):
    def kappa(self, d2):
        return np.exp(-d2 / 2)


class Matern12Kernel(_SimpleKernel):
    sq = False

    def kappa(self, d):
        return np.exp(-d)


class Matern32Kernel(_SimpleKernel):
    sq = False

    def kappa(self, d):
        s = math.sqrt(3.0) * d
        return (1 + s) * np.exp(-s)


class Matern52Kernel(_SimpleKernel):
    sq = False

    def kappa(self, d):
        s = math.sqrt(5.0) * d
        return (1 + s + 5 * d * d / 3) * np.exp(-s)


class WhiteKernel(Kernel):
    """k(x,y) = (x == y) ? 1 : 0  -- exact equality of the input points."""

    def matrix(self, x, y=None):
        X = _as_matrix(x)
        Y = X if y is None else _as_matrix(y)
        eq = np.all(X[:, :, None] == Y[:, None, :], axis=0)
        return eq.astype(np.result_type(X.dtype, np.float32))

    def diag(self, x, y=None):
        X = _as_matrix(x)
        if y is None:
            return np.ones(X.shape[1], dtype=X.dtype)
        return np.all(X == _as_matrix(y), axis=0).astype(X.dtype)


class ConstantKernel(Kernel):
    def __init__(self, c=1.0):
        self.c = c

    def matrix(self, x, y=None):
        n = _length(x)
        m = n if y is None else _length(y)
        return np.full((n, m), self.c, dtype=_as_matrix(x).dtype)

    def diag(self, x, y=None):
        return np.full(_length(x), self.c, dtype=_as_matrix(x).dtype)


class ScaledKernel(Kernel):
    def __init__(self, k, s2):
        self.k, self.s2 = k, s2

    def matrix(self, x, y=None):
        return self.s2 * self.k.matrix(x, y)

    def diag(self, x, y=None):
        return self.s2 * self.k.diag(x, y)


class KernelSum(Kernel):
    def __init__(self, a, b):
        self.a, self.b = a, b

    def matrix(self, x, y=None):
        return self.a.matrix(x, y) + self.b.matrix(x, y)

    def diag(self, x, y=None):
        return self.a.diag(x, y) + self.b.diag(x, y)


class TransformedKernel(Kernel):
    """k o ScaleTransform(s): k(s*x, s*y)."""

    def __init__(self, k, s):
        self.k, self.s = k, s

    def _t(self, x):
        if x is None:
            return None
        return ColVecs(self.s * x.X) if isinstance(x, ColVecs) else self.s * np.asarray(x)

    def matrix(self, x, y=None):
        return self.k.matrix(self._t(x), self._t(y))

    def diag(self, x, y=None):
        return self.k.diag(self._t(x), self._t(y))


def with_lengthscale(k, ell):
    return TransformedKernel(k, 1.0 / ell)


def kernelmatrix(k, x, y=None):
    return k.matrix(x, y)


def kernelmatrix_diag(k, x, y=None):
    return k.diag(x, y)


# --------------------------------------------------------------------------------------
# AbstractGPs.GP  (mean function + kernel)
# --------------------------------------------------------------------------------------


class GP:
    """AbstractGPs.GP(mean, kernel): GP(k) zero mean; GP(c, k) constant; GP(fn, k) custom."""

    def __init__(self, *args):
        if len(args) == 1:
            self.mean_fn, self.kernel = 0.0, args[0]
        else:
            self.mean_fn, self.kernel = args

    def mean(self, x):
        n = _length(x)
        if callable(self.mean_fn):
            return np.array([self.mean_fn(v) for v in _iter_points(x)], dtype=float)
        return np.full(n, float(self.mean_fn), dtype=_as_matrix(x).dtype)

    def cov(self, x, y=None):
        return self.kernel.matrix(x, y)

    def var(self, x, y=None):
        return self.kernel.diag(x, y)


# --------------------------------------------------------------------------------------
# src/gp/util.jl, atomic_gp.jl, derived_gp.jl
# --------------------------------------------------------------------------------------


class GPC:  # src/gp/util.jl:18-25
    def __init__(self):
        self.n = 0


class SthenoGP:
    n: int
    gpc: GPC

    def __add__(self, other):
        return add(self, other)

    def __radd__(self, other):
        return add(other, self)

    def __sub__(self, other):  # addition.jl:12, :64-65
        if isinstance(other, SthenoGP):
            return add(self, neg(other))
        return add(self, -other)

    def __rsub__(self, other):
        return add(other, neg(self))

    def __mul__(self, other):
        return mul(other, self)

    def __rmul__(self, other):
        return mul(other, self)

    def __neg__(self):
        return neg(self)

    def __call__(self, x, noise=1e-18):
        return FiniteGP(self, x, noise)


class AtomicGP(SthenoGP):
    """src/gp/atomic_gp.jl:11-20."""

    def __init__(self, gp, gpc: GPC):
        self.gp = gp
        self.n = gpc.n + 1
        self.gpc = gpc
        gpc.n += 1


def atomic(gp, gpc):  # atomic_gp.jl:22
    return AtomicGP(gp, gpc)


class DerivedGP(SthenoGP):
    """src/gp/derived_gp.jl:7-17: args = (op, operands...)."""

    def __init__(self, args, gpc: GPC):
        self.args = args
        self.n = gpc.n + 1
        self.gpc = gpc
        gpc.n += 1


def add(a, b):
    """addition.jl:8-11 (GP+GP) and :62-65 (known + GP)."""
    if isinstance(a, SthenoGP) and isinstance(b, SthenoGP):
        assert a.gpc is b.gpc
        return DerivedGP(("+", a, b), a.gpc)
    if isinstance(b, SthenoGP):
        return DerivedGP(("+known", a, b), b.gpc)
    return DerivedGP(("+known", b, a), a.gpc)


def mul(f, g):
    """product.jl:11-13."""
    if isinstance(f, SthenoGP) and isinstance(g, SthenoGP):
        raise ValueError("Cannot multiply two GPs together.")  # ArgumentError
    if isinstance(g, SthenoGP):
        return DerivedGP(("*", f, g), g.gpc)
    return DerivedGP(("*", g, f), f.gpc)


def neg(f):  # product.jl:73
    return mul(-1, f)


def compose(f, g):  # compose.jl:8
    return DerivedGP(("o", f, g), f.gpc)


def cross(fs):  # cross.jl:37-45
    assert len(fs) >= 1
    assert all(f.gpc is fs[0].gpc for f in fs)
    return DerivedGP(("cross", list(fs)), fs[0].gpc)


# -- input maps (compose.jl:36-127) ------------------------------------------------------


def _map_input(g, x):
    """`g.(x)` with the reference's fast `broadcasted` methods."""
    if hasattr(g, "broadcast"):
        return g.broadcast(x)
    pts = [g(v) for v in _iter_points(x)]
    if len(pts) and np.ndim(pts[0]) == 1:
        return ColVecs(np.stack(pts, axis=1))
    return np.asarray(pts)


class Stretch:  # compose.jl:36-42
    def __init__(self, l):
        self.l = l

    def broadcast(self, x):
        if isinstance(x, ColVecs):
            return ColVecs(self.l * x.X if np.ndim(self.l) == 0 else np.asarray(self.l) @ x.X)
        return self.l * np.asarray(x)


def stretch(f, l):  # compose.jl:57-59
    if np.ndim(l) == 1:
        l = np.diag(np.asarray(l, dtype=float))
    return compose(f, Stretch(l))


class Select:  # compose.jl:72-77
    def __init__(self, idx):
        self.idx = idx

    def broadcast(self, x):
        assert isinstance(x, ColVecs)
        if isinstance(self.idx, (int, np.integer)):
            return x.X[self.idx, :]
        return ColVecs(x.X[np.asarray(self.idx), :])


def select(f, idx):  # compose.jl:84
    return compose(f, Select(idx))


class Periodic:  # compose.jl:93-99
    def __init__(self, f):
        self.f = f

    def broadcast(self, x):
        w = (2 * math.pi * self.f) * np.asarray(x)
        return ColVecs(np.vstack([np.cos(w), np.sin(w)]))


def periodic(g, f):  # compose.jl:106
    return compose(g, Periodic(f))


class Shift:  # compose.jl:114-119
    def __init__(self, a):
        self.a = a

    def broadcast(self, x):
        if isinstance(x, ColVecs):
            a = np.asarray(self.a)
            return ColVecs(x.X - (a.reshape(-1, 1) if a.ndim == 1 else a))
        return np.asarray(x) - self.a


def shift(f, a):  # compose.jl:127
    return compose(f, Shift(a))


def additive_gp(fs, indices=None):  # additive_gp.jl:10, :26-29
    if indices is None:
        indices = list(range(len(fs)))
    proj = [compose(f, Select(idx)) for f, idx in zip(fs, indices)]
    out = proj[0]
    for p in proj[1:]:
        out = out + p
    return out


# -- scale evaluation ------------------------------------------------------------------


def _scale(s, x):
    """`s.(x)` column vector, or the scalar itself (prod_args{<:Real})."""
    if callable(s):
        return np.array([s(v) for v in _iter_points(x)], dtype=float)
    return s


# -- unary statistics: mean / cov / var of a node --------------------------------------


def mean(f, x):
    if isinstance(f, GPPP):
        fs, vs = extract_components(f, x)
        return mean(fs, vs)
    if isinstance(f, AtomicGP):
        if isinstance(f.gp, GPPP):
            return mean(f.gp, x)
        return f.gp.mean(x)  # atomic_gp.jl:28
    op = f.args[0]
    if op == "+":  # addition.jl:26
        return mean(f.args[1], x) + mean(f.args[2], x)
    if op == "+known":  # addition.jl:73-74
        b = f.args[1]
        bx = np.array([b(v) for v in _iter_points(x)], dtype=float) if callable(b) else b
        return bx + mean(f.args[2], x)
    if op == "*":  # product.jl:25, :54
        return _scale(f.args[1], x) * mean(f.args[2], x)
    if op == "o":  # compose.jl:16
        return mean(f.args[1], _map_input(f.args[2], x))
    if op == "cross":  # cross.jl:54-57
        return np.concatenate([mean(g, blk) for g, blk in zip(f.args[1], x.blocks())])
    raise AssertionError(op)


def cov(f, x, y=None, g=None):
    """cov(f, x) / cov(f, x, x') / cov(f, f', x, x') (pass g=f')."""
    if isinstance(f, FiniteGP):
        return finite_cov(f, x)
    if g is not None:
        return _cov4(f, g, x, y)
    if isinstance(f, GPPP):
        if y is None:
            fs, vs = extract_components(f, x)  # gppp.jl:50-53
            return cov(fs, vs)
        fs, vs = extract_components(f, x)  # gppp.jl:60-64
        fs2, vs2 = extract_components(f, y)
        return _cov4(fs, fs2, vs, vs2)
    if isinstance(f, AtomicGP):  # atomic_gp.jl:30-33
        if isinstance(f.gp, GPPP):
            return cov(f.gp, x, y)
        return f.gp.cov(x, y)
    op = f.args[0]
    if op == "+":  # addition.jl:28-30, :35-37
        fa, fb = f.args[1], f.args[2]
        yy = x if y is None else y
        return cov(fa, x, y) + cov(fb, x, y) + _cov4(fa, fb, x, yy) + _cov4(fb, fa, x, yy)
    if op == "+known":  # addition.jl:76, :79
        return cov(f.args[2], x, y)
    if op == "*":  # product.jl:27-35, :56-59
        s, h = f.args[1], f.args[2]
        if callable(s):
            sx = _scale(s, x)
            sy = sx if y is None else _scale(s, y)
            return sx[:, None] * cov(h, x, y) * sy[None, :]
        return (s ** 2) * cov(h, x, y)
    if op == "o":  # compose.jl:18, :21
        h, m = f.args[1], f.args[2]
        return cov(h, _map_input(m, x), None if y is None else _map_input(m, y))
    if op == "cross":  # cross.jl:59-62, :69-72
        fs = f.args[1]
        yy = x if y is None else y
        rows = [_cov4(h, f, blk, yy) for h, blk in zip(fs, x.blocks())]
        return np.vstack(rows)
    raise AssertionError(op)


def var(f, x, y=None, g=None):
    if g is not None:
        return _var4(f, g, x, y)
    if isinstance(f, GPPP):
        if y is None:
            fs, vs = extract_components(f, x)
            return var(fs, vs)
        fs, vs = extract_components(f, x)
        fs2, vs2 = extract_components(f, y)
        return _var4(fs, fs2, vs, vs2)
    if isinstance(f, AtomicGP):  # atomic_gp.jl:31,34 ; gp/util.jl:5-7
        if isinstance(f.gp, GPPP):
            return var(f.gp, x, y)
        return f.gp.var(x, y)
    op = f.args[0]
    if op == "+":  # addition.jl:31-33, :38-40
        fa, fb = f.args[1], f.args[2]
        yy = x if y is None else y
        return var(fa, x, y) + var(fb, x, y) + _var4(fa, fb, x, yy) + _var4(fb, fa, x, yy)
    if op == "+known":
        return var(f.args[2], x, y)
    if op == "*":  # product.jl:32, :36-38, :57, :60
        s, h = f.args[1], f.args[2]
        if callable(s):
            sx = _scale(s, x)
            sy = sx if y is None else _scale(s, y)
            return sx * var(h, x, y) * sy
        return (s ** 2) * var(h, x, y)
    if op == "o":  # compose.jl:19, :22
        h, m = f.args[1], f.args[2]
        return var(h, _map_input(m, x), None if y is None else _map_input(m, y))
    if op == "cross":  # cross.jl:64-67, :74-77
        fs = f.args[1]
        if y is None:
            return np.concatenate([var(h, blk) for h, blk in zip(fs, x.blocks())])
        return np.concatenate([var(h, bx, by) for h, bx, by in zip(fs, x.blocks(), y.blocks())])
    raise AssertionError(op)


# -- binary (cross-process) statistics: the id-ordered recursion -----------------------


def _cov4(f, g, x, y):
    """src/gp/derived_gp.jl:31-44 + leaf rule src/gp/atomic_gp.jl:36-38."""
    assert f.gpc is g.gpc
    if isinstance(f, AtomicGP) and isinstance(g, AtomicGP):
        return cov(f, x, y) if f is g else np.zeros((_length(x), _length(y)))
    if f.n == g.n:
        return cov(f, x, y)
    if (isinstance(f, AtomicGP) and f.n > g.n) or (isinstance(g, AtomicGP) and g.n > f.n):
        return np.zeros((_length(x), _length(y)))
    if f.n >= g.n:
        return _cov_args_left(f.args, g, x, y)
    return _cov_args_right(f, g.args, x, y)


def _cov_args_left(args, g, x, y):
    op = args[0]
    if op == "+":  # addition.jl:42-44
        return _cov4(args[1], g, x, y) + _cov4(args[2], g, x, y)
    if op == "+known":  # addition.jl:82
        return _cov4(args[2], g, x, y)
    if op == "*":  # product.jl:40, :62
        s = _scale(args[1], x)
        c = _cov4(args[2], g, x, y)
        return (s[:, None] if np.ndim(s) else s) * c
    if op == "o":  # compose.jl:24
        return _cov4(args[1], g, _map_input(args[2], x), y)
    if op == "cross":  # cross.jl:79-82
        return np.vstack([_cov4(h, g, blk, y) for h, blk in zip(args[1], x.blocks())])
    raise AssertionError(op)


def _cov_args_right(f, args, x, y):
    op = args[0]
    if op == "+":  # addition.jl:45-47
        return _cov4(f, args[1], x, y) + _cov4(f, args[2], x, y)
    if op == "+known":  # addition.jl:83
        return _cov4(f, args[2], x, y)
    if op == "*":  # product.jl:41, :63
        s = _scale(args[1], y)
        c = _cov4(f, args[2], x, y)
        return c * (s[None, :] if np.ndim(s) else s)
    if op == "o":  # compose.jl:25
        return _cov4(f, args[1], x, _map_input(args[2], y))
    if op == "cross":  # cross.jl:83-86
        return np.hstack([_cov4(f, h, x, blk) for h, blk in zip(args[1], y.blocks())])
    raise AssertionError(op)


def _var4(f, g, x, y):
    """src/gp/derived_gp.jl:46-59 + atomic_gp.jl:39-41."""
    assert f.gpc is g.gpc
    if isinstance(f, AtomicGP) and isinstance(g, AtomicGP):
        return var(f, x, y) if f is g else np.zeros(_length(x))
    if f.n == g.n:
        return var(f, x, y)
    if (isinstance(f, AtomicGP) and f.n > g.n) or (isinstance(g, AtomicGP) and g.n > f.n):
        return np.zeros(_length(x))
    if f.n >= g.n:
        args = f.args
        op = args[0]
        if op == "+":
            return _var4(args[1], g, x, y) + _var4(args[2], g, x, y)
        if op == "+known":
            return _var4(args[2], g, x, y)
        if op == "*":
            return _scale(args[1], x) * _var4(args[2], g, x, y)
        if op == "o":
            return _var4(args[1], g, _map_input(args[2], x), y)
        if op == "cross":  # cross.jl:88-90
            return np.diag(_cov_args_left(args, g, x, y)).copy()
        raise AssertionError(op)
    args = g.args
    op = args[0]
    if op == "+":
        return _var4(f, args[1], x, y) + _var4(f, args[2], x, y)
    if op == "+known":
        return _var4(f, args[2], x, y)
    if op == "*":
        return _var4(f, args[2], x, y) * _scale(args[1], y)
    if op == "o":
        return _var4(f, args[1], x, _map_input(args[2], y))
    if op == "cross":  # cross.jl:91-93
        return np.diag(_cov_args_right(f, args, x, y)).copy()
    raise AssertionError(op)


# --------------------------------------------------------------------------------------
# src/gaussian_process_probabilistic_programme.jl
# --------------------------------------------------------------------------------------


class GPPP:
    """gppp.jl:13-18.  `fs` is an ordered mapping name -> process."""

    def __init__(self, fs: dict, gpc: GPC):
        self.fs = dict(fs)
        self.gpc = gpc

    def __call__(self, x, noise=1e-18):
        return FiniteGP(self, x, noise)


def gppp(build: Callable):
    """Stand-in for the `@gppp let ... end` macro (gppp.jl:166-201): `build(GPf)` receives a
    `GP`-like constructor that wraps every GP(...) in `atomic(..., gpc)` and returns the dict
    of named processes."""
    gpc = GPC()
    fs = build(lambda *a: atomic(GP(*a), gpc))
    return GPPP(fs, gpc)


def extract_components(f: GPPP, x):
    """gppp.jl:25, :27-30, :32-43."""
    if isinstance(x, GPPPInput):
        return f.fs[x.p], x.x
    if isinstance(x, BlockData):
        pairs = [extract_components(f, b) for b in x.X]
        return cross([p[0] for p in pairs]), BlockData([p[1] for p in pairs])
    # AbstractVector{<:Tuple}: regroup by unique symbol in first-occurrence order.
    x = list(x)
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
        elif len(sel) and isinstance(sel[0], tuple):
            blocks.append(GPPPInput(s, sel))
        else:
            blocks.append(GPPPInput(s, np.asarray(sel)))
    return extract_components(f, BlockData(blocks))


# --------------------------------------------------------------------------------------
# AbstractGPs.jl (un-vendored; SURVEY.md Appendix A): FiniteGP, logpdf, rand, posterior, VFE
# --------------------------------------------------------------------------------------


def _noise_matrix(noise, n):
    noise = np.asarray(noise, dtype=float) if not np.isscalar(noise) else noise
    if np.isscalar(noise):
        return "scalar", float(noise)
    if noise.ndim == 1:
        return "diag", noise
    return "dense", noise


class FiniteGP:
    def __init__(self, f, x, noise=1e-18):
        self.f, self.x = f, x
        self.kind, self.noise = _noise_matrix(noise, _length(x))

    def __len__(self):
        return _length(self.x)

    def noise_diag(self):
        n = len(self)
        if self.kind == "scalar":
            return np.full(n, self.noise)
        if self.kind == "diag":
            return self.noise
        return np.diag(self.noise)

    def add_noise(self, K):
        if self.kind == "dense":
            return K + self.noise
        K = K.copy()
        K[np.diag_indices_from(K)] += self.noise_diag()
        return K


def finite_mean(fx: FiniteGP):
    return mean(fx.f, fx.x)


def finite_cov(fx: FiniteGP, gx: FiniteGP | None = None):
    if gx is None:
        return fx.add_noise(cov(fx.f, fx.x))  # cov(fx) = cov(f,x) + Sigma_y
    if isinstance(fx.f, GPPP) or isinstance(gx.f, GPPP):
        assert fx.f is gx.f
        return cov(fx.f, fx.x, gx.x)
    return _cov4(fx.f, gx.f, fx.x, gx.x)  # src/gp/util.jl:12-14


def finite_var(fx: FiniteGP):
    return var(fx.f, fx.x) + fx.noise_diag()


def marginals(fx: FiniteGP):
    """Normal.(mean, sqrt.(var)) -> (mean, std)."""
    return finite_mean(fx), np.sqrt(finite_var(fx))


def _chol_upper(C):
    """cholesky(Symmetric(C)).U via LAPACK dpotrf (upper triangle of C is used, like Julia)."""
    U = sla.cholesky(np.asfortranarray(C), lower=False, overwrite_a=False, check_finite=False)
    return U


def rand(fx: FiniteGP, z):
    """rand(rng, fx, S) = m .+ chol(Symmetric(C)).U' * randn(rng, N, S) with the normals `z`
    supplied by the caller (shape (N,) or (N, S))."""
    m = finite_mean(fx)
    U = _chol_upper(finite_cov(fx))
    z = np.asarray(z)
    out = U.T @ z
    return out + (m if z.ndim == 1 else m[:, None])


def logpdf(fx, Y):
    """logpdf(fx, Y) = -(N log 2pi + logdet(C) .+ colsumsq(C.U' \\ (Y .- m))) ./ 2."""
    if isinstance(fx, SparseFiniteGP):  # sparse_finite_gp.jl:52-58
        Y = np.asarray(Y)
        if Y.ndim == 2:
            return np.array([elbo(VFE(fx.finducing), fx.fobs, Y[:, j]) for j in range(Y.shape[1])])
        return elbo(VFE(fx.finducing), fx.fobs, Y)
    Y = np.asarray(Y, dtype=float)
    m = finite_mean(fx)
    U = _chol_upper(finite_cov(fx))
    n = len(fx)
    logdet = 2.0 * np.sum(np.log(np.diag(U)))
    delta = Y - (m if Y.ndim == 1 else m[:, None])
    V = sla.solve_triangular(U, delta, trans="T", lower=False, check_finite=False)
    q = np.sum(V * V, axis=0)
    return -(n * math.log(2 * math.pi) + logdet + q) / 2


class PosteriorGP:
    """AbstractGPs.PosteriorGP: data = (alpha, C, x, delta)."""

    def __init__(self, prior, alpha, U, x, delta):
        self.prior, self.alpha, self.U, self.x, self.delta = prior, alpha, U, x, delta

    def __call__(self, x, noise=1e-18):
        return FiniteGP(self, x, noise)


def posterior(fx, y):
    if isinstance(fx, SparseFiniteGP):  # sparse_finite_gp.jl:60-62
        return vfe_posterior(VFE(fx.finducing), fx.fobs, y)
    if isinstance(fx, VFE):
        raise TypeError("use vfe_posterior(VFE(fz), fx, y)")
    m = finite_mean(fx)
    U = _chol_upper(finite_cov(fx))
    delta = np.asarray(y, dtype=float) - m
    alpha = sla.cho_solve((U, False), delta, check_finite=False)
    return PosteriorGP(fx.f, alpha, U, fx.x, delta)


def _prior_cov(prior, x, y=None):
    if isinstance(prior, (GPPP, SthenoGP)):
        return cov(prior, x, y)
    raise TypeError(type(prior))


def _post_mean(fp: PosteriorGP, x):
    return mean(fp.prior, x) + cov(fp.prior, x, fp.x) @ fp.alpha


def _post_cov(fp: PosteriorGP, x, z=None):
    Kfx = cov(fp.prior, fp.x, x)
    Vx = sla.solve_triangular(fp.U, Kfx, trans="T", lower=False, check_finite=False)
    if z is None:
        return cov(fp.prior, x) - Vx.T @ Vx
    Kfz = cov(fp.prior, fp.x, z)
    Vz = sla.solve_triangular(fp.U, Kfz, trans="T", lower=False, check_finite=False)
    return cov(fp.prior, x, z) - Vx.T @ Vz


def _post_var(fp: PosteriorGP, x):
    Kfx = cov(fp.prior, fp.x, x)
    Vx = sla.solve_triangular(fp.U, Kfx, trans="T", lower=False, check_finite=False)
    return var(fp.prior, x) - np.sum(Vx * Vx, axis=0)


# route PosteriorGP / ApproxPosteriorGP through the generic mean/cov/var entry points
_mean0, _cov0, _var0 = mean, cov, var


def mean(f, x):  # noqa: F811
    if isinstance(f, FiniteGP):
        return finite_mean(f)
    if isinstance(f, PosteriorGP):
        return _post_mean(f, x)
    if isinstance(f, ApproxPosteriorGP):
        return f.mean(x)
    return _mean0(f, x)


def cov(f, x=None, y=None, g=None):  # noqa: F811
    if isinstance(f, FiniteGP):
        return finite_cov(f, x)
    if isinstance(f, SparseFiniteGP):  # sparse_finite_gp.jl:39-43
        raise RuntimeError(COVARIANCE_ERROR)
    if isinstance(f, PosteriorGP):
        return _post_cov(f, x, y)
    if isinstance(f, ApproxPosteriorGP):
        return f.cov(x, y)
    return _cov0(f, x, y, g)


def var(f, x=None, y=None, g=None):  # noqa: F811
    if isinstance(f, FiniteGP):
        return finite_var(f)
    if isinstance(f, PosteriorGP):
        return _post_var(f, x)
    if isinstance(f, ApproxPosteriorGP):
        return f.var(x)
    return _var0(f, x, y, g)


def mean_and_var(f, x):
    return mean(f, x), var(f, x)


def mean_and_cov(f, x):
    return mean(f, x), cov(f, x)


# -- VFE / elbo (Titsias) ---------------------------------------------------------------


class VFE:
    def __init__(self, fz: FiniteGP):
        self.fz = fz


def _vfe_intermediates(v: VFE, fx: FiniteGP, y):
    """AbstractGPs._compute_intermediates (SURVEY App. A): diagonal / isotropic noise."""
    assert fx.kind in ("scalar", "diag")
    fz = v.fz
    sy = np.sqrt(fx.noise_diag())  # U_y (diagonal)
    U = _chol_upper(finite_cov(fz))
    Kxz = cov(fx.f, fx.x, fz.x)  # N x M
    B = (Kxz / sy[:, None]).T  # (U_y' \ Kxz)'  M x N
    A = sla.solve_triangular(U, B, trans="T", lower=False, check_finite=False)
    M = A.shape[0]
    Lam = _chol_upper(A @ A.T + np.eye(M))
    delta = (np.asarray(y, dtype=float) - finite_mean(fx)) / sy
    return dict(U=U, A=A, Lam=Lam, delta=delta, sy=sy)


def dtc(v: VFE, fx: FiniteGP, y):
    t = _vfe_intermediates(v, fx, y)
    return _dtc_from(t, len(fx))


def _dtc_from(t, n):
    Ad = t["A"] @ t["delta"]
    w = sla.solve_triangular(t["Lam"], Ad, trans="T", lower=False, check_finite=False)
    logdet_sy = 2.0 * np.sum(np.log(t["sy"]))
    logdet_lam = 2.0 * np.sum(np.log(np.diag(t["Lam"])))
    return -(n * math.log(2 * math.pi) + logdet_sy + logdet_lam
             + t["delta"] @ t["delta"] - w @ w) / 2


def elbo(v, fx=None, y=None):
    if isinstance(v, SparseFiniteGP):  # sparse_finite_gp.jl:52
        return elbo(VFE(v.finducing), v.fobs, fx)
    t = _vfe_intermediates(v, fx, y)
    tr = np.sum(var(fx.f, fx.x) / fx.noise_diag())
    return _dtc_from(t, len(fx)) - (tr - np.sum(t["A"] * t["A"])) / 2


class ApproxPosteriorGP:
    """AbstractGPs approximate posterior under VFE (SURVEY App. A)."""

    def __init__(self, prior, z, U, Lam, alpha):
        self.prior, self.z, self.U, self.Lam, self.alpha = prior, z, U, Lam, alpha

    def __call__(self, x, noise=1e-18):
        return FiniteGP(self, x, noise)

    def mean(self, x):
        return mean(self.prior, x) + cov(self.prior, x, self.z) @ self.alpha

    def _BD(self, x):
        Kzx = cov(self.prior, self.z, x)
        B = sla.solve_triangular(self.U, Kzx, trans="T", lower=False, check_finite=False)
        D = sla.solve_triangular(self.Lam, B, trans="T", lower=False, check_finite=False)
        return B, D

    def cov(self, x, y=None):
        B, D = self._BD(x)
        if y is None:
            return cov(self.prior, x) - B.T @ B + D.T @ D
        B2, D2 = self._BD(y)
        return cov(self.prior, x, y) - B.T @ B2 + D.T @ D2

    def var(self, x):
        B, D = self._BD(x)
        return var(self.prior, x) - np.sum(B * B, axis=0) + np.sum(D * D, axis=0)


def vfe_posterior(v: VFE, fx: FiniteGP, y):
    t = _vfe_intermediates(v, fx, y)
    Ad = t["A"] @ t["delta"]
    m_eps = sla.cho_solve((t["Lam"], False), Ad, check_finite=False)
    alpha = sla.solve_triangular(t["U"], m_eps, lower=False, check_finite=False)
    return ApproxPosteriorGP(fx.f, v.fz.x, t["U"], t["Lam"], alpha)


# -- src/gp/sparse_finite_gp.jl ---------------------------------------------------------

COVARIANCE_ERROR = (
    "The covariance matrix of a sparse GP can often be dense and can cause the computer to "
    "run out of memory. If you are sure you have enough memory, you can use `cov(f.fobs)`."
)


class SparseFiniteGP:  # sparse_finite_gp.jl:30-33
    def __init__(self, fobs: FiniteGP, finducing: FiniteGP):
        self.fobs, self.finducing = fobs, finducing

    def __len__(self):  # :35
        return len(self.fobs)
