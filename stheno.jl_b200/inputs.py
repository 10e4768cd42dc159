"""Input containers of the hot path: GPPPInput, BlockData, ColVecs, split.

Host-side mirror of Stheno.jl src/input_collection_types.jl:24-95 and
src/gaussian_process_probabilistic_programme.jl:121-135.  Integer/index semantics are
bit-exact requirements (tests/test_inputs.py ports test/input_collection_types.jl:4-49).
Indices are 0-based here (Python); `eachindex` / `block_ranges` return the reference's 1-based
ranges so they can be compared verbatim.
"""
from __future__ import annotations

import numpy as np


class ColVecs:
    """KernelFunctions.ColVecs: a (D, N) matrix viewed as N points of dimension D."""

    __slots__ = ("X",)

    def __init__(self, X):
        X = np.asarray(X)
        if X.ndim != 2:
            raise ValueError("ColVecs expects a (D, N) matrix")
        self.X = X

    def __len__(self):
        return self.X.shape[1]

    def __getitem__(self, idx):
        if isinstance(idx, (int, np.integer)):
            return self.X[:, idx]
        return ColVecs(self.X[:, idx])

    def __iter__(self):
        for i in range(self.X.shape[1]):
            yield self.X[:, i]

    def __eq__(self, other):
        return isinstance(other, ColVecs) and np.array_equal(self.X, other.X)

    __hash__ = None


def npoints(x) -> int:
    return len(x)


def iter_points(x):
    if isinstance(x, (ColVecs, GPPPInput, BlockData)):
        yield from x
    else:
        yield from np.asarray(x)


def points_equal(a, b) -> bool:
    if isinstance(a, (ColVecs, GPPPInput, BlockData)) or isinstance(b, (ColVecs, GPPPInput, BlockData)):
        return type(a) is type(b) and a == b
    return np.array_equal(np.asarray(a), np.asarray(b))


class GPPPInput:
    """`GPPPInput(p, x)`: the vector `x` belongs to process `p`
    (src/input_collection_types.jl:24-33).  Behaves as a vector of `(p, x_i)` tuples."""

    __slots__ = ("p", "x")

    def __init__(self, p, x):
        self.p = p
        # torch CUDA tensors (inputs already resident in HBM) are passed through untouched
        self.x = x if isinstance(x, (ColVecs, GPPPInput, BlockData)) or hasattr(x, "data_ptr") else np.asarray(x)

    def __len__(self):
        return npoints(self.x)

    def __getitem__(self, idx):
        if isinstance(idx, (int, np.integer)):
            return (self.p, self.x[idx])
        return [(self.p, v) for v in iter_points(self.x[idx])]

    def __iter__(self):
        for v in iter_points(self.x):
            yield (self.p, v)

    def __eq__(self, other):
        if isinstance(other, GPPPInput):
            return self.p == other.p and points_equal(self.x, other.x)
        if isinstance(other, (list, tuple)):
            return len(other) == len(self) and all(
                a[0] == b[0] and np.array_equal(a[1], b[1]) for a, b in zip(self, other))
        return NotImplemented

    __hash__ = None

    def __repr__(self):
        return f"GPPPInput({self.p!r}, n={len(self)})"


class BlockData:
    """Ordered ragged collection of input vectors behaving as one flat vector
    (src/input_collection_types.jl:61-95)."""

    __slots__ = ("X",)

    def __init__(self, *xs):
        if len(xs) == 1 and isinstance(xs[0], (list, tuple)):
            xs = tuple(xs[0])
        self.X = [x if isinstance(x, (ColVecs, GPPPInput, BlockData)) else np.asarray(x) for x in xs]

    # size / length  (:69)
    def __len__(self):
        return sum(npoints(b) for b in self.X)

    def block_lengths(self):
        return [npoints(b) for b in self.X]

    def locate(self, n: int):
        """Linear 0-based index -> (block, offset): the walk of :71-78."""
        n = int(n)
        if n < 0:
            n += len(self)
        b = 0
        while n >= npoints(self.X[b]):
            n -= npoints(self.X[b])
            b += 1
        return b, n

    def __getitem__(self, n):
        b, off = self.locate(n)
        return self.X[b][off]

    def __iter__(self):
        for b in self.X:
            yield from iter_points(b)

    def __eq__(self, other):  # :80
        if isinstance(other, BlockData):
            return len(self.X) == len(other.X) and all(points_equal(a, b) for a, b in zip(self.X, other.X))
        if isinstance(other, (list, tuple)):
            return len(other) == len(self) and all(_elt_equal(a, b) for a, b in zip(self, other))
        return NotImplemented

    __hash__ = None

    def blocks(self):  # :82
        return self.X

    def view(self, b: int, n):  # :84
        return self.X[b][n]

    def eachindex(self):
        """1-based index ranges per block: `BlockArray(1:sum(lengths), lengths)` (:88-91)."""
        out, start = [], 1
        for L in self.block_lengths():
            out.append(np.arange(start, start + L, dtype=np.int64))
            start += L
        return out

    def block_ranges(self):
        """`_get_indices` (gppp.jl:131-134): 1-based inclusive (first, last) per block."""
        lengths = self.block_lengths()
        sz = np.cumsum(lengths, dtype=np.int64)
        return [(int(sz[n] - lengths[n] + 1), int(sz[n])) for n in range(len(lengths))]

    def eltype(self):
        """Element type rule of :86 / test/input_collection_types.jl:33-36."""
        kinds = set()
        for b in self.X:
            if isinstance(b, ColVecs):
                kinds.add(("vec", b.X.dtype))
            elif isinstance(b, GPPPInput):
                kinds.add(("tuple", type(b.p)))
            elif isinstance(b, BlockData):
                kinds.add(("any", None))
            else:
                kinds.add(("scalar", b.dtype))
        return kinds.pop() if len(kinds) == 1 else ("any", None)

    def __repr__(self):
        return f"BlockData({self.block_lengths()})"


def _elt_equal(a, b):
    if isinstance(a, tuple) and isinstance(b, tuple):
        return a[0] == b[0] and _elt_equal(a[1], b[1])
    return np.array_equal(a, b)


def blocks(x: BlockData):
    return x.X


def vcat(*xs):
    """`vcat(::GPPPInput...)` -> BlockData (:93-95)."""
    return BlockData(list(xs))


def split(x: BlockData, Y):
    """`Base.split(x::BlockData, Y)`: rows of Y grouped by the blocks of x (gppp.jl:121-129).
    Raises RuntimeError (Julia ErrorException) on a length mismatch, with the reference text."""
    Y = np.asarray(Y)
    if Y.ndim == 2:
        if len(x) != Y.shape[0]:
            raise RuntimeError("Expected length(x) == size(Y, 1)")
        return [Y[a - 1:b, :] for a, b in x.block_ranges()]
    if len(x) != Y.shape[0]:
        raise RuntimeError("Expected length(x) == length(y)")
    return [Y[a - 1:b] for a, b in x.block_ranges()]
