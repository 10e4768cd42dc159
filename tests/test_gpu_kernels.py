"""The hot-path kernels on their own, against exact references, through the test-only probe library
(tests/kernels/probe.cu -> build/libsb_probe.so), which calls the launchers directly.

Calling the launchers directly reaches what the C ABI never does on one GPU: the `rank` / `world`
partitions of the trailing updates and of the assembly (each rank of a simulated world is run in turn
on one device), the look-ahead driver's T^A / T^B ranges and SM reservations, the split of an int8
Ozaki trailing update into tile ranges, ownership wrap-around in the triangular sweep, and the
segment addressing and alpha / beta epilogue of the NT product.

Exact references.  Operands are integers: the fp64 DMMA product of entries |a|, |b| <= 2^10 over
K <= 512 has every partial sum below 2^53, so the kernel's result equals the integer product bit for
bit.  The int8 Ozaki product is exact as well when every row of an operand holds integers and its
maximum is below 2^20: every entry then lies in the top digit planes, no dropped digit pair is
non-zero, and the recombination is exact (checked on the CPU by test_ozaki_slicing_premise, a
restatement of the slicer and of the kernel's recombination order).

Layouts restated here: the packed lower block-column layout of sb_common.cuh (`Packed::off/ld/at`)
and the tiled panel layout of gemm_nt.cu, addr(rb, k, r) = (rb 128 + k) 132 + r.
"""
import ctypes as C
import os

import numpy as np
import pytest

import exact_refs as er

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NB = 128
TP = NB + 4          # padded column of the tiled panel layout
OUTER_BLOCKS = 4
LOOKAHEAD_SMS = 8
RESERVES = (0, 8, 64, 131)   # 131 leaves one SM: a grid of 2 CTAs, the TMA ring wraps over many tiles
WORLDS = (1, 2, 3, 4, 8)
K_SE, K_WHITE = 0, 4
gpu = pytest.mark.gpu


# ---- packed lower block-column layout (sb_common.cuh, struct Packed) ------------------------------------

def p_ld(Np, j):
    return Np - j * NB


def p_off(Np, j):
    return NB * (j * Np - NB * (j * (j - 1) // 2))


def p_total(Np):
    return p_off(Np, Np // NB)


def p_col(v, Np, j):
    """View of block column j: element [r - j NB, c - j NB] is (r, c), column-major with ld_j."""
    o = p_off(Np, j)
    return v[o:o + NB * p_ld(Np, j)].reshape(NB, p_ld(Np, j)).T


def p_blockcols(Np):
    """Block column index of every element of the packed storage."""
    out = np.empty(p_total(Np), dtype=np.int64)
    for j in range(Np // NB):
        out[p_off(Np, j):p_off(Np, j + 1)] = j
    return out


def p_rows_cols(Np):
    """Row and column index of every element of the packed storage."""
    r = np.empty(p_total(Np), dtype=np.int64)
    c = np.empty(p_total(Np), dtype=np.int64)
    for j in range(Np // NB):
        ld = p_ld(Np, j)
        o = p_off(Np, j)
        r[o:o + NB * ld] = np.tile(j * NB + np.arange(ld), NB)
        c[o:o + NB * ld] = np.repeat(j * NB + np.arange(NB), ld)
    return r, c


def pack(A):
    Np = A.shape[0]
    v = np.empty(p_total(Np))
    for j in range(Np // NB):
        p_col(v, Np, j)[:] = A[j * NB:, j * NB:(j + 1) * NB]
    return v


# ---- tiled panel layout (gemm_nt.cu, TilePtrs) -----------------------------------------------------------

def tile(P):
    """(nrb 128) x 128 panel -> tiled buffer; the 4 pad doubles of every column hold NaN."""
    nrb = P.shape[0] // NB
    t = np.full((nrb, NB, TP), np.nan)
    t[:, :, :NB] = P.reshape(nrb, NB, NB).transpose(0, 2, 1)
    return t.ravel()


def untile(buf, nrb):
    return buf.reshape(nrb, NB, TP)[:, :, :NB].transpose(0, 2, 1).reshape(nrb * NB, NB)


# ---- device plumbing -------------------------------------------------------------------------------------

def ints(rng, lo, hi, shape):
    return rng.integers(lo, hi + 1, size=shape).astype(np.float64)


class Probe:
    def __init__(self):
        import torch
        from stheno_jl_b200 import lib
        lib.load()
        path = os.path.join(ROOT, "build", "libsb_probe.so")
        assert os.path.exists(path), f"{path} missing: run stheno.jl_b200/csrc/build.sh"
        self.torch = torch
        self.dev = torch.device("cuda:0")
        self.lib = C.CDLL(path)
        i32, i64, f64, vp = C.c_int, C.c_int64, C.c_double, C.c_void_p
        P64 = C.POINTER(i64)
        sigs = {
            "pb_gemm_nt": [i64, i64, i64, i64, i64, i64, i64, i64, i64, f64, f64],
            "pb_gemm_nt_seg": [i32, P64, P64, P64, P64, i64, i64, i64, i64, f64, f64],
            "pb_trsm_tiled": [i64, i64, i64, i64, i64],
            "pb_untile_panel": [i64, i64, i64, i64, i64],
            "pb_syrk_packed_tiles": [i64, i64, i64, i64, i32, i32],
            "pb_syrk_packed": [i64, i64, i64, P64, i32, i64, i64, i32, i32, i32],
            "pb_oz_planes_bytes": [i64],
            "pb_oz_maps_bytes": [],
            "pb_oz_make_maps": [i64, i64, vp],
            "pb_oz_slice": [i32, P64, P64, P64, P64, P64, i32, i64, i64, i64, i64, i64, i64, i64],
            "pb_syrk_ozaki": [i64, i64, i64, i32, i64, i64, i32, i32, vp, i64, i32, i64, i64],
            "pb_gemm_ozaki": [i64, i64, i64, i64, i32, vp, i64, i64, vp, i64, i64],
            "pb_panel_solve_ozaki": [P64, P64, i64, vp, i64, i64, vp, i64],
            "pb_assemble_packed": [i64, i64, i64, i64, i64, i64, i64, i32, i32, C.POINTER(i32), C.POINTER(i32),
                                   C.POINTER(f64), C.POINTER(f64), P64, P64, P64, P64, f64, i64, i32, i32],
            "pb_sweep": [i64, i64, i64, i64, i32, i32, i64, i32],
        }
        for name, args in sigs.items():
            fn = getattr(self.lib, name)
            fn.argtypes = args
            fn.restype = i64 if name in ("pb_syrk_packed_tiles", "pb_oz_planes_bytes", "pb_oz_maps_bytes") else i32
        self.num_sms = torch.cuda.get_device_properties(0).multi_processor_count

    def __call__(self, name, *args):
        self.torch.cuda.synchronize()
        rc = getattr(self.lib, name)(*args)
        assert rc == 0, f"{name} returned {rc}"

    def up(self, a):
        return self.torch.from_numpy(np.ascontiguousarray(a)).to(self.dev)

    def down(self, t):
        self.torch.cuda.synchronize()
        return t.cpu().numpy()

    def maps(self, planes, rows):
        """Tensor maps over a digit-plane buffer: a 64-byte aligned host blob."""
        n = self.lib.pb_oz_maps_bytes()
        buf = C.create_string_buffer(n + 64)
        addr = (C.addressof(buf) + 63) & ~63
        self("pb_oz_make_maps", planes.data_ptr(), rows, C.c_void_p(addr))
        return buf, C.c_void_p(addr)   # keep buf alive with the address

    def planes(self, rows):
        t = self.torch
        return (t.zeros(self.lib.pb_oz_planes_bytes(rows), dtype=t.int8, device=self.dev),
                t.zeros(rows, dtype=t.float64, device=self.dev), t.zeros(rows, dtype=t.int32, device=self.dev))

    def slice(self, segs, lds, rb_lo, nrb, out_row_base, plane_rows, planes, diag=None, dlds=None, colsign=0):
        """launch_oz_slice over column-major segments (device tensors) with row-block stride 128."""
        n = len(segs)
        pl, scale, expo = planes
        diag = diag or [0] * n
        self("pb_oz_slice", n, a64([s.data_ptr() for s in segs]), a64(lds), a64([NB] * n),
             a64([d if isinstance(d, int) else d.data_ptr() for d in diag]), a64(dlds or [0] * n), colsign,
             rb_lo, nrb, out_row_base, plane_rows, scale.data_ptr(), expo.data_ptr(), pl.data_ptr())


def a64(vals):
    return (C.c_int64 * max(1, len(vals)))(*[int(v) for v in vals])


@pytest.fixture(scope="module")
def pb():
    return Probe()


def assert_same(got, exp, what):
    """Equal values, NaN where NaN expected (canaries), and no NaN anywhere else."""
    bad = ~((got == exp) | (np.isnan(got) & np.isnan(exp)))
    assert not bad.any(), f"{what}: {int(bad.sum())} elements differ, first at {np.flatnonzero(bad)[:8]}"


# ---- the int8 Ozaki premise, on the CPU ------------------------------------------------------------------

OZ_S = 7


def oz_slice_rows(X):
    """Restatement of oz_rowscale_kernel + oz_slice_kernel for a dense block of rows: digit planes
    d[p, i, k] (int64 values of the int8 digits) and row exponents e_i (scale 2^(e_i - 31))."""
    m = np.max(np.abs(X), axis=1)
    e = np.frexp(m)[1] - 1 + 2                                   # ilogb(m) + 2
    Z = np.rint(np.ldexp(X, (55 - e)[:, None])).astype(np.int64) + 0x0000808080808080
    d = np.empty((OZ_S,) + X.shape, dtype=np.int64)
    d[0] = ((Z >> 48) & 0xff).astype(np.uint8).astype(np.int8)
    for p in range(1, OZ_S):
        d[p] = (((Z >> (8 * (OZ_S - 1 - p))) & 0xff) ^ 0x80).astype(np.uint8).astype(np.int8)
    return d, e


def oz_product(da, ea, db, eb):
    """sum_k a_ik b_jk as ozaki_syrk_kernel forms it: G_t in exact integers, then in fp64 in the kernel's
    group order (pass 0: groups 0..3 from planes 0..3, pass 1: groups 4..6), times s_i s_j."""
    acc = np.zeros((da.shape[1], db.shape[1]))
    for grp in range(OZ_S):
        G = sum(da[p] @ db[grp - p].T for p in range(grp + 1))
        assert np.max(np.abs(G)) < 2 ** 31
        acc = acc + G.astype(np.float64) * float(2 ** (8 * (OZ_S - 1 - grp)))
    return np.ldexp(np.ldexp(acc, (ea - 31)[:, None]), (eb - 31)[None, :])


def test_ozaki_slicing_premise():
    """Integer rows with maximum below 2^20 have digits in planes 0..3 only (no dropped pair p + q > 6 is
    non-zero) and the slicer's recombination reproduces the integer product exactly, at K = 512."""
    rng = np.random.default_rng(7)
    for amp in (1, 3, 1024, 2 ** 20 - 1):
        A = ints(rng, -amp, amp, (64, 512))
        B = ints(rng, -amp, amp, (48, 512))
        A[0, 5], B[0, 9] = amp, -amp                   # row maxima at the bound
        A[1], B[1] = 0.0, 0.0                          # zero rows: scale 0 on the device, no digits here
        A[1, 3], B[1, 3] = 1.0, 1.0
        da, ea = oz_slice_rows(A)
        db, eb = oz_slice_rows(B)
        assert not da[4:].any() and not db[4:].any()
        exact = A.astype(np.int64) @ B.astype(np.int64).T
        got = oz_product(da, ea, db, eb)
        assert np.array_equal(got, exact.astype(np.float64)), amp


# ---- K3: launch_gemm_nt / launch_gemm_nt_seg ------------------------------------------------------------

def _gemm_case(pb, rng, M, ncols, lda, ldb, ks):
    """Column-major segments with NaN in the rows a read with a wrong leading dimension would reach."""
    A, B, Ad, Bd = [], [], [], []
    for q, K in enumerate(ks):
        a = np.full((K, lda[q]), np.nan)
        a[:, :M] = ints(rng, -1024, 1024, (K, M))
        b = np.full((K, ldb[q]), np.nan)
        b[:, :ncols] = ints(rng, -1024, 1024, (K, ncols))
        A.append(a[:, :M].T)
        B.append(b[:, :ncols].T)
        Ad.append(pb.up(a))
        Bd.append(pb.up(b))
    return np.hstack(A), np.hstack(B), Ad, Bd


def _check_gemm(pb, launch, M, ncols, A, B, rng):
    """C window at rows [2, 2 + M), columns [1, 1 + ncols) of an ldc = M + 6 buffer; everything else
    of the buffer is a guard and must not change.  beta = 0 runs over a NaN-filled C."""
    ldc = M + 6
    prod = A @ B.T                                      # exact: integers below 2^53
    for alpha in (1.0, -1.0, 0.5):
        for beta in (0.0, 1.0):
            buf = np.full((ncols + 2, ldc), np.nan) if beta == 0.0 else ints(rng, -2 ** 20, 2 ** 20, (ncols + 2, ldc))
            Cd = pb.up(buf)
            launch(Cd.data_ptr() + 8 * (ldc + 2), ldc, alpha, beta)
            exp = buf.copy()
            win = exp[1:1 + ncols, 2:2 + M]
            win[:] = (alpha * prod + beta * win.T).T if beta else (alpha * prod).T
            assert_same(pb.down(Cd), exp, f"alpha={alpha} beta={beta}")


@gpu
@pytest.mark.parametrize("ncols", [64, 192])
@pytest.mark.parametrize("M", [128, 384])
@pytest.mark.parametrize("nseg", [1, 2, 3, 4])
def test_gemm_nt_seg(pb, nseg, M, ncols):
    """K-segmented NT product: every segment in its own allocation with its own lda / ldb."""
    rng = np.random.default_rng(100 * nseg + M + ncols)
    lda = [M + 2 + 6 * q for q in range(nseg)]
    ldb = [ncols + 4 + 2 * q for q in range(nseg)]
    A, B, Ad, Bd = _gemm_case(pb, rng, M, ncols, lda, ldb, [NB] * nseg)

    def launch(c, ldc, alpha, beta):
        pb("pb_gemm_nt_seg", nseg, a64([t.data_ptr() for t in Ad]), a64(lda), a64([t.data_ptr() for t in Bd]),
           a64(ldb), c, ldc, M, ncols, alpha, beta)
    _check_gemm(pb, launch, M, ncols, A, B, rng)


@gpu
@pytest.mark.parametrize("K", [16, 144, 512])
def test_gemm_nt_plain(pb, K):
    """One operand pair, K any multiple of 16."""
    rng = np.random.default_rng(K)
    M, ncols = 384, 192
    A, B, Ad, Bd = _gemm_case(pb, rng, M, ncols, [M + 10], [ncols + 2], [K])

    def launch(c, ldc, alpha, beta):
        pb("pb_gemm_nt", Ad[0].data_ptr(), M + 10, Bd[0].data_ptr(), ncols + 2, c, ldc, M, ncols, K, alpha, beta)
    _check_gemm(pb, launch, M, ncols, A, B, rng)


@gpu
@pytest.mark.parametrize("kq,q", [(0, 0), (2, 1), (3, 3)])
def test_trsm_tiled_and_untile(pb, kq, q):
    """Panel TRSM (A invL^T into the tiled buffer at row block q) then untile into block column kq of the
    packed matrix: exactly A invL^T there, nothing else of the matrix or of the tiled pads changes."""
    nblk = 6
    Np = nblk * NB
    rng = np.random.default_rng(10 * kq + q)
    v0 = ints(rng, -1024, 1024, p_total(Np))
    invL = np.tril(ints(rng, -4, 4, (NB, NB)), -1) + np.eye(NB)
    m = Np - (kq + 1) * NB
    A = p_col(v0, Np, kq)[NB:].copy()
    vd = pb.up(v0)
    Pbuf = pb.up(np.full(nblk * NB * TP, np.nan))
    invLd = pb.up(invL.T)                                  # column-major
    blk = vd.data_ptr() + 8 * (p_off(Np, kq) + NB)         # Packed::blk(kq + 1, kq)
    pb("pb_trsm_tiled", blk, p_ld(Np, kq), invLd.data_ptr(), Pbuf.data_ptr() + 8 * q * NB * TP, m)
    X = A @ invL.T
    tiled = pb.down(Pbuf)
    exp_t = np.full(nblk * NB * TP, np.nan)
    exp_t[q * NB * TP:q * NB * TP + m * TP] = tile(X)
    assert_same(tiled, exp_t, "tiled panel")
    pb("pb_untile_panel", Pbuf.data_ptr(), q, m // NB, blk, p_ld(Np, kq))
    exp = v0.copy()
    p_col(exp, Np, kq)[NB:] = X
    assert_same(pb.down(vd), exp, "packed matrix")


# ---- K3 / K3': packed trailing updates and their partitions ----------------------------------------------

class SyrkCase:
    """Panels P_q (rows of block rows k+1 .. nblk-1), an integer packed matrix A0 and the exact
    A0 - sum_q P_q P_q^T on every block column J > k."""

    def __init__(self, pb, nblk, k, nseg, seed):
        rng = np.random.default_rng(seed)
        self.Np, self.nblk, self.k, self.nseg = nblk * NB, nblk, k, nseg
        Np = self.Np
        nrb = nblk - k - 1
        self.P = [ints(rng, -1024, 1024, (nrb * NB, NB)) for _ in range(nseg)]
        self.v0 = ints(rng, -2 ** 20, 2 ** 20, p_total(Np))
        Pc = np.hstack(self.P)
        D = Pc @ Pc.T                                      # exact: integers below 2^53
        self.ref = self.v0.copy()
        for J in range(k + 1, nblk):
            s = (J - k - 1) * NB
            p_col(self.ref, Np, J)[:] -= D[s:, s:s + NB]
        self.bc = pb.up(p_blockcols(Np))
        self.v0d, self.refd = pb.up(self.v0), pb.up(self.ref)

    def ranges(self):
        """(jlo, jhi) as the drivers issue them, plus an empty range and one the launcher clamps."""
        jt = self.k + self.nseg
        jA = min(jt + OUTER_BLOCKS, self.nblk)
        return [(jt, self.nblk), (jt, jA), (jA, self.nblk), (jt, jt), (0, self.nblk)]

    def mask(self, jlo, jhi, rank=None, world=1):
        m = (self.bc >= max(jlo, self.k + 1)) & (self.bc < jhi)
        if rank is not None:
            m &= (self.bc % world) == rank
        return m

    def check(self, pb, got, m, what):
        exp = pb.torch.where(m, self.refd, self.v0d)
        if not pb.torch.equal(got, exp):
            g, e = pb.down(got), pb.down(exp)
            assert_same(g, e, what)


def _partition_sweep(pb, case, run):
    """run(A, jlo, jhi, rank, world, reserve) on every rank of every world over every range: the union of
    the ranks equals the exact update of the range; each rank alone changes exactly its own columns."""
    for wi, world in enumerate(WORLDS):
        for ri, (jlo, jhi) in enumerate(case.ranges()):
            reserve = RESERVES[(wi + ri) % len(RESERVES)]
            A = case.v0d.clone()
            for rank in range(world):
                run(A, jlo, jhi, rank, world, reserve)
            case.check(pb, A, case.mask(jlo, jhi), f"union world={world} [{jlo},{jhi}) reserve={reserve}")
            if world == 1:
                continue
            for rank in range(world):
                A = case.v0d.clone()
                run(A, jlo, jhi, rank, world, reserve)
                case.check(pb, A, case.mask(jlo, jhi, rank, world),
                           f"rank {rank}/{world} [{jlo},{jhi}) reserve={reserve}")


SYRK_SHAPES = [(nblk, k) for nblk in (9, 13, 24) for k in (0, 3, nblk - 2)]


@gpu
@pytest.mark.parametrize("nseg", [1, 2, 3, 4])
@pytest.mark.parametrize("nblk,k", SYRK_SHAPES)
def test_syrk_packed_partitions(pb, nblk, k, nseg):
    case = SyrkCase(pb, nblk, k, nseg, seed=1000 * nblk + 10 * k + nseg)
    Pt = [pb.up(tile(P)) for P in case.P]
    ptrs = a64([t.data_ptr() for t in Pt])

    def run(A, jlo, jhi, rank, world, reserve):
        pb("pb_syrk_packed", A.data_ptr(), case.Np, k, ptrs, nseg, jlo, jhi, rank, world, reserve)
    _partition_sweep(pb, case, run)
    # every reservation on the serial range, one rank of three
    for reserve in RESERVES:
        A = case.v0d.clone()
        run(A, k + nseg, nblk, 1, 3, reserve)
        case.check(pb, A, case.mask(k + nseg, nblk, 1, 3), f"reserve={reserve}")


def _oz_syrk_setup(pb, case):
    """Digit planes of the panel as cholesky_wide prepares them for the trailing update: launch_oz_slice over
    the block columns' rows below the step, plane row = matrix row, no column equilibration."""
    Np, k = case.Np, case.k
    segs = []
    for P in case.P:
        full = np.zeros((NB, Np))                          # column-major Np x 128
        full[:, (k + 1) * NB:] = P.T
        segs.append(pb.up(full))
    planes = pb.planes(Np)
    pb.slice(segs, [Np] * case.nseg, k + 1, case.nblk - k - 1, 0, Np, planes)
    return segs, planes, pb.maps(planes[0], Np)


@gpu
@pytest.mark.parametrize("nseg", [1, 2, 3, 4])
@pytest.mark.parametrize("nblk,k", SYRK_SHAPES)
def test_syrk_ozaki_partitions(pb, nblk, k, nseg):
    case = SyrkCase(pb, nblk, k, nseg, seed=2000 * nblk + 10 * k + nseg)
    segs, planes, (keep, maps) = _oz_syrk_setup(pb, case)
    scale = planes[1].data_ptr()

    def run(A, jlo, jhi, rank, world, reserve, lo=0, hi=0):
        pb("pb_syrk_ozaki", A.data_ptr(), case.Np, k, nseg, jlo, jhi, rank, world, maps, scale, reserve, lo, hi)
    _partition_sweep(pb, case, run)
    # T^B split into tile ranges [0, cut) (with the look-ahead reservation) and [cut, total), as cholesky_wide
    # issues them: cut at 0, at an odd count (a block's two half-tiles apart), in the middle and at the total
    jA = min(k + nseg + OUTER_BLOCKS, nblk)
    for world in (1, 3):
        for rank in range(world):
            total = 2 * pb.lib.pb_syrk_packed_tiles(nblk, k, jA, nblk, rank, world)
            whole = case.v0d.clone()
            run(whole, jA, nblk, rank, world, 0)
            case.check(pb, whole, case.mask(jA, nblk, rank, world), f"T^B rank {rank}/{world}")
            for cut in sorted({0, min(total, 2 * (total // 4) + 1), total // 2, total}):
                A = case.v0d.clone()
                if cut > 0:
                    run(A, jA, nblk, rank, world, LOOKAHEAD_SMS, 0, cut)
                if cut < total:
                    run(A, jA, nblk, rank, world, 0, cut, total)
                assert pb.torch.equal(A, whole), f"T^B cut at {cut} of {total}, rank {rank}/{world}"


def _oz_src(pb, rng, rows, nseg, lds, amp, mult=1):
    """nseg column-major segments of `rows` x 128 integers (multiples of `mult`, |x| <= amp), own ld each."""
    host, dev = [], []
    for q in range(nseg):
        a = np.zeros((NB, lds[q]))
        a[:, :rows] = mult * ints(rng, -(amp // mult), amp // mult, (NB, rows))
        host.append(a[:, :rows].T)
        dev.append(pb.up(a))
    return np.hstack(host), dev


@gpu
@pytest.mark.parametrize("nseg", [1, 2, 3, 4])
def test_gemm_ozaki_row_offsets(pb, nseg):
    """C[M x Ncols] -= A B^T from plane rows rowA0.. / rowB0.. of two plane sets; the rows of the sets
    outside the operands hold other data, and C's guard rows / columns do not change."""
    rng = np.random.default_rng(300 + nseg)
    M, ncols, rowA0, rowB0 = 256, 192, 256, 192
    ra, rbr = rowA0 + M + NB, 512                          # plane rows of the two sets
    Afull, Ad = _oz_src(pb, rng, ra, nseg, [ra + 2 * q for q in range(nseg)], 1024)
    Bfull, Bd = _oz_src(pb, rng, rbr, nseg, [rbr + 6 + 2 * q for q in range(nseg)], 1024)
    pa, pbs = pb.planes(ra), pb.planes(rbr)
    pb.slice(Ad, [ra + 2 * q for q in range(nseg)], 0, ra // NB, 0, ra, pa)
    pb.slice(Bd, [rbr + 6 + 2 * q for q in range(nseg)], 0, rbr // NB, 0, rbr, pbs)
    (ka, ma), (kb, mb) = pb.maps(pa[0], ra), pb.maps(pbs[0], rbr)
    ldc = M + 10
    buf = ints(rng, -2 ** 20, 2 ** 20, (ncols + 2, ldc))
    Cd = pb.up(buf)
    pb("pb_gemm_ozaki", Cd.data_ptr() + 8 * (ldc + 4), ldc, M, ncols, nseg, ma, pa[1].data_ptr(), rowA0, mb,
       pbs[1].data_ptr(), rowB0)
    exp = buf.copy()
    exp[1:1 + ncols, 4:4 + M] -= (Afull[rowA0:rowA0 + M] @ Bfull[rowB0:rowB0 + ncols].T).T
    assert_same(pb.down(Cd), exp, "C")


@gpu
@pytest.mark.parametrize("colsign", [0, 1])
def test_panel_solve_ozaki(pb, colsign):
    """X = A W^T (W 512 x 512 block lower triangular) into four column buffers with distinct ldx.  W's
    blocks above the diagonal hold non-zero garbage the kernel must skip.  With colsign = 1 the columns of
    A are sliced times 2^-e and those of W times 2^+e (e = ilogb of a diagonal, as the wide panel phase
    does): the result must be bit-identical to the plain slicing, and exact."""
    rng = np.random.default_rng(400 + colsign)
    M, rowA0 = 384, 256
    ra = rowA0 + M + NB
    lds = [ra + 4 * q for q in range(4)]
    Afull, Ad = _oz_src(pb, rng, ra, 4, lds, 1024, mult=8)
    W = ints(rng, -64, 64, (512, 512))
    Wt = W.copy()
    for q in range(4):
        Wt[q * NB:(q + 1) * NB, (q + 1) * NB:] = 0.0       # what the product uses
    Wd = [pb.up(np.ascontiguousarray(W[:, q * NB:(q + 1) * NB].T)) for q in range(4)]   # segment q: K cols q
    diag, dld = [], []
    for q in range(4):
        ld = NB + 2 * q + 2
        d = np.zeros((NB, ld))
        d[np.arange(NB), np.arange(NB)] = 2.0 ** rng.integers(0, 4, NB) * (1 + rng.random(NB))
        diag.append(pb.up(d))
        dld.append(ld)
    pa, pw = pb.planes(ra), pb.planes(512)
    sign = (-colsign, colsign)
    pb.slice(Ad, lds, 0, ra // NB, 0, ra, pa, diag if colsign else None, dld if colsign else None, sign[0])
    pb.slice(Wd, [512] * 4, 0, 4, 0, 512, pw, diag if colsign else None, dld if colsign else None, sign[1])
    (ka, ma), (kw, mw) = pb.maps(pa[0], ra), pb.maps(pw[0], 512)
    ldx = [M + 2, M + 8, M + 4, M + 14]
    bufs = [pb.up(np.full((NB + 1, ldx[q]), np.nan)) for q in range(4)]
    xcol = a64([bufs[q].data_ptr() + 8 * (ldx[q] + 2) for q in range(4)])
    pb("pb_panel_solve_ozaki", xcol, a64(ldx), M, ma, pa[1].data_ptr(), rowA0, mw, pw[1].data_ptr())
    X = Afull[rowA0:rowA0 + M] @ Wt.T
    for q in range(4):
        exp = np.full((NB + 1, ldx[q]), np.nan)
        exp[1:, 2:2 + M] = X[:, q * NB:(q + 1) * NB].T
        assert_same(pb.down(bufs[q]), exp, f"column buffer {q}")


# ---- K1: packed assembly with rank / world ---------------------------------------------------------------

class Term:
    def __init__(self, kernel, coeff, zl, zr, sl=None, sr=None, dim=1, param=0.0):
        self.kernel, self.coeff, self.zl, self.zr, self.sl, self.sr = kernel, coeff, zl, zr, sl, sr
        self.dim, self.param = dim, param

    def value(self):
        """The term on its block, restated (Distances.jl GEMM-trick squared distance)."""
        x, y = self.zl.reshape(-1, self.dim), self.zr.reshape(-1, self.dim)
        if self.kernel == K_WHITE:
            k = np.all(x[:, None, :] == y[None, :, :], axis=2).astype(np.float64)
        else:
            d2 = np.maximum((x * x).sum(1)[:, None] + (y * y).sum(1)[None, :] - 2.0 * (x @ y.T), 0.0)
            k = np.exp(-0.5 * d2)
        s = self.coeff * (self.sl[:, None] if self.sl is not None else 1.0) * \
            (self.sr[None, :] if self.sr is not None else 1.0)
        return s * k


def _assemble(pb, vd, Np, N, blk, terms, accumulate, sigma2, noise, rank, world, keep):
    row0, nrows, col0, ncols = blk
    n = len(terms)
    dev = lambda a: 0 if a is None else keep.setdefault(id(a), pb.up(a)).data_ptr()
    pb("pb_assemble_packed", vd.data_ptr(), Np, N, row0, nrows, col0, ncols, n, accumulate,
       (C.c_int * n)(*[t.kernel for t in terms]), (C.c_int * n)(*[t.dim for t in terms]),
       (C.c_double * n)(*[t.coeff for t in terms]), (C.c_double * n)(*[t.param for t in terms]),
       a64([dev(t.zl) for t in terms]), a64([dev(t.zr) for t in terms]), a64([dev(t.sl) for t in terms]),
       a64([dev(t.sr) for t in terms]), sigma2, dev(noise), rank, world)


def _assembly_cases(rng):
    N = 700
    x = np.round(rng.uniform(0, 30, N), 3)
    x[::7] = x[3]                                          # repeated inputs: White is 1 off the diagonal too
    x2 = rng.uniform(0, 5, 2 * N)
    s = rng.uniform(0.5, 2.0, N)
    noise = rng.uniform(0.01, 0.1, N)
    se = lambda c, a, b, **kw: Term(K_SE, c, a, b, **kw)
    return N, [
        ("SE + White, sigma2", (0, N, 0, N), [se(1.3, x / 2.1, x / 2.1), Term(K_WHITE, 0.2, x, x)], 0.05, None),
        ("SE, diagonal noise", (0, N, 0, N), [se(0.7, x, x, sl=s, sr=s)], 0.0, noise),
        ("2-D SE, unaligned origin", (200, 300, 72, 260), [se(1.1, x2[:600], x2[:520], dim=2)], 0.0, None),
        ("8 terms", (0, N, 0, N), [se(0.1 * (i + 1), x / (i + 1), x / (i + 1)) for i in range(7)]
         + [Term(K_WHITE, 0.3, x, x)], 0.02, None),
    ]


@gpu
@pytest.mark.parametrize("case", range(4))
def test_assemble_packed_partitions(pb, case):
    """The union over ranks is bit-identical to world = 1 (and matches the restated kernel values); each
    rank alone writes exactly the elements of its own block columns (NaN canaries everywhere else)."""
    rng = np.random.default_rng(500)
    N, cases = _assembly_cases(rng)
    name, blk, terms, sigma2, noise = cases[case]
    Np = 6 * NB
    row0, nrows, col0, ncols = blk
    r, c = p_rows_cols(Np)
    inblk = (r >= row0) & (r < row0 + nrows) & (c >= col0) & (c < col0 + ncols)
    base = pb.up(ints(rng, -8, 8, p_total(Np)))
    canary = np.full(p_total(Np), np.nan)
    keep = {}

    def run(vd, rank, world):
        chunks = [terms[i:i + 6] for i in range(0, len(terms), 6)]     # > MAX_TERMS terms: accumulate
        for i, ch in enumerate(chunks):
            _assemble(pb, vd, Np, N, blk, ch, int(i > 0), sigma2, noise, rank, world, keep)

    one = base.clone()
    run(one, 0, 1)
    one_h = pb.down(one)
    # values: sum of the terms, plus the noise on the diagonal
    K = sum(t.value() for t in terms)
    exp = pb.down(base).copy()
    exp[inblk] = K[r[inblk] - row0, c[inblk] - col0]
    diag = inblk & (r == c)
    exp[diag] += noise[c[diag]] if noise is not None else sigma2
    np.testing.assert_allclose(one_h, exp, rtol=1e-14, atol=0, err_msg=name)
    assert np.array_equal(one_h[~inblk], pb.down(base)[~inblk]), name
    bc = c // NB
    for world in WORLDS[1:]:
        union = base.clone()
        for rank in range(world):
            run(union, rank, world)
            alone = pb.up(canary)
            run(alone, rank, world)
            got = pb.down(alone)
            own = inblk & (bc % world == rank)
            assert np.isnan(got[~own]).all(), f"{name}: rank {rank}/{world} wrote outside its block columns"
            if len(terms) <= 6:
                assert np.array_equal(got[own], one_h[own]), f"{name}: rank {rank}/{world}"
        assert pb.torch.equal(union, one), f"{name}: union over {world} ranks"


# ---- triangular sweep ------------------------------------------------------------------------------------

@gpu
@pytest.mark.parametrize("backward", [False, True])
@pytest.mark.parametrize("S", [1, 8, 9])
@pytest.mark.parametrize("nblk", [3, 4, 9, 17])
def test_sweep_worker_counts(pb, nblk, S, backward):
    """b <- L^-1 b (L^-T b) on the exact factor for every grid size: each block's updates are applied in k
    order by one CTA whatever the number of workers W, so results are bit-identical across num_sms (W
    from 1 to nblk, blocks owned round-robin), and within 1e-12 of the exact integer solution."""
    n = nblk * NB
    L = er.exact_factor(n, seed=3000 + n)
    X = er.int_matrix(n, S, seed=3100 + n, amp=16)
    b = (L.T if backward else L) @ X                       # exact (exact_refs.py)
    invL = np.concatenate([np.linalg.inv(L[j * NB:(j + 1) * NB, j * NB:(j + 1) * NB]).T.ravel()
                           for j in range(nblk)])          # column-major diagonal-block inverses
    Ld, invLd = pb.up(pack(L)), pb.up(invL)
    flags = pb.torch.zeros(2 * nblk, dtype=pb.torch.int32, device=pb.dev)
    first = None
    for sms in sorted({1, 2, 3, 7, min(132, pb.num_sms)}):
        bd = pb.up(b.T)                                    # column-major n x S, ld n
        for s0 in range(0, S, 8):                          # at most 8 right-hand sides per launch
            pb("pb_sweep", Ld.data_ptr(), n, invLd.data_ptr(), bd.data_ptr() + 8 * s0 * n, min(8, S - s0),
               int(backward), flags.data_ptr(), sms)
        got = pb.down(bd).T
        err = np.max(np.abs(got - X))
        assert err <= 1e-12 * np.max(np.abs(X)), (sms, err)
        if first is None:
            first = got
        else:
            assert np.array_equal(got, first), f"num_sms={sms} differs from num_sms=1"
