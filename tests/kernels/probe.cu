// Test-only C entry points onto the kernel launchers of libstheno_b200 (tests/test_gpu_kernels.py).
//
// Every wrapper takes device pointers and plain integers, builds the launcher's argument structs,
// calls the one launcher on the legacy default stream, synchronises and returns the CUDA status
// (or, for the int-returning Ozaki launchers, their non-zero launch status, negated and offset by
// 1000).  The launchers are called with whatever rank / world / range / SM reservation the test
// passes, so the multi-GPU partitions of the trailing update and the assembly run on one device.
#include <cstring>

#include "../../stheno.jl_b200/csrc/sb_common.cuh"

using namespace sb;

namespace {

int finish() {
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return (int)e;
    return (int)cudaStreamSynchronize(0);
}

int finish_oz(int rc) {
    if (rc != 0) return -1000 - rc;
    return finish();
}

Packed packed(double* base, int64_t Np) { return Packed{base, Np}; }

template <typename T>
void ptrs(const int64_t* in, int n, T** out) {
    for (int i = 0; i < n; i++) out[i] = reinterpret_cast<T*>(in[i]);
}

}  // namespace

extern "C" {

int pb_gemm_nt(int64_t A, int64_t lda, int64_t B, int64_t ldb, int64_t Cp, int64_t ldc, int64_t M, int64_t Ncols,
               int64_t K, double alpha, double beta) {
    launch_gemm_nt((const double*)A, lda, (const double*)B, ldb, (double*)Cp, ldc, M, Ncols, K, alpha, beta, 0);
    return finish();
}

int pb_gemm_nt_seg(int nseg, const int64_t* A, const int64_t* lda, const int64_t* B, const int64_t* ldb, int64_t Cp,
                   int64_t ldc, int64_t M, int64_t Ncols, double alpha, double beta) {
    const double* a[4];
    const double* b[4];
    ptrs(A, nseg, a);
    ptrs(B, nseg, b);
    launch_gemm_nt_seg(nseg, a, lda, b, ldb, (double*)Cp, ldc, M, Ncols, alpha, beta, 0);
    return finish();
}

int pb_trsm_tiled(int64_t A, int64_t lda, int64_t invL, int64_t Pt, int64_t m) {
    launch_trsm_tiled((const double*)A, lda, (const double*)invL, (double*)Pt, m, 0);
    return finish();
}

int pb_untile_panel(int64_t Pt, int64_t row_blk0, int64_t nrow_blks, int64_t dst, int64_t ld) {
    launch_untile_panel((const double*)Pt, row_blk0, nrow_blks, (double*)dst, ld, 0);
    return finish();
}

int64_t pb_syrk_packed_tiles(int64_t nblk, int64_t k, int64_t jlo, int64_t jhi, int rank, int world) {
    return syrk_packed_tiles(nblk, k, jlo, jhi, rank, world);
}

int pb_syrk_packed(int64_t base, int64_t Np, int64_t k, const int64_t* Pt, int nseg, int64_t jlo, int64_t jhi,
                   int rank, int world, int reserve_sms) {
    const double* p[4];
    ptrs(Pt, nseg, p);
    launch_syrk_packed(packed((double*)base, Np), k, p, nseg, jlo, jhi, rank, world, 0, reserve_sms);
    return finish();
}

int64_t pb_oz_planes_bytes(int64_t Np) { return (int64_t)oz_planes_bytes(Np); }
int64_t pb_oz_maps_bytes() { return (int64_t)sizeof(OzMaps); }

// maps: host buffer of pb_oz_maps_bytes() bytes, 64-byte aligned
int pb_oz_make_maps(int64_t planes, int64_t Np, void* maps) {
    const int rc = oz_make_maps((signed char*)planes, Np, reinterpret_cast<OzMaps*>(maps));
    return rc != 0 ? -1000 - rc : 0;
}

int pb_oz_slice(int nseg, const int64_t* base, const int64_t* ld, const int64_t* rbs, const int64_t* diag,
                const int64_t* dld, int colsign, int64_t rb_lo, int64_t nrb, int64_t out_row_base, int64_t plane_rows,
                int64_t scale, int64_t expo, int64_t planes) {
    OzSrc s{};
    s.nseg = nseg;
    s.colsign = colsign;
    for (int q = 0; q < nseg; q++) {
        s.base[q] = (const double*)base[q];
        s.ld[q] = ld[q];
        s.rbs[q] = rbs[q];
        s.diag[q] = (const double*)diag[q];
        s.dld[q] = dld[q];
    }
    launch_oz_slice(s, rb_lo, nrb, out_row_base, plane_rows, (double*)scale, (int*)expo, (signed char*)planes, 0);
    return finish();
}

int pb_syrk_ozaki(int64_t base, int64_t Np, int64_t k, int nseg, int64_t jlo, int64_t jhi, int rank, int world,
                  const void* maps, int64_t scale, int reserve_sms, int64_t tile_lo, int64_t tile_hi) {
    return finish_oz(launch_syrk_ozaki(packed((double*)base, Np), k, nseg, jlo, jhi, rank, world,
                                       reinterpret_cast<const OzMaps*>(maps), (const double*)scale, 0, reserve_sms,
                                       tile_lo, tile_hi));
}

int pb_gemm_ozaki(int64_t Cp, int64_t ldc, int64_t M, int64_t Ncols, int nseg, const void* mapsA, int64_t scaleA,
                  int64_t rowA0, const void* mapsB, int64_t scaleB, int64_t rowB0) {
    return finish_oz(launch_gemm_ozaki((double*)Cp, ldc, M, Ncols, nseg, reinterpret_cast<const OzMaps*>(mapsA),
                                       (const double*)scaleA, rowA0, reinterpret_cast<const OzMaps*>(mapsB),
                                       (const double*)scaleB, rowB0, 0));
}

int pb_panel_solve_ozaki(const int64_t* Xcol, const int64_t* ldx, int64_t M, const void* mapsA, int64_t scaleA,
                         int64_t rowA0, const void* mapsW, int64_t scaleW) {
    double* x[4];
    ptrs(Xcol, 4, x);
    return finish_oz(launch_panel_solve_ozaki(x, ldx, M, reinterpret_cast<const OzMaps*>(mapsA), (const double*)scaleA,
                                              rowA0, reinterpret_cast<const OzMaps*>(mapsW), (const double*)scaleW, 0));
}

// one block of at most MAX_TERMS terms; zl/zr/sl/sr: device pointers (0 = none for sl/sr)
int pb_assemble_packed(int64_t base, int64_t Np, int64_t N, int64_t row0, int64_t nrows, int64_t col0, int64_t ncols,
                       int nterms, int accumulate, const int* kernel, const int* dim, const double* coeff,
                       const double* param, const int64_t* zl, const int64_t* zr, const int64_t* sl,
                       const int64_t* sr, double sigma2, int64_t noise_diag, int rank, int world) {
    if (nterms < 0 || nterms > MAX_TERMS) return -1;
    BlockDev b;
    std::memset(&b, 0, sizeof(b));
    b.row0 = row0; b.nrows = nrows; b.col0 = col0; b.ncols = ncols;
    b.nterms = nterms; b.accumulate = accumulate;
    for (int t = 0; t < nterms; t++) {
        b.t[t] = TermDev{kernel[t], dim[t], coeff[t], param[t], (const double*)zl[t], (const double*)zr[t],
                         (const double*)sl[t], (const double*)sr[t]};
        b.tix[t] = t;
    }
    launch_assemble_packed(b, packed((double*)base, Np), N, sigma2, (const double*)noise_diag, 0, rank, world);
    return finish();
}

int pb_sweep(int64_t base, int64_t Np, int64_t invL, int64_t b, int S, int backward, int64_t flags, int num_sms) {
    launch_sweep(packed((double*)base, Np), (const double*)invL, (double*)b, S, backward != 0, (unsigned*)flags,
                 num_sms, 0);
    return finish();
}

}  // extern "C"
