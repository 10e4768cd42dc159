// Shared definitions for libstheno_b200 (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <string>

#include "../../include/stheno_b200.h"

namespace sb {

constexpr int NB = 128;  // block size of the packed-lower layout == Cholesky panel width

// ---- error plumbing ---------------------------------------------------------------------
void set_error(const std::string& msg);
int32_t cuda_fail(cudaError_t e, const char* what, const char* file, int line);

#define SB_CUDA(call)                                                              \
    do {                                                                           \
        cudaError_t _e = (call);                                                   \
        if (_e != cudaSuccess) return ::sb::cuda_fail(_e, #call, __FILE__, __LINE__); \
    } while (0)

#define SB_CHECK(cond, msg)                    \
    do {                                       \
        if (!(cond)) {                         \
            ::sb::set_error(msg);              \
            return SB_ERR_INVALID;             \
        }                                      \
    } while (0)

#define SB_TRY(expr)                    \
    do {                                \
        int32_t _s = (expr);            \
        if (_s != SB_OK) return _s;     \
    } while (0)

// ---- packed lower block-column layout ---------------------------------------------------
// The symmetric matrix / its Cholesky factor is stored as nblk block columns; block column j
// (NB columns wide) keeps only rows >= j*NB, column-major with leading dimension
// ld_j = Np - j*NB, and the block columns are concatenated.  Every sub-diagonal panel
// L[(j+1)*NB:, j*NB:(j+1)*NB] is therefore one contiguous, TMA/NCCL-friendly slab and the whole
// factor takes Np(Np+NB)/2 elements (17.2 GB at N=65536 fp64 instead of 34.4 GB).
struct Packed {
    double* base;
    int64_t Np;  // padded order, multiple of NB
    __host__ __device__ int64_t nblk() const { return Np / NB; }
    __host__ __device__ int64_t ld(int64_t j) const { return Np - j * NB; }
    __host__ __device__ int64_t off(int64_t j) const {
        return (int64_t)NB * (j * Np - (int64_t)NB * (j * (j - 1) / 2));
    }
    // pointer to element (r, c), r >= (c/NB)*NB
    __host__ __device__ double* at(int64_t r, int64_t c) const {
        int64_t j = c / NB;
        return base + off(j) + (c - j * NB) * ld(j) + (r - j * NB);
    }
    // pointer to the top-left element of block (I, J), I >= J
    __host__ __device__ double* blk(int64_t I, int64_t J) const {
        return base + off(J) + (I - J) * NB;
    }
    __host__ __device__ int64_t total() const { return off(nblk()); }
};

inline int64_t round_up(int64_t x, int64_t m) { return (x + m - 1) / m * m; }

// ---- device-side term/block descriptors for the assembly kernels -------------------------
constexpr int MAX_TERMS = 6;
constexpr int MAX_DIM = 8;

struct TermDev {
    int32_t kernel;
    int32_t dim;
    double coeff;
    double param;
    const double* zl;  // device, [nrows * dim] point-major, indexed by local row
    const double* zr;  // device, [ncols * dim]
    const double* sl;  // device or nullptr
    const double* sr;
};

struct BlockDev {
    int64_t row0, nrows, col0, ncols;
    int32_t nterms;
    int32_t accumulate;  // 1: add to existing output (blocks with > MAX_TERMS terms)
    TermDev t[MAX_TERMS];
    int32_t tix[MAX_TERMS];  // index of each term in the caller's sb_covspec (gradient output slot)
};

// output target of the assembly kernel
struct OutDense {
    double* p;
    int64_t ld;
};

// ---- kernel launchers (defined in the .cu files) ------------------------------------------
void launch_assemble_dense(const BlockDev& b, OutDense out, cudaStream_t s);
// world > 1: only tiles in block columns J with J % world == rank are generated
void launch_assemble_packed(const BlockDev& b, Packed out, int64_t N, double sigma2,
                            const double* noise_diag, cudaStream_t s, int rank = 0, int world = 1);
void launch_fill_padding(Packed out, int64_t N, cudaStream_t s);
void launch_assemble_diag(const BlockDev& b, double* out, cudaStream_t s);
// gradient reduction (sb_logpdf_grad): for every term t of block b
//   g[2*tix]   += w * sum_ij Q_ij sl_i sr_j kappa_t(i,j)              (d/d coeff_t)
//   g[2*tix+1] += w * sum_ij Q_ij coeff sl_i sr_j dkappa_t/dlog(s)    (d/d log input-scale)
// with Q_ij = (alpha_i alpha_j - Kinv_ij)/2, Kinv dense column-major (ld); w = 2 for strictly
// off-diagonal blocks of a symmetric spec.
void launch_grad_reduce(const BlockDev& b, const double* alpha, const double* Kinv, int64_t ld, double w,
                        double* g, cudaStream_t s);
// the same reduction with Q_ij = a u_i v_j + bw G_ij  (sb_vfe_grad; G dense column-major, ld)
void launch_grad_reduce_outer(const BlockDev& b, double a, const double* u, const double* v, double bw,
                              const double* G, int64_t ld, double w, double* g, cudaStream_t s);
// diag spec: the same two sums over the paired points i of each block, weighted by wdiag[row0 + i]
void launch_grad_diag(const BlockDev& b, const double* wdiag, double* g, cudaStream_t s);

// potrf of diagonal block k (in place in the packed matrix) + explicit inverse of L_kk
// (dense NB x NB, ld NB) + per-block sum of log pivots + first failing pivot (1-based, 0 = ok)
// ldiag != nullptr: also store a contiguous copy of L_kk at ldiag + k*NB*NB (multi-GPU: it is
// broadcast together with the panel so every rank ends up with the complete factor)
// src != nullptr: the input block is read from src (column-major, ld_src) instead of the packed matrix
void launch_potrf_inv(Packed A, int64_t k, int64_t N, double* invL, double* logdet_blk,
                      long long* info, cudaStream_t s, double* ldiag = nullptr, const double* src = nullptr,
                      int64_t ld_src = 0);

// C = beta*C + alpha * A * B^T  (all column-major), M x Ncols x K, multiples of 128 / 64 / 16
void launch_gemm_nt(const double* A, int64_t lda, const double* B, int64_t ldb, double* C,
                    int64_t ldc, int64_t M, int64_t Ncols, int64_t K, double alpha, double beta,
                    cudaStream_t s);
// Panel TRSM writing the panel in TILED (k-slab image) layout: [row block][128 cols][132 padded
// rows]; see gemm_nt.cu.  tiled_panel_elems(m) doubles per half panel.
void launch_trsm_tiled(const double* A, int64_t lda, const double* invL, double* Pt, int64_t m,
                       cudaStream_t s);
inline int64_t tiled_panel_elems(int64_t m) { return (m / NB) * (int64_t)NB * (NB + 4); }
// tiled panel -> column-major block column of the packed matrix (rows below the diagonal block)
void launch_untile_panel(const double* Pt, int64_t row_blk0, int64_t nrow_blks, double* dst, int64_t ld,
                         cudaStream_t s);
// trailing update of the packed matrix with the nseg panels of the outer step starting at block
// column k, all in TILED layout:  A[I,J] -= sum_q P_q,I * P_q,J^T   for block columns J in
// [jlo, jhi) with (J % world) == rank, I >= J.  Row block 0 of the tiled buffers <-> block row k+1.
constexpr int OUTER_BLOCKS = 4;  // block columns per outer step: trailing updates use K = 512
// reserve_sms > 0: the persistent grid leaves that many SMs free (look-ahead: the next panel
// phase and its NCCL broadcast run there concurrently)
void launch_syrk_packed(Packed A, int64_t k, const double* const* Pt, int nseg, int64_t jlo, int64_t jhi,
                        int rank, int world, cudaStream_t s, int reserve_sms = 0);
// plain product with K-segmented operands (each segment 128 columns with its own base / ld)
void launch_gemm_nt_seg(int nseg, const double* const* A, const int64_t* lda, const double* const* B,
                        const int64_t* ldb, double* C, int64_t ldc, int64_t M, int64_t Ncols, double alpha,
                        double beta, cudaStream_t s);
int64_t syrk_packed_tiles(int64_t nblk, int64_t k, int64_t jlo, int64_t jhi, int rank, int world);

// one-launch persistent triangular sweep on the packed factor (solve.cu): S right-hand sides, column-major
// with ld = Np; flags = 2*nblk unsigned scratch
void launch_sweep(Packed L, const double* invL, double* b, int S, bool backward, unsigned* flags, int num_sms,
                  cudaStream_t s);
void launch_colsumsq(const double* v, int64_t n, int64_t ld, int S, double* out, cudaStream_t s);
// y[M] (+)= W[M x n] * a[n]   (W column-major, ld)
void launch_gemv_n(const double* W, int64_t ld, int64_t M, int64_t n, const double* a, double* y,
                   cudaStream_t s);
// acc[i] += sum_c X[i, c]^2 over ncols columns
void launch_rowsumsq_acc(const double* X, int64_t ld, int64_t M, int64_t ncols, double* acc,
                         cudaStream_t s);
void launch_sub(double* out, const double* a, const double* b, int64_t n, cudaStream_t s);
void launch_axpy1(double* y, const double* x, int64_t n, cudaStream_t s);
// dense lower-triangular L (N x N, ld N) from packed
void launch_unpack_lower(Packed L, int64_t N, double* out, cudaStream_t s);
// out[N x S] = L * z   (z: N x S, ld Np) -- used by sb_rand
void launch_trmv_lower(Packed L, int64_t N, const double* z, double* out, int S, cudaStream_t s);

// VFE helpers
void launch_rowscale(double* W, int64_t ld, int64_t rows, int64_t cols, const double* s, cudaStream_t st);
void launch_gemv_t(const double* W, int64_t ld, int64_t rows, int64_t cols, const double* x, double* y,
                   cudaStream_t st);
void launch_transpose(const double* in, int64_t ld_in, int64_t rows, int64_t cols, double* out,
                      int64_t ld_out, cudaStream_t st);
void launch_pack_lower(Packed L, const double* D, int64_t ld, double shift, cudaStream_t st);
void launch_add_dense_lower(Packed L, const double* D, int64_t ld, int64_t n, cudaStream_t st);
// appending observations (append.cu)
// packed S (order Ns) <- M M' + blockdiag(0_r, C) with M = [T; V]: T r x r lower (ld ldt), V (Ns - r) x r (ld ldv),
// C (Ns - r) x (Ns - r) (ld ldc, lower triangle read).  r = 0 packs C alone.
void launch_pack_schur(Packed S, int64_t Ns, int r, const double* C, int64_t ldc, const double* T, int64_t ldt,
                       const double* V, int64_t ldv, cudaStream_t st);
// C (n x n, ld) += Sigma on and below the diagonal: dense (n x n, ld n), else diag (n), else s2 I
void launch_add_noise_dense(double* C, int64_t ld, int64_t n, double s2, const double* diag, const double* dense,
                            cudaStream_t st);
// joint packed factor J, block columns [0, h / NB): rows [NB j, N1) of the old factor O, then the N2 rows of
// V (column-major, ld ldv, column = joint column), zero padding below
void launch_append_relayout(Packed J, Packed O, int64_t N1, int64_t N2, const double* V, int64_t ldv, int64_t h,
                            cudaStream_t st);
// VFE gradient helpers (sb_vfe_grad)
// D (n x n, ld n) <- s I
void launch_set_scaled_identity(double* D, int64_t n, double s, cudaStream_t st);
// beta[r] = (delta[r] - t[r]) / sigma2[r] for r < rows, 0 for rows <= r < rows_p
void launch_vfe_beta(const double* delta, const double* t, const double* sigma2, int64_t rows, int64_t rows_p,
                     double* beta, cudaStream_t st);
// d elbo / d sigma2_r = (beta_r^2 - (1 - lb_r) / sigma2_r) / 2 + (kff_r - sigma2_r la_r) / (2 sigma2_r^2),
// la_r = |a_r|^2, lb_r = |L_B^{-1} a_r|^2
void launch_vfe_noise_grad(const double* beta, const double* la, const double* lb, const double* kff,
                           const double* sigma2, int64_t rows, double* out, cudaStream_t st);
// out[i] = -(alpha_i^2 + P[i, i]) / 2 for i < n  (d elbo / d (K_uu + jitter)_ii)
void launch_vfe_uu_diag(const double* alpha, const double* P, int64_t ld, int64_t n, double* out, cudaStream_t st);

// ---- K3': trailing update on the int8 tensor cores (wgmma, int8 Ozaki slicing), ozaki.cu ------------------
struct alignas(64) OzMaps { unsigned char a[128]; unsigned char b[128]; };  // CUtensorMap blobs: A box (128 rows), B box (64 rows)
size_t oz_planes_bytes(int64_t Np);                       // 7 digit planes, 512-byte row pitch
int oz_make_maps(signed char* planes, int64_t Np, OzMaps* out);
// source panel of the slicer: up to 4 segments of 128 columns; element (row block rb, col k, row r) of
// segment q at base[q] + rb*rbs[q] + k*ld[q] + r.
// Column equilibration (colsign = -1 or +1, 0 = off): column k of segment q is multiplied by 2^(colsign * e),
// e = ilogb of the diagonal entry  diag[q][k * dld[q] + k]  (the step's L_kk).  The panel solve scales the columns
// of A21 by 2^-e and the same columns of inv(L_512) by 2^+e: the product is unchanged, and the digit planes of a row
// no longer span the range of the diagonal.
struct OzSrc {
    const double* base[4]; int64_t ld[4]; int64_t rbs[4]; int nseg;
    const double* diag[4]; int64_t dld[4]; int colsign;
};
void launch_oz_slice(const OzSrc& src, int64_t rb_lo, int64_t nrb, int64_t out_row_base, int64_t plane_rows,
                     double* scale, int* expo, signed char* planes, cudaStream_t s);
int launch_syrk_ozaki(Packed A, int64_t k, int nseg, int64_t jlo, int64_t jhi, int rank, int world,
                      const OzMaps* maps, const double* scale, cudaStream_t s, int reserve_sms = 0,
                      int64_t tile_lo = 0, int64_t tile_hi = 0);

// plain product C[M x Ncols] -= A B^T through the same kernel (dense column-major C)
int launch_gemm_ozaki(double* C, int64_t ldc, int64_t M, int64_t Ncols, int nseg, const OzMaps* mapsA,
                      const double* scaleA, int64_t rowA0, const OzMaps* mapsB, const double* scaleB, int64_t rowB0,
                      cudaStream_t s);
// X = A inv(L_512)^T over four block columns of the packed matrix (wide panel phase, ozaki.cu)
int launch_panel_solve_ozaki(double* const* Xcol, const int64_t* ldx, int64_t M, const OzMaps* mapsA, const double* scaleA,
                             int64_t rowA0, const OzMaps* mapsW, const double* scaleW, cudaStream_t s);

extern thread_local int64_t g_launch_count;

}  // namespace sb
