/* stheno_b200.h -- C ABI of the H100-native (sm_90a) dense-GP hot path (libstheno_b200.so).
 *
 * The reference (Stheno.jl) has no FFI: its seam is Julia dispatch on the
 * "internal AbstractGPs API" (docs/src/internals.md:8-24) -- AbstractGPs calls
 * mean/cov/var(f, x[, x']) on the GPPP (src/gaussian_process_probabilistic_programme.jl:45-80)
 * and then does cholesky/logdet/solves itself on host matrices.  This ABI intercepts ONE LEVEL
 * HIGHER (FiniteGP methods) so the covariance matrix never exists on the host.  Each entry
 * point cites the reference call path it replaces.  The Julia `ccall` stub that binds each
 * symbol is in INTEGRATION.md / stheno.jl_b200/julia/SthenoB200.jl; tests and bench drive the
 * very same symbols through ctypes (stheno.jl_b200/lib.py).
 *
 * Conventions
 *   - extern "C", plain pointers and sizes; every function returns an int32 status
 *     (SB_OK == 0, negative = error class; text via sb_last_error()).
 *   - All real data is IEEE fp64 (sb_dtype SB_F64; SB_F32 is reserved, returns
 *     SB_ERR_UNSUPPORTED in this round).
 *   - Data pointers may be HOST or DEVICE pointers (classified with
 *     cudaPointerGetAttributes): host buffers are staged through pinned memory inside the
 *     call; device buffers are used in place.  Outputs likewise.  The library works on its
 *     own non-blocking streams: a DEVICE buffer must be complete (its producer stream
 *     synchronised, e.g. CUDA.synchronize() / torch.cuda.synchronize()) before the call.
 *   - The caller owns every buffer it passes for the duration of the call (Julia:
 *     GC.@preserve).  The library owns device memory and the opaque handles; handles are
 *     released with the matching *_destroy (Julia: finalizer).
 *   - A ctx is bound to one CUDA device and one stream; calls are synchronous and a ctx is
 *     not thread-safe (the reference is not either: `cross` mutates the GPC counter during
 *     `cov`, src/affine_transformations/cross.jl:37-40).
 *   - Means are host-side (user closures, src/affine_transformations/addition.jl:73-74): the
 *     ABI takes delta = y - mean(x) and the caller adds mean(x*) back.
 *   - Matrices are column-major (Julia `Matrix`).
 *
 * Covariance specification ("lowered plan")
 *   The host flattens cov(f_p, f_q)(x, x') for every block pair of the requested
 *   BlockData x BlockData grid (src/affine_transformations/cross.jl:59-86 with the recursion
 *   of src/gp/derived_gp.jl:31-59) into a list of terms
 *        K[i, j] = sum_t  coeff_t * sl_t[i] * sr_t[j] * kappa_t( zl_t[i], zr_t[j] )
 *   where kappa is a fixed stationary base kernel (KernelFunctions semantics), zl/zr are the
 *   host-evaluated transformed inputs (compose.jl:16-28), sl/sr the host-evaluated scale
 *   vectors (product.jl:25-70).  A block with zero terms is the `zeros(...)` of
 *   src/gp/atomic_gp.jl:36-38 / src/gp/derived_gp.jl:37-38.
 */
#ifndef STHENO_B200_H
#define STHENO_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SB_ABI_VERSION 1

/* status codes */
#define SB_OK 0
#define SB_ERR_INVALID (-1)     /* bad argument / malformed spec */
#define SB_ERR_CUDA (-2)        /* CUDA runtime error (text in sb_last_error) */
#define SB_ERR_NOT_POSDEF (-3)  /* Cholesky pivot <= 0; *info = 1-based index (LAPACK info) */
#define SB_ERR_UNSUPPORTED (-4) /* feature reserved in the ABI but not built in this round */
#define SB_ERR_NCCL (-5)
#define SB_ERR_NOMEM (-6)

/* base kernels: KernelFunctions.jl semantics (SURVEY.md Appendix A) */
typedef enum {
    SB_K_SE = 0,       /* exp(-d^2/2),  d^2 = max(|x|^2+|y|^2-2x'y, 0)   (SqEuclidean)   */
    SB_K_MATERN12 = 1, /* exp(-d),      d = sqrt(d^2)                     (Euclidean)     */
    SB_K_MATERN32 = 2, /* (1+sqrt3 d) exp(-sqrt3 d)                                        */
    SB_K_MATERN52 = 3, /* (1+sqrt5 d+5d^2/3) exp(-sqrt5 d)                                 */
    SB_K_WHITE = 4,    /* x == y ? 1 : 0   (exact equality of every coordinate)            */
    SB_K_CONST = 5     /* param                                                            */
} sb_kernel_id;

typedef enum { SB_F64 = 0, SB_F32 = 1 } sb_dtype;

/* point-major array of n points of dimension dim  (== Julia ColVecs D x n column-major, or
 * Vector{Float64} for dim == 1); dim == 0 marks a scale vector of length n. */
typedef struct {
    const void* data;
    int64_t n;
    int32_t dim;
    int32_t reserved;
} sb_array;

typedef struct {
    int32_t kernel; /* sb_kernel_id */
    int32_t zl;     /* index into arrays: transformed row inputs  (length = block nrows) */
    int32_t zr;     /* index into arrays: transformed col inputs  (length = block ncols) */
    int32_t sl;     /* index of row scale vector or -1 (== ones) */
    int32_t sr;     /* index of col scale vector or -1 */
    int32_t reserved;
    double coeff;
    double param;
} sb_term;

typedef struct {
    int64_t row0, nrows; /* 0-based rows of the block in the assembled matrix */
    int64_t col0, ncols;
    int32_t term0, nterms; /* terms[term0 .. term0+nterms) */
} sb_block;

typedef struct {
    int64_t nrows, ncols;
    int32_t symmetric; /* 1: only blocks on/below the block diagonal are listed (factor path) */
    int32_t narrays;
    const sb_array* arrays;
    int32_t nterms;
    const sb_term* terms;
    int32_t nblocks;
    const sb_block* blocks;
} sb_covspec;

/* observation noise Sigma_y (AbstractGPs FiniteGP(f, x, Sigma)): scalar -> sigma2*I;
 * diag != NULL -> Diagonal(diag) (n values); dense != NULL -> full symmetric PSD matrix
 * (n x n column-major, only its lower triangle is read), as exercised by
 * test/affine_transformations/test_util.jl:114-127.  Exactly one form is used:
 * dense, else diag, else scalar. */
typedef struct {
    double sigma2;
    const void* diag;  /* NULL or n values */
    const void* dense; /* NULL or n*n values, column-major, leading dimension n */
} sb_noise;

typedef struct {
    double assemble_ms; /* K1 tile assembly */
    double panel_ms;    /* panel work on the critical path: first serial phase + the tensor-core panel solves */
    double trailing_ms; /* SYRK/GEMM trailing updates (DMMA, or int8 Ozaki slices) */
    double solve_ms;    /* vector triangular solves + reductions */
    double predict_ms;  /* cross assembly + matrix TRSM + mean/var */
    double comm_ms;     /* block-column exchange (peer copies; NCCL broadcast on the fallback path), incl. waiting for the owners */
    double total_ms;
    double trailing_flops; /* algorithmic flops executed by the trailing-update kernel */
    double trailing_kernel_ms; /* sum of per-launch CUDA-event durations of that kernel */
    int64_t trailing_launches;
    int64_t kernel_launches; /* all kernels launched by this library since last reset */
    double trailing_int8_ops; /* int8 tensor-core ops (2 * MACs) issued by the int8 Ozaki trailing kernel; 0 on the DMMA path */
    double panel_chain_ms;    /* total duration of the serial panel phases on the second stream (hidden under T^B) */
} sb_timings;

typedef struct sb_ctx sb_ctx;
typedef struct sb_factor sb_factor;
typedef struct sb_vfe sb_vfe;

int32_t sb_abi_version(void);
const char* sb_last_error(void);

/* ---- context -------------------------------------------------------------------------- */
int32_t sb_ctx_create(int32_t device, sb_ctx** out);
/* Multi-GPU (one process per GPU): nccl_id = 128-byte ncclUniqueId obtained from
 * sb_nccl_unique_id on rank 0 and distributed by the host (torch.distributed / MPI / file). */
int32_t sb_nccl_unique_id(void* id128);
int32_t sb_ctx_create_dist(int32_t device, int32_t rank, int32_t world, const void* nccl_id128,
                           sb_ctx** out);
int32_t sb_ctx_destroy(sb_ctx* ctx);
int32_t sb_ctx_timings(sb_ctx* ctx, sb_timings* out, int32_t reset);
/* options: "trailing" = 0 fp64 DMMA (mma.sync, default) | 1 int8 Ozaki slices on wgmma (also env
 * SB_TRAILING=dmma|ozaki at context creation); "fine_timing" = 0 | 1. */
int32_t sb_ctx_set_option(sb_ctx* ctx, const char* key, int64_t value);
/* benchmark support: record a CUDA event on the library's stream into slot 0..7 / read the
 * elapsed device time between two recorded slots (synchronises on the later one). */
int32_t sb_ctx_mark(sb_ctx* ctx, int32_t slot);
int32_t sb_ctx_elapsed_ms(sb_ctx* ctx, int32_t slot_a, int32_t slot_b, double* ms);

/* ---- multi-GPU partition helpers (pure host arithmetic; also what the CPU gloo tests check) --
 * sb_owner_of_block: rank owning block column J (1-D block-cyclic).
 * sb_owned_trailing_tiles: number of 128x128 trailing tiles (k < J <= I < nblk) rank updates at
 *   step k.  sb_row_chunk: contiguous [lo, hi) share of ns posterior test points for a rank. */
int32_t sb_owner_of_block(int64_t J, int32_t world);
int64_t sb_owned_trailing_tiles(int64_t nblk, int64_t k, int32_t rank, int32_t world);
int32_t sb_row_chunk(int64_t ns, int32_t rank, int32_t world, int64_t* lo, int64_t* hi);

/* ---- covariance assembly ---------------------------------------------------------------
 * sb_cov_dense replaces  cov(f::GPPP, x[, x'])  -> Matrix
 *   (gaussian_process_probabilistic_programme.jl:50-64 -> cross.jl:59-86 ->
 *    KernelFunctions.kernelmatrix); spec lists ALL blocks (symmetric == 0).
 *   K_out: column-major nrows x ncols, leading dimension nrows.
 * sb_cov_diag replaces  var(f::GPPP, x[, x'])  (gppp.jl:55-58,66-70 -> cross.jl:64-77 ->
 *   kernelmatrix_diag, src/gp/util.jl:5-7): every block has nrows == ncols and is evaluated
 *   elementwise (point i with point i, direct-difference distance as Distances.colwise). */
int32_t sb_cov_dense(sb_ctx* ctx, const sb_covspec* spec, void* K_out);
int32_t sb_cov_diag(sb_ctx* ctx, const sb_covspec* spec, void* out);

/* ---- exact inference ---------------------------------------------------------------------
 * sb_factor_create replaces  cholesky(Symmetric(cov(fx)))  with cov(fx) = cov(f,x) + Sigma_y
 *   (AbstractGPs logpdf/posterior/rand; call sites README.md:61-96, test/gp/util.jl:82-87).
 *   spec.symmetric must be 1.  On SB_ERR_NOT_POSDEF *info is LAPACK's info (PosDefException).
 * sb_logpdf replaces  logpdf(fx, y) / logpdf(fx, Y):  out[s] = -(N log 2pi + logdet +
 *   |L^{-1} delta_s|^2)/2 for the S columns of delta (N x S, column-major).
 * sb_factor_set_data replaces  posterior(fx, y): stores alpha = C \ delta in the handle.
 * sb_predict replaces  mean/var/mean_and_var/marginals(f_post(x*)): cross = cov(prior, x*, x)
 *   (N* x N, all blocks), prior_diag = var(prior, x*) as a diag spec.
 *   mean_out = cross*alpha (caller adds m(x*)),  var_out = prior_diag - colsumsq(L^{-1} cross').
 *   Either output may be NULL.
 * sb_predict_cov replaces  cov(f_post(x*)) : prior_full = cov(prior, x*) dense spec;
 *   cov_out = prior_full - V'V, column-major N* x N*.
 * sb_rand replaces  rand(rng, fx, S):  out = L * z  (z = randn(rng, N, S) drawn by the host,
 *   caller adds the mean).  */
int32_t sb_factor_create(sb_ctx* ctx, const sb_covspec* spec, const sb_noise* noise,
                         sb_factor** out, int64_t* info);
int32_t sb_factor_destroy(sb_factor* f);
int32_t sb_factor_logdet(sb_ctx* ctx, sb_factor* f, double* out);
int32_t sb_logpdf(sb_ctx* ctx, sb_factor* f, const void* delta, int32_t S, double* out);
int32_t sb_factor_set_data(sb_ctx* ctx, sb_factor* f, const void* delta);
int32_t sb_factor_alpha(sb_ctx* ctx, sb_factor* f, void* alpha_out);
/* sb_factor_set_alpha: install a previously computed alpha (N values) as the handle's current
 * posterior weights.  `posterior(fx, y)` is a pure function in the reference (AbstractGPs
 * PosteriorGP keeps its own alpha next to the shared Cholesky): two posteriors built from one fx
 * share the device factor and each re-installs its alpha before predicting. */
int32_t sb_factor_set_alpha(sb_ctx* ctx, sb_factor* f, const void* alpha);
int32_t sb_predict(sb_ctx* ctx, sb_factor* f, const sb_covspec* cross,
                   const sb_covspec* prior_diag, void* mean_out, void* var_out);
int32_t sb_predict_cov(sb_ctx* ctx, sb_factor* f, const sb_covspec* cross,
                       const sb_covspec* prior_full, void* cov_out);
int32_t sb_rand(sb_ctx* ctx, sb_factor* f, const void* z, int32_t S, void* out);
/* sb_predict_factor replaces  cholesky(Symmetric(cov(f_post(x*, noise))))  -- what
 * rand / logpdf of a POSTERIOR FiniteGP do (README.md:96, examples/process_decomposition/
 * script.jl:36): the N* x N* posterior covariance  prior_full - V'V + noise  is formed and
 * factorised on the device; the returned handle works with sb_rand / sb_logpdf / sb_factor_logdet. */
int32_t sb_predict_factor(sb_ctx* ctx, sb_factor* f, const sb_covspec* cross, const sb_covspec* prior_full,
                          const sb_noise* noise, sb_factor** out, int64_t* info);
/* sb_factor_append replaces posterior(f_post(x2, Sigma2), y2)'s factor update (AbstractGPs update_chol):
 * *out = cholesky of the covariance of the stacked observations [x; x2] with block-diagonal noise
 * (f's own noise, then Sigma2).  cross = cov(prior, x2, x) dense spec (N2 x N, all blocks); prior_full =
 * cov(prior, x2) dense spec (N2 x N2) -- the same two specs sb_predict_factor takes.  f is not modified;
 * the new handle has no alpha (call sb_factor_set_data).  On SB_ERR_NOT_POSDEF *info is the 1-based
 * pivot in the JOINT order (> N).  Multi-GPU: every rank calls it; the work is replicated (no communication).
 * Cost O(N2 N^2 + N2^2 N + N2^3): f's full 128-wide block columns are kept, only the rows of its partial
 * last block are factorised again together with the new ones. */
int32_t sb_factor_append(sb_ctx* ctx, sb_factor* f, const sb_covspec* cross, const sb_covspec* prior_full,
                         const sb_noise* noise, sb_factor** out, int64_t* info);
/* sb_logpdf_grad replaces the reverse-mode pass through logpdf(fx, y) (Zygote + the ChainRules
 * glue of src/affine_transformations/cross.jl:8-22; examples/getting_started/script.jl:154-213):
 *   dlogpdf/dtheta = 1/2 tr((alpha alpha' - K^{-1}) dK/dtheta)
 * spec = the symmetric spec the factor was built from; sb_factor_set_data(delta) must have been
 * called.  g_terms[2t] = d/d coeff_t, g_terms[2t+1] = d/d log(s_t) where the term's inputs are
 * z = s_t x (lengthscale derivative; 0 for White / Constant).  g_noise_diag[i] = 1/2 (alpha_i^2 -
 * (K^{-1})_ii) = d/d Sigma_y[i,i]  (scalar noise: sum them).  The host applies the chain rule to its
 * own hyper-parameters (kernel variance multiplies coeff, 1/lengthscale is s). */
int32_t sb_logpdf_grad(sb_ctx* ctx, sb_factor* f, const sb_covspec* spec, double* g_terms,
                       void* g_noise_diag);
/* Factor checkpoint (SURVEY.md 8f.4; the reference's PosteriorGP is a plain serialisable struct
 * (alpha, C, x, delta)): sb_factor_export writes header | packed L | diagonal-block inverses | alpha
 * into a caller buffer (host or device) of sb_factor_export_size bytes; sb_factor_import rebuilds a
 * handle that behaves exactly like the original (logpdf / predict / rand, bit-identical). */
int32_t sb_factor_export_size(sb_ctx* ctx, sb_factor* f, int64_t* nbytes);
int32_t sb_factor_export(sb_ctx* ctx, sb_factor* f, void* blob, int64_t nbytes);
int32_t sb_factor_import(sb_ctx* ctx, const void* blob, int64_t nbytes, sb_factor** out);
/* debug / parity: copy the lower-triangular factor out as a dense column-major N x N matrix */
int32_t sb_factor_get_L(sb_ctx* ctx, sb_factor* f, void* L_out);

/* ---- VFE / elbo --------------------------------------------------------------------------
 * Replaces AbstractGPs elbo/dtc/posterior(VFE(fz), fx, y) reached through
 * src/gp/sparse_finite_gp.jl:52-62.  uu = cov(fz) (symmetric spec, M x M) with its jitter
 * noise_u; xu = cov(f, x, z) dense spec (N x M, all blocks); ff_diag = var(f, x) diag spec;
 * noise_f the (diagonal) observation noise; delta = y - m(x).  out2 = {elbo, dtc}.
 * K_fu is streamed in row chunks and never held whole; multi-GPU: chunks are sharded and the
 * M x M accumulator is all-reduced. */
int32_t sb_vfe_create(sb_ctx* ctx, const sb_covspec* uu, const sb_noise* noise_u,
                      const sb_covspec* xu, const sb_covspec* ff_diag, const sb_noise* noise_f,
                      const void* delta, sb_vfe** out, double* out2, int64_t* info);
/* sb_vfe_grad: gradient of the elbo of handle v (reverse mode of AbstractGPs elbo(VFE(fz), fx, y),
 * src/gp/sparse_finite_gp.jl:52-58).  uu, xu, ff_diag, noise_f and delta are the ones v was created from
 * (N and M must match the handle, noise_f diagonal and > 0).
 * g_uu / g_xu / g_ff: 2 * nterms of each spec, [2t] = d/d coeff_t, [2t+1] = d/d log(input scale_t).
 * g_noise_u_diag[M] = d/d (K_uu + jitter)_ii,  g_noise_f_diag[N] = d/d Sigma_y[i,i].
 * The K_fu chunks of sb_vfe_create are streamed again (sharded over ranks, one all-reduce). */
int32_t sb_vfe_grad(sb_ctx* ctx, sb_vfe* v, const sb_covspec* uu, const sb_covspec* xu,
                    const sb_covspec* ff_diag, const sb_noise* noise_f, const void* delta,
                    double* g_uu, double* g_xu, double* g_ff, void* g_noise_u_diag, void* g_noise_f_diag);
int32_t sb_vfe_predict(sb_ctx* ctx, sb_vfe* v, const sb_covspec* cross /* N* x M */,
                       const sb_covspec* prior_diag, void* mean_out, void* var_out);
/* sb_vfe_predict_cov replaces  cov(f_approx_post(x*)) = K** - B'B + (L_Lambda^{-1}B)'(L_Lambda^{-1}B)
 * with B = L_u^{-1} K_u*  (AbstractGPs approximate posterior; SURVEY.md App. A);
 * prior_full = cov(prior, x*) dense spec, cov_out column-major N* x N*. */
int32_t sb_vfe_predict_cov(sb_ctx* ctx, sb_vfe* v, const sb_covspec* cross /* N* x M */,
                           const sb_covspec* prior_full, void* cov_out);
int32_t sb_vfe_destroy(sb_vfe* v);

#ifdef __cplusplus
}
#endif
#endif /* STHENO_B200_H */
