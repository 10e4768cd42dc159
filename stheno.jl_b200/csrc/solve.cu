// K4/K5/K6: vector triangular solves on the packed factor, reductions, posterior mean/var
// helpers.  All HBM-bound streaming kernels: every element of L is read exactly once per
// sweep with coalesced, row-contiguous accesses; reductions use warp shuffles.
// Replaces `C.U' \ delta`, `C \ delta`, `logdet(C)`, `sum(abs2, .)`, `diag_At_A`,
// `K_{*f} * alpha` of AbstractGPs (SURVEY.md App. A).
#include "sb_common.cuh"

namespace sb {
namespace {

constexpr int MAXS = 8;  // right-hand sides processed per pass

// ---- persistent triangular sweep ------------------------------------------------------------
// One launch per sweep instead of 2 launches per 128-wide block (1024 tiny dependent launches at
// N = 65536 would leave the sweep launch-latency bound).  Right-looking data flow with static ownership:
//   forward  b <- L^{-1} b :  when x_k = invL_kk b_k is final, every block row i > k applies
//                             b_i -= L[i,k] x_k;  b_{k+1} is final after k+1 such updates.
//   backward b <- L^{-T} b :  when x_k = invL_kk^T b_k is final, every block j < k applies
//                             b_j -= L[k,j]^T x_k.
// Block i (resp. j) is owned by worker CTA (i mod W) for the whole sweep, so updates of one block
// are sequential inside one CTA: no atomics on b, bit-reproducible results.  After each update the
// owner bumps done[i]; one dedicated CTA waits until block k has all its updates, does the diagonal
// solve and publishes ready[k] (release/acquire; x_k is read with ld.cg on the other SMs).  The serial
// chain per block is flag -> x_k -> one 128x128 product with L[k+1,k] -> flag -> one with invL_{k+1}
// -> flag, with each operand prefetched into L2 before the wait.  Each element of L is read once
// (17.2 GB/sweep).
struct SweepArgs {
    Packed L;
    const double* invL;
    double* b;        // Np x S, leading dimension L.Np
    int S;
    unsigned* ready;  // [nblk]
    unsigned* done;   // [nblk]
};

__device__ __forceinline__ unsigned ld_acquire(const unsigned* p) {
    unsigned v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_release(unsigned* p, unsigned v) {
    asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ void red_release_add(unsigned* p, unsigned v) {
    asm volatile("red.release.gpu.global.add.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ void spin_until(const unsigned* p, unsigned target) {
    long long t0 = 0;
    for (unsigned it = 0; ld_acquire(p) < target; it++) {
        if ((it & 0x3ff) == 0x3ff) {
            long long now = clock64();
            if (t0 == 0) t0 = now;
            else if (now - t0 > 40000000000LL) __trap();  // ~20 s: protocol bug, never hang the box
        }
    }
}

// out[r] (+)= sign * sum_c M[r, c] x[c]  for a 128 x 128 column-major block (ld), x in shared memory.
// 256 threads: thread (r, h) sums 64 columns; halves are combined through shared memory.
template <bool OVERWRITE>
__device__ __forceinline__ void block_matvec_n(const double* __restrict__ M, int64_t ld, const double (*xs)[NB],
                                               double* __restrict__ out, int64_t ldo, int S, double (*red)[NB]) {
    const int r = threadIdx.x & 127, h = threadIdx.x >> 7;
    const double* p = M + r + (int64_t)(h * 64) * ld;
    double acc[MAXS];
#pragma unroll
    for (int s = 0; s < MAXS; s++) acc[s] = 0.0;
#pragma unroll 16
    for (int c = 0; c < 64; c++) {
        const double l = __ldcs(p + (int64_t)c * ld);
#pragma unroll
        for (int s = 0; s < MAXS; s++)
            if (s < S) acc[s] = fma(l, xs[s][h * 64 + c], acc[s]);
    }
    if (h == 1) {
#pragma unroll
        for (int s = 0; s < MAXS; s++)
            if (s < S) red[s][r] = acc[s];
    }
    __syncthreads();
    if (h == 0) {
#pragma unroll
        for (int s = 0; s < MAXS; s++)
            if (s < S) {
                const double t = acc[s] + red[s][r];
                if (OVERWRITE) out[(int64_t)s * ldo + r] = t;
                else out[(int64_t)s * ldo + r] -= t;
            }
    }
    __syncthreads();
}

// out[c] (+)= sign * sum_r M[r, c] x[r]  (transposed product); warp w owns columns 16w .. 16w+15
template <bool OVERWRITE>
__device__ __forceinline__ void block_matvec_t(const double* __restrict__ M, int64_t ld, const double (*xs)[NB],
                                               double* __restrict__ out, int64_t ldo, int S) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int s = 0; s < S; s++) {
        double xr[4];
#pragma unroll
        for (int i = 0; i < 4; i++) xr[i] = xs[s][lane + 32 * i];
        double part[16];
#pragma unroll
        for (int cc = 0; cc < 16; cc++) {
            const double* colp = M + (int64_t)(warp * 16 + cc) * ld + lane;
            double a = 0.0;
#pragma unroll
            for (int i = 0; i < 4; i++) a = fma(__ldcs(colp + 32 * i), xr[i], a);
            part[cc] = a;
        }
#pragma unroll
        for (int cc = 0; cc < 16; cc++) {
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) part[cc] += __shfl_xor_sync(0xffffffffu, part[cc], o);
        }
        if (lane < 16) {
            double v = 0.0;
#pragma unroll
            for (int cc = 0; cc < 16; cc++) v = (lane == cc) ? part[cc] : v;
            double* o = out + (int64_t)s * ldo + warp * 16 + lane;
            if (OVERWRITE) *o = v; else *o -= v;
        }
    }
    __syncthreads();
}

__device__ __forceinline__ void prefetch_block_l2(const double* M, int64_t ld) {
    // 128 x 128 doubles = 1024 lines of 128 B: 4 per thread
    for (int idx = threadIdx.x; idx < 1024; idx += 256) {
        const double* p = M + (int64_t)(idx >> 3) * ld + (idx & 7) * 16;
        asm volatile("prefetch.global.L2 [%0];" ::"l"(p));
    }
}

template <bool BACKWARD>
__global__ void __launch_bounds__(256) sweep_kernel_a(SweepArgs a) {
    __shared__ double xs[MAXS][NB];
    __shared__ double red[MAXS][NB];
    const int64_t nblk = a.L.nblk(), Np = a.L.Np;
    const int S = a.S;
    const int G = gridDim.x;
    const int W = G > 1 ? G - 1 : 1;              // worker CTAs; CTA G-1 does the diagonal solves
    auto load_x = [&](int64_t k) {                 // x_k (written by another SM) -> shared memory
        for (int idx = threadIdx.x; idx < S * NB; idx += 256) {
            const int s = idx / NB, c = idx % NB;
            xs[s][c] = __ldcg(a.b + (int64_t)s * Np + k * NB + c);
        }
        __syncthreads();
    };
    auto diag_solve = [&](int64_t k) {
        load_x(k);
        const double* Mk = a.invL + k * (int64_t)NB * NB;
        if (!BACKWARD) block_matvec_n<true>(Mk, NB, xs, a.b + k * NB, Np, S, red);
        else block_matvec_t<true>(Mk, NB, xs, a.b + k * NB, Np, S);
    };
    auto update = [&](int64_t tgt, int64_t k) {   // block `tgt` absorbs x_k (already in xs)
        if (!BACKWARD) block_matvec_n<false>(a.L.blk(tgt, k), a.L.ld(k), xs, a.b + tgt * NB, Np, S, red);
        else block_matvec_t<false>(a.L.blk(k, tgt), a.L.ld(tgt), xs, a.b + tgt * NB, Np, S);
    };

    if (G == 1) {  // tiny problems: one CTA does everything in order
        for (int64_t kk = 0; kk < nblk; kk++) {
            const int64_t k = BACKWARD ? nblk - 1 - kk : kk;
            diag_solve(k);
            __syncthreads();
            load_x(k);
            if (!BACKWARD) { for (int64_t i = k + 1; i < nblk; i++) update(i, k); }
            else           { for (int64_t j = k - 1; j >= 0; j--) update(j, k); }
        }
        return;
    }

    if ((int)blockIdx.x == G - 1) {
        // ---- diagonal solves, in dependency order ----
        for (int64_t kk = 0; kk < nblk; kk++) {
            const int64_t k = BACKWARD ? nblk - 1 - kk : kk;
            prefetch_block_l2(a.invL + k * (int64_t)NB * NB, NB);
            if (threadIdx.x == 0) spin_until(a.done + k, (unsigned)kk);  // all kk updates of b_k applied
            __syncthreads();
            diag_solve(k);
            if (threadIdx.x == 0) { __threadfence(); st_release(a.ready + k, 1u); }
        }
        return;
    }
    // ---- workers ----
    const int me = blockIdx.x;
    for (int64_t kk = 0; kk + 1 < nblk; kk++) {
        const int64_t k = BACKWARD ? nblk - 1 - kk : kk;
        // nearest owned target first (it gates the next diagonal solve); skip steps with no work
        int64_t first;
        if (!BACKWARD) { first = k + 1 + (((me - (k + 1)) % W) + W) % W; if (first >= nblk) continue; }
        else           { first = k - 1 - ((((k - 1) - me) % W) + W) % W; if (first < 0) continue; }
        if (!BACKWARD) prefetch_block_l2(a.L.blk(first, k), a.L.ld(k));
        else prefetch_block_l2(a.L.blk(k, first), a.L.ld(first));
        if (threadIdx.x == 0) spin_until(a.ready + k, 1u);
        __syncthreads();
        load_x(k);
        if (!BACKWARD) {
            for (int64_t i = first; i < nblk; i += W) {
                update(i, k);
                if (threadIdx.x == 0) { __threadfence(); red_release_add(a.done + i, 1u); }
            }
        } else {
            for (int64_t j = first; j >= 0; j -= W) {
                update(j, k);
                if (threadIdx.x == 0) { __threadfence(); red_release_add(a.done + j, 1u); }
            }
        }
    }
}

// Deterministic reductions: per-block partial sums land in a scratch buffer and are added in
// a fixed order by a second tiny kernel -- no fp64 atomics, so logpdf / mean / var are bit-reproducible
// from run to run (and an imported factor reproduces the original bit for bit).
__global__ void __launch_bounds__(256)
colsumsq_kernel(const double* __restrict__ v, int64_t n, int64_t ld, double* __restrict__ partial) {
    const double* p = v + (int64_t)blockIdx.y * ld;
    double acc = 0.0;
    for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < n; i += (int64_t)gridDim.x * 256)
        acc = fma(p[i], p[i], acc);
    __shared__ double red[8];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        double t = 0.0;
        for (int w = 0; w < 8; w++) t += red[w];
        partial[(int64_t)blockIdx.y * gridDim.x + blockIdx.x] = t;
    }
}

// out[j] = sum_i partial[j * m + i]  in index order (one thread per output)
__global__ void sum_partials_kernel(const double* __restrict__ partial, int64_t m, int64_t nout, double* __restrict__ out,
                                    int accumulate) {
    int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= nout) return;
    double t = 0.0;
    for (int64_t i = 0; i < m; i++) t += partial[j * m + i];
    out[j] = accumulate ? out[j] + t : t;
}

// partial[cy * M + r] = sum over the 512 columns of chunk cy of W[r, c] a[c]
constexpr int GN_COLS = 512;
__global__ void __launch_bounds__(256)
gemv_n_kernel(const double* __restrict__ W, int64_t ld, int64_t M, int64_t n,
              const double* __restrict__ a, double* __restrict__ y) {
    __shared__ double as[GN_COLS];
    int64_t c0 = (int64_t)blockIdx.y * GN_COLS;
    int64_t nc = n - c0 < GN_COLS ? n - c0 : GN_COLS;
    for (int i = threadIdx.x; i < nc; i += 256) as[i] = a[c0 + i];
    __syncthreads();
    int64_t r = (int64_t)blockIdx.x * 256 + threadIdx.x;
    if (r >= M) return;
    const double* p = W + c0 * ld + r;
    double acc = 0.0;
#pragma unroll 8
    for (int c = 0; c < nc; c++) acc = fma(p[(int64_t)c * ld], as[c], acc);
    y[(int64_t)blockIdx.y * M + r] = acc;   // y = partial buffer [chunks][M]
}

// y[r] = sum over chunks (fixed order)
__global__ void sum_chunks_kernel(const double* __restrict__ partial, int64_t M, int64_t chunks, double* __restrict__ y) {
    int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= M) return;
    double t = 0.0;
    for (int64_t c = 0; c < chunks; c++) t += partial[c * M + r];
    y[r] = t;
}

// acc[r] += sum_c X[r, c]^2: 4 lanes per row (32 columns each, interleaved), combined by shuffles in a
// fixed order -- deterministic, and 4x the parallelism of one thread per row
__global__ void __launch_bounds__(256)
rowsumsq_acc_kernel(const double* __restrict__ X, int64_t ld, int64_t M, int64_t ncols,
                    double* __restrict__ acc_out) {
    const int part = threadIdx.x & 3;
    int64_t r = (int64_t)blockIdx.x * 64 + (threadIdx.x >> 2);
    double acc = 0.0;
    if (r < M) {
#pragma unroll 8
        for (int64_t c = part; c < ncols; c += 4) {
            double v = X[c * ld + r];
            acc = fma(v, v, acc);
        }
    }
    acc += __shfl_xor_sync(0xffffffffu, acc, 1);
    acc += __shfl_xor_sync(0xffffffffu, acc, 2);
    if (part == 0 && r < M) acc_out[r] += acc;
}

__global__ void axpy1_kernel(double* y, const double* x, int64_t n) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) y[i] += x[i];
}

__global__ void sub_kernel(double* out, const double* a, const double* b, int64_t n) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = a[i] - b[i];
}

__global__ void unpack_lower_kernel(Packed L, int64_t N, double* __restrict__ out) {
    int64_t c = blockIdx.x;
    int64_t r = (int64_t)blockIdx.y * 256 + threadIdx.x;
    if (r >= N || c >= N) return;
    out[c * N + r] = (r >= c) ? *L.at(r, c) : 0.0;
}

// out[rows of block I, sample s] = sum_{J <= I} L[I, J] z_J: one CTA per (block row, sample), the J loop is
// sequential inside the CTA (deterministic; rand(rng, fx) reproduces bit for bit)
__global__ void __launch_bounds__(NB)
trmv_lower_kernel(Packed L, int64_t N, const double* __restrict__ z, double* __restrict__ out,
                  int S) {
    const int64_t I = blockIdx.x;
    const int s = blockIdx.y;
    __shared__ double zs[NB];
    const int i = threadIdx.x;
    double acc = 0.0;
    for (int64_t J = 0; J <= I; J++) {
        __syncthreads();
        zs[i] = z[(int64_t)s * L.Np + J * NB + i];
        __syncthreads();
        const double* blk = L.blk(I, J);
        const int64_t ld = L.ld(J);
        const int cmax = (I == J) ? i + 1 : NB;
#pragma unroll 8
        for (int c = 0; c < cmax; c++) acc = fma(blk[(int64_t)c * ld + i], zs[c], acc);
    }
    out[(int64_t)s * L.Np + I * NB + i] = acc;
}

// W[r, c] *= s[r]
__global__ void __launch_bounds__(256)
rowscale_kernel(double* __restrict__ W, int64_t ld, int64_t rows, const double* __restrict__ s) {
    int64_t r = (int64_t)blockIdx.x * 256 + threadIdx.x;
    if (r >= rows) return;
    W[(int64_t)blockIdx.y * ld + r] *= s[r];
}

// y[c] += sum_r W[r, c] * x[r]   (columns are contiguous: one warp per column chunk)
__global__ void __launch_bounds__(256)
gemv_t_kernel(const double* __restrict__ W, int64_t ld, int64_t rows, const double* __restrict__ x,
              double* __restrict__ y) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int64_t c = (int64_t)blockIdx.y * 8 + warp;
    const int64_t r0 = (int64_t)blockIdx.x * 4096;
    const int64_t r1 = r0 + 4096 < rows ? r0 + 4096 : rows;
    const double* col = W + c * ld;
    double acc = 0.0;
#pragma unroll 8
    for (int64_t r = r0 + lane; r < r1; r += 32) acc = fma(col[r], x[r], acc);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if (lane == 0) atomicAdd(&y[c], acc);
}

// out[c, r] = in[r, c]  (in: rows x cols, ld_in; out: cols x rows, ld_out), 32x32 smem tiles
__global__ void __launch_bounds__(256)
transpose_kernel(const double* __restrict__ in, int64_t ld_in, double* __restrict__ out, int64_t ld_out) {
    __shared__ double t[32][33];
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    const int64_t r0 = (int64_t)blockIdx.x * 32, c0 = (int64_t)blockIdx.y * 32;
#pragma unroll
    for (int j = ty; j < 32; j += 8) t[j][tx] = in[(c0 + j) * ld_in + r0 + tx];
    __syncthreads();
#pragma unroll
    for (int j = ty; j < 32; j += 8) out[(r0 + j) * ld_out + c0 + tx] = t[tx][j];
}

// packed lower <- dense (n x n, ld), plus `shift` added on the diagonal
__global__ void __launch_bounds__(256)
pack_lower_kernel(Packed L, const double* __restrict__ D, int64_t ld, double shift) {
    int64_t c = blockIdx.x;
    int64_t r = (int64_t)blockIdx.y * 256 + threadIdx.x;
    if (r >= L.Np || r / NB < c / NB) return;
    double v = D[c * ld + r];
    if (r == c) v += shift;
    *L.at(r, c) = v;
}

// dst[(c) * ld + rb*128 + r] = Pt[((row_blk0 + rb) * 128 + c) * 132 + r]
__global__ void __launch_bounds__(128)
untile_panel_kernel(const double* __restrict__ Pt, int64_t row_blk0, double* __restrict__ dst, int64_t ld) {
    const int64_t rb = blockIdx.x;
    const int c = blockIdx.y, r = threadIdx.x;
    dst[(int64_t)c * ld + rb * NB + r] = Pt[((row_blk0 + rb) * NB + c) * (int64_t)(NB + 4) + r];
}

// packed lower += dense symmetric matrix (n x n, ld), lower triangle only
__global__ void __launch_bounds__(256)
add_dense_lower_kernel(Packed L, const double* __restrict__ D, int64_t ld, int64_t n) {
    int64_t c = blockIdx.x;
    int64_t r = (int64_t)blockIdx.y * 256 + threadIdx.x;
    if (r >= n || c >= n || r < c) return;
    *L.at(r, c) += D[c * ld + r];
}

__global__ void set_scaled_identity_kernel(double* D, int64_t n, double s) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) D[i * n + i] = s;
}

__global__ void vfe_beta_kernel(const double* __restrict__ delta, const double* __restrict__ t,
                                const double* __restrict__ sigma2, int64_t rows, int64_t rows_p,
                                double* __restrict__ beta) {
    int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r < rows_p) beta[r] = r < rows ? (delta[r] - t[r]) / sigma2[r] : 0.0;
}

__global__ void vfe_noise_grad_kernel(const double* __restrict__ beta, const double* __restrict__ la,
                                      const double* __restrict__ lb, const double* __restrict__ kff,
                                      const double* __restrict__ sigma2, int64_t rows, double* __restrict__ out) {
    int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= rows) return;
    const double s = sigma2[r];
    out[r] = 0.5 * (beta[r] * beta[r] - (1.0 - lb[r]) / s) + 0.5 * (kff[r] - s * la[r]) / (s * s);
}

__global__ void vfe_uu_diag_kernel(const double* __restrict__ alpha, const double* __restrict__ P, int64_t ld,
                                   int64_t n, double* __restrict__ out) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = -0.5 * (alpha[i] * alpha[i] + P[i * ld + i]);
}

}  // namespace

void launch_set_scaled_identity(double* D, int64_t n, double s, cudaStream_t st) {
    if (n <= 0) return;
    set_scaled_identity_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(D, n, s);
    g_launch_count++;
}

void launch_vfe_beta(const double* delta, const double* t, const double* sigma2, int64_t rows, int64_t rows_p,
                     double* beta, cudaStream_t st) {
    if (rows_p <= 0) return;
    vfe_beta_kernel<<<(unsigned)((rows_p + 255) / 256), 256, 0, st>>>(delta, t, sigma2, rows, rows_p, beta);
    g_launch_count++;
}

void launch_vfe_noise_grad(const double* beta, const double* la, const double* lb, const double* kff,
                           const double* sigma2, int64_t rows, double* out, cudaStream_t st) {
    if (rows <= 0) return;
    vfe_noise_grad_kernel<<<(unsigned)((rows + 255) / 256), 256, 0, st>>>(beta, la, lb, kff, sigma2, rows, out);
    g_launch_count++;
}

void launch_vfe_uu_diag(const double* alpha, const double* P, int64_t ld, int64_t n, double* out, cudaStream_t st) {
    if (n <= 0) return;
    vfe_uu_diag_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(alpha, P, ld, n, out);
    g_launch_count++;
}


// whole forward (backward = true: transposed) sweep b <- L^{-1} b / L^{-T} b in ONE launch;
// flags: 2*nblk unsigned scratch (zeroed here)
void launch_sweep(Packed L, const double* invL, double* b, int S, bool backward, unsigned* flags, int num_sms,
                  cudaStream_t s) {
    const int64_t nblk = L.nblk();
    cudaMemsetAsync(flags, 0, 2 * nblk * sizeof(unsigned), s);
    SweepArgs a{L, invL, b, S, flags, flags + nblk};
    const int grid = nblk < 4 ? 1 : (int)(nblk + 1 < num_sms ? nblk + 1 : num_sms);
    if (backward) sweep_kernel_a<true><<<grid, 256, 0, s>>>(a);
    else sweep_kernel_a<false><<<grid, 256, 0, s>>>(a);
    g_launch_count++;
}

void launch_add_dense_lower(Packed L, const double* D, int64_t ld, int64_t n, cudaStream_t st) {
    if (n <= 0) return;
    add_dense_lower_kernel<<<dim3((unsigned)n, (unsigned)((n + 255) / 256)), 256, 0, st>>>(L, D, ld, n);
    g_launch_count++;
}

void launch_untile_panel(const double* Pt, int64_t row_blk0, int64_t nrow_blks, double* dst, int64_t ld,
                         cudaStream_t st) {
    if (nrow_blks <= 0) return;
    untile_panel_kernel<<<dim3((unsigned)nrow_blks, NB), NB, 0, st>>>(Pt, row_blk0, dst, ld);
    g_launch_count++;
}

void launch_rowscale(double* W, int64_t ld, int64_t rows, int64_t cols, const double* s, cudaStream_t st) {
    if (rows <= 0 || cols <= 0) return;
    rowscale_kernel<<<dim3((unsigned)((rows + 255) / 256), (unsigned)cols), 256, 0, st>>>(W, ld, rows, s);
    g_launch_count++;
}

void launch_gemv_t(const double* W, int64_t ld, int64_t rows, int64_t cols, const double* x, double* y,
                   cudaStream_t st) {
    if (rows <= 0 || cols <= 0) return;  // cols must be a multiple of 8
    gemv_t_kernel<<<dim3((unsigned)((rows + 4095) / 4096), (unsigned)(cols / 8)), 256, 0, st>>>(W, ld, rows, x, y);
    g_launch_count++;
}

void launch_transpose(const double* in, int64_t ld_in, int64_t rows, int64_t cols, double* out, int64_t ld_out,
                      cudaStream_t st) {
    // rows, cols multiples of 32
    transpose_kernel<<<dim3((unsigned)(rows / 32), (unsigned)(cols / 32)), 256, 0, st>>>(in, ld_in, out, ld_out);
    g_launch_count++;
}

void launch_pack_lower(Packed L, const double* D, int64_t ld, double shift, cudaStream_t st) {
    pack_lower_kernel<<<dim3((unsigned)L.Np, (unsigned)((L.Np + 255) / 256)), 256, 0, st>>>(L, D, ld, shift);
    g_launch_count++;
}

// scratch for the two-stage reductions (grown on demand, one per thread / context)
static thread_local double* g_red_scratch = nullptr;
static thread_local size_t g_red_scratch_elems = 0;
static double* red_scratch(size_t elems) {
    if (elems > g_red_scratch_elems) {
        if (g_red_scratch) cudaFree(g_red_scratch);
        g_red_scratch = nullptr;
        if (cudaMalloc(&g_red_scratch, elems * sizeof(double)) != cudaSuccess) { g_red_scratch_elems = 0; return nullptr; }
        g_red_scratch_elems = elems;
    }
    return g_red_scratch;
}

void launch_colsumsq(const double* v, int64_t n, int64_t ld, int S, double* out, cudaStream_t s) {
    int64_t gx = (n + 255) / 256;
    if (gx > 256) gx = 256;
    double* part = red_scratch((size_t)gx * S);
    if (!part) return;
    colsumsq_kernel<<<dim3((unsigned)gx, S), 256, 0, s>>>(v, n, ld, part);
    sum_partials_kernel<<<(unsigned)((S + 63) / 64), 64, 0, s>>>(part, gx, S, out, 0);
    g_launch_count += 2;
}

void launch_gemv_n(const double* W, int64_t ld, int64_t M, int64_t n, const double* a, double* y,
                   cudaStream_t s) {
    const int64_t chunks = (n + GN_COLS - 1) / GN_COLS;
    double* part = red_scratch((size_t)chunks * M);
    if (!part) return;
    dim3 grid((unsigned)((M + 255) / 256), (unsigned)chunks);
    gemv_n_kernel<<<grid, 256, 0, s>>>(W, ld, M, n, a, part);
    sum_chunks_kernel<<<(unsigned)((M + 255) / 256), 256, 0, s>>>(part, M, chunks, y);
    g_launch_count += 2;
}

void launch_rowsumsq_acc(const double* X, int64_t ld, int64_t M, int64_t ncols, double* acc,
                         cudaStream_t s) {
    rowsumsq_acc_kernel<<<(unsigned)((M + 63) / 64), 256, 0, s>>>(X, ld, M, ncols, acc);
    g_launch_count++;
}

void launch_axpy1(double* y, const double* x, int64_t n, cudaStream_t s) {
    if (n <= 0) return;
    axpy1_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(y, x, n);
    g_launch_count++;
}

void launch_sub(double* out, const double* a, const double* b, int64_t n, cudaStream_t s) {
    if (n <= 0) return;
    sub_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(out, a, b, n);
    g_launch_count++;
}

void launch_unpack_lower(Packed L, int64_t N, double* out, cudaStream_t s) {
    dim3 grid((unsigned)N, (unsigned)((N + 255) / 256));
    unpack_lower_kernel<<<grid, 256, 0, s>>>(L, N, out);
    g_launch_count++;
}

void launch_trmv_lower(Packed L, int64_t N, const double* z, double* out, int S, cudaStream_t s) {
    dim3 grid((unsigned)L.nblk(), (unsigned)S);
    trmv_lower_kernel<<<grid, NB, 0, s>>>(L, N, z, out, S);
    g_launch_count++;
}

}  // namespace sb
