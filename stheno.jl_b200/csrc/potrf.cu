// K2: Cholesky of one NB x NB diagonal block, entirely in shared memory, plus the explicit
// inverse of the resulting triangle (used to turn the panel TRSM and every later block
// triangular solve into tensor-core products) and the block's share of logdet.
// Replaces the unblocked dpotf2 step inside LAPACK dpotrf (AbstractGPs
// `cholesky(Symmetric(cov(fx)))`, SURVEY.md App. A).  Latency-bound, one CTA: it is the serial
// critical path of the factorisation (and of the multi-GPU pipeline), so it is blocked by 8
// columns: 16 outer steps (instead of 128) with rank-8 trailing updates from registers, and a
// blocked triangular inverse (8x8 diagonal inverses + block back-substitution).
#include "sb_common.cuh"

namespace sb {
namespace {

constexpr int LDS = NB + 4;
constexpr int PT = 512;
constexpr int PB = 8;            // panel width inside the block
constexpr int NPB = NB / PB;     // 16 panels
constexpr size_t POTRF_SMEM = (size_t)NB * LDS * 8 + (size_t)NPB * PB * PB * 8 + (size_t)NB * PB * 8 + NB * 8 + 64;

__global__ void __launch_bounds__(PT, 1)
potrf_inv_kernel(Packed A, int64_t k, int64_t N, double* __restrict__ invL,
                 double* __restrict__ logdet_blk, long long* __restrict__ info,
                 double* __restrict__ ldiag, const double* __restrict__ src, int64_t ld_src) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    double* s = reinterpret_cast<double*>(smem_raw);   // s[c*LDS + r]: the block, column-major
    double* dinv = s + NB * LDS;                       // [NPB][PB*PB]: inverses of the 8x8 diagonal blocks (col-major)
    double* ybuf = dinv + NPB * PB * PB;               // [PB][NB] staging for the inverse sweep
    double* rdiag = ybuf + NB * PB;                    // [NB] reciprocals of the pivots
    int* bad = reinterpret_cast<int*>(rdiag + NB);

    const int tid = threadIdx.x;
    double* Akk = A.blk(k, k);
    const int64_t ld = A.ld(k);

    // the block is read from `src` when given (wide panel phase: the step's dense diagonal scratch) and
    // always written to the packed matrix
    const double* Ain = src != nullptr ? src : Akk;
    const int64_t ldin = src != nullptr ? ld_src : ld;
    for (int idx = tid; idx < NB * NB; idx += PT) {
        int r = idx % NB, c = idx / NB;
        s[c * LDS + r] = (r >= c) ? Ain[(int64_t)c * ldin + r] : 0.0;
    }
    if (tid == 0) *bad = 0;
    __syncthreads();

    // ================= blocked right-looking Cholesky =================
    const int ri = tid % NB, lg = tid / NB;  // row, column group (4 groups)
    for (int jb = 0; jb < NPB; jb++) {
        const int j0 = jb * PB;
        // (a1) 8x8 diagonal block, one thread, fully unrolled in registers
        if (tid == 0) {
            double d[PB][PB];
#pragma unroll
            for (int c = 0; c < PB; c++)
#pragma unroll
                for (int r = 0; r < PB; r++) d[r][c] = (r >= c) ? s[(j0 + c) * LDS + j0 + r] : 0.0;
#pragma unroll
            for (int c = 0; c < PB; c++) {
                double piv = d[c][c];
                if (!(piv > 0.0)) {  // also catches NaN
                    if (*bad == 0) *bad = j0 + c + 1;
                    piv = 1.0;       // keep going with finite garbage; info reports the failure
                }
                // one slow op (rsqrt) instead of sqrt + divide on the serial critical path
                double rinv = rsqrt(piv), r = piv * rinv;
                r = fma(fma(-r, r, piv), 0.5 * rinv, r);  // one Newton step: r is sqrt(piv) to < 1 ulp
                rinv = fma(fma(-r, rinv, 1.0), rinv, rinv);  // Newton step for 1/r (no divide)
                d[c][c] = r;
                rdiag[j0 + c] = rinv;
#pragma unroll
                for (int i = c + 1; i < PB; i++) d[i][c] *= rinv;
#pragma unroll
                for (int l = c + 1; l < PB; l++)
#pragma unroll
                    for (int i = l; i < PB; i++) d[i][l] -= d[i][c] * d[l][c];
            }
#pragma unroll
            for (int c = 0; c < PB; c++)
#pragma unroll
                for (int r = c; r < PB; r++) s[(j0 + c) * LDS + j0 + r] = d[r][c];
        }
        __syncthreads();
        // (a2) rows below the diagonal block: x * L8^T = a  (forward substitution per row)
        if (tid < NB && tid >= j0 + PB) {
            double a[PB];
#pragma unroll
            for (int c = 0; c < PB; c++) a[c] = s[(j0 + c) * LDS + tid];
#pragma unroll
            for (int c = 0; c < PB; c++) {
                double acc = a[c];
#pragma unroll
                for (int p = 0; p < c; p++) acc -= a[p] * s[(j0 + p) * LDS + j0 + c];
                a[c] = acc * rdiag[j0 + c];
            }
#pragma unroll
            for (int c = 0; c < PB; c++) s[(j0 + c) * LDS + tid] = a[c];
        }
        __syncthreads();
        // (b) rank-8 update of the trailing triangle: A[i][l] -= sum_p L[i][j0+p] L[l][j0+p]
        if (ri >= j0 + PB) {
            double li[PB];
#pragma unroll
            for (int p = 0; p < PB; p++) li[p] = s[(j0 + p) * LDS + ri];
            // two columns per iteration: two independent FMA chains (the 8-deep dependent chain was
            // latency-bound, and potrf_inv is the serial panel chain)
            int l = j0 + PB + lg;
            for (; l + PT / NB <= ri; l += 2 * (PT / NB)) {
                const int l2 = l + PT / NB;
                double acc = s[l * LDS + ri], acc2 = s[l2 * LDS + ri];
#pragma unroll
                for (int p = 0; p < PB; p++) {
                    acc = fma(-li[p], s[(j0 + p) * LDS + l], acc);
                    acc2 = fma(-li[p], s[(j0 + p) * LDS + l2], acc2);
                }
                s[l * LDS + ri] = acc;
                s[l2 * LDS + ri] = acc2;
            }
            for (; l <= ri; l += PT / NB) {
                double acc = s[l * LDS + ri];
#pragma unroll
                for (int p = 0; p < PB; p++) acc = fma(-li[p], s[(j0 + p) * LDS + l], acc);
                s[l * LDS + ri] = acc;
            }
        }
        __syncthreads();
    }

    // write L_kk back (clean upper triangle), per-block logdet share and info
    for (int idx = tid; idx < NB * NB; idx += PT) {
        int r = idx % NB, c = idx / NB;
        Akk[(int64_t)c * ld + r] = s[c * LDS + r];
    }
    // multi-GPU: a contiguous copy of L_kk rides along with the panel broadcast
    if (ldiag != nullptr) {
        double* ld_out = ldiag + k * (int64_t)NB * NB;
        for (int idx = tid; idx < NB * NB; idx += PT) ld_out[idx] = s[(idx / NB) * LDS + (idx % NB)];
    }
    if (tid < 32) {
        double acc = 0.0;
        for (int j = tid; j < NB; j += 32) acc += log(s[j * LDS + j]);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
        if (tid == 0) {
            logdet_blk[k] = 2.0 * acc;
            if (*bad != 0) {
                long long v = (long long)(k * NB + *bad);
                long long old = *info;  // keep the FIRST failing pivot (smallest index); 0 = ok so far
                if (old == 0 || v < old) *info = v;
            }
        }
    }

    // ================= blocked inverse of the lower triangle (in place) =================
    // (1) inverses of the 16 diagonal 8x8 triangles, one thread each
    if (tid < NPB) {
        const int j0 = tid * PB;
        double d[PB][PB], x[PB][PB];
#pragma unroll
        for (int c = 0; c < PB; c++)
#pragma unroll
            for (int r = 0; r < PB; r++) d[r][c] = (r >= c) ? s[(j0 + c) * LDS + j0 + r] : 0.0;
#pragma unroll
        for (int c = 0; c < PB; c++) {          // column c of the inverse: L x = e_c
#pragma unroll
            for (int r = 0; r < PB; r++) {
                if (r < c) { x[r][c] = 0.0; continue; }
                double acc = (r == c) ? 1.0 : 0.0;
#pragma unroll
                for (int p = 0; p < r; p++)
                    if (p >= c) acc -= d[r][p] * x[p][c];
                x[r][c] = acc * rdiag[j0 + r];
            }
        }
#pragma unroll
        for (int c = 0; c < PB; c++)
#pragma unroll
            for (int r = 0; r < PB; r++) dinv[tid * PB * PB + c * PB + r] = x[r][c];
    }
    __syncthreads();
    // (2) block columns right to left:  X[below, jb] = -X[below, below] * L[below, jb] * Dinv_jb
    //     thread (row i, q): columns 2q, 2q+1 of the 8-wide block
    const int q = tid / NB;
    for (int jb = NPB - 1; jb >= 0; jb--) {
        const int j0 = jb * PB;
        // Y[i][c] = sum_{p = j0+8 .. i} X[i][p] * L[p][j0+c]
        double y0 = 0.0, y1 = 0.0;
        if (ri >= j0 + PB) {
            const double* t0 = s + (j0 + 2 * q) * LDS;
            const double* t1 = t0 + LDS;
            double y0b = 0.0, y1b = 0.0;   // four independent chains instead of two
            int p = j0 + PB;
#pragma unroll 2
            for (; p + 1 <= ri; p += 2) {
                const double xv = s[p * LDS + ri], xw = s[(p + 1) * LDS + ri];
                y0 = fma(xv, t0[p], y0);
                y1 = fma(xv, t1[p], y1);
                y0b = fma(xw, t0[p + 1], y0b);
                y1b = fma(xw, t1[p + 1], y1b);
            }
            if (p <= ri) {
                const double xv = s[p * LDS + ri];
                y0 = fma(xv, t0[p], y0);
                y1 = fma(xv, t1[p], y1);
            }
            y0 += y0b;
            y1 += y1b;
            ybuf[(2 * q) * NB + ri] = y0;
            ybuf[(2 * q + 1) * NB + ri] = y1;
        }
        __syncthreads();  // all reads of the original L[:, jb] are done
        // X[i][j0+c] = -sum_{p >= c} Y[i][p] * Dinv[p][c]   (Dinv lower triangular)
        const double* di = dinv + jb * PB * PB;
        if (ri >= j0 + PB) {
            double z0 = 0.0, z1 = 0.0;
#pragma unroll
            for (int p = 0; p < PB; p++) {
                double yv = ybuf[p * NB + ri];
                z0 = fma(yv, di[(2 * q) * PB + p], z0);       // Dinv[p][2q] stored col-major: [c*PB + r]
                z1 = fma(yv, di[(2 * q + 1) * PB + p], z1);
            }
            s[(j0 + 2 * q) * LDS + ri] = -z0;
            s[(j0 + 2 * q + 1) * LDS + ri] = -z1;
        } else if (ri >= j0 && ri < j0 + PB) {
            // diagonal 8x8 block of the inverse
            int r = ri - j0;
            s[(j0 + 2 * q) * LDS + ri] = (r >= 2 * q) ? di[(2 * q) * PB + r] : 0.0;
            s[(j0 + 2 * q + 1) * LDS + ri] = (r >= 2 * q + 1) ? di[(2 * q + 1) * PB + r] : 0.0;
        }
        __syncthreads();
    }
    double* out = invL + k * (int64_t)NB * NB;
    for (int idx = tid; idx < NB * NB; idx += PT) {
        int r = idx % NB, c = idx / NB;
        out[idx] = (r >= c) ? s[c * LDS + r] : 0.0;
    }
}

bool g_attr = false;

}  // namespace

void launch_potrf_inv(Packed A, int64_t k, int64_t N, double* invL, double* logdet_blk,
                      long long* info, cudaStream_t st, double* ldiag, const double* src, int64_t ld_src) {
    if (!g_attr) {
        cudaFuncSetAttribute(potrf_inv_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                             (int)POTRF_SMEM);
        g_attr = true;
    }
    potrf_inv_kernel<<<1, PT, POTRF_SMEM, st>>>(A, k, N, invL, logdet_blk, info, ldiag, src, ld_src);
    g_launch_count++;
}

}  // namespace sb
