// Appending observations to a factor (sb_factor_append): the kernels that build the joint packed factor of
// [old; new] from the old one without refactorising it.  With h = NB floor(N1 / NB) (the full old block
// columns) and r = N1 - h (the old rows of the partial last block):
//   * block columns j < h/NB of the joint factor are the old ones, rows [NB j, N1) verbatim, followed by the N2
//     rows of V = K21 L^{-T} (append_relayout_kernel);
//   * the rest is the Cholesky factor of  S = M M' + blockdiag(0_r, P),  M = [L_TT; V[:, h:N1)],
//     P = K22 + Sigma2 - V V'  (schur_pack_kernel packs S; the Cholesky driver factors it).  S starts on a
//     block boundary, so its packed storage is byte-identical to the tail of the joint packed layout.
// With r = 0, S = P: the same kernel packs the posterior covariance for sb_predict_factor.
#include "sb_common.cuh"

namespace sb {
namespace {

// Packed S (order Ns, padded to S.Np) <- M M' + blockdiag(0_r, C), every stored entry of the block-lower layout;
// rows/cols >= Ns are zero (the caller fills the padding).  M = [T; V]: T (r x r lower, ld ldt), V (Ns - r rows,
// ld ldv, r columns).  C: (Ns - r) x (Ns - r), ld ldc, lower triangle read.  One CTA column per column of S.
__global__ void __launch_bounds__(256)
schur_pack_kernel(Packed S, int64_t Ns, int r, const double* __restrict__ C, int64_t ldc,
                  const double* __restrict__ T, int64_t ldt, const double* __restrict__ V, int64_t ldv) {
    const int64_t k = blockIdx.x;
    const int64_t i = (int64_t)blockIdx.y * 256 + threadIdx.x;
    if (i >= S.Np || i / NB < k / NB) return;
    const int64_t a = i > k ? i : k, b = i > k ? k : i;  // the upper entries of a diagonal block mirror (a, b)
    double v = 0.0;
    if (a < Ns) {
        if (b >= r) v = C[(b - r) * ldc + (a - r)];
        const int cend = b < r ? (int)b + 1 : r;         // T is lower triangular
        const double* ma = a < r ? T + a : V + (a - r);
        const double* mb = b < r ? T + b : V + (b - r);
        const int64_t lda = a < r ? ldt : ldv, ldb = b < r ? ldt : ldv;
        for (int c = 0; c < cend; c++) v = fma(ma[c * lda], mb[c * ldb], v);
    }
    *S.at(i, k) = v;
}

// C (n x n, ld) += noise, lower triangle: scalar s2, diag[n], or dense[n x n] (ld n)
__global__ void __launch_bounds__(256)
add_noise_kernel(double* __restrict__ C, int64_t ld, int64_t n, double s2, const double* __restrict__ diag,
                 const double* __restrict__ dense) {
    const int64_t j = blockIdx.x;
    const int64_t i = (int64_t)blockIdx.y * 256 + threadIdx.x;
    if (i >= n || i < j) return;
    if (dense) C[j * ld + i] += dense[j * n + i];
    else if (i == j) C[j * ld + i] += diag ? diag[i] : s2;
}

// Joint block columns j < nh (one CTA per column):  rows [NB j, N1) from the old packed factor O, rows
// [N1, N1 + N2) from column NB j + c of V (ld ldv), zero below.  Every destination pair is one 16-byte store, and
// so is every source pair that does not straddle a seam or sit at an odd offset of V (V starts at joint row N1).
__global__ void __launch_bounds__(256)
append_relayout_kernel(Packed J, Packed O, int64_t N1, int64_t N2, const double* __restrict__ V, int64_t ldv) {
    const int64_t col = blockIdx.x;
    const int64_t j = col / NB, c = col - j * NB;
    const int64_t ldj = J.ld(j);
    const double* __restrict__ src = O.base + O.off(j) + c * O.ld(j);
    const double* __restrict__ vs = V + col * ldv;
    double* __restrict__ dst = J.base + J.off(j) + c * ldj;
    const int64_t t1 = N1 - j * NB, t2 = t1 + N2;          // local rows where V starts / the padding starts
    for (int64_t t = 2 * threadIdx.x; t < ldj; t += 512) {  // ldj is a multiple of NB: pairs never run past it
        double2 p;
        if (t + 1 < t1) {
            p = __ldcs(reinterpret_cast<const double2*>(src + t));
        } else if (t >= t1 && t + 1 < t2 && ((t - t1) & 1) == 0) {
            p = __ldcs(reinterpret_cast<const double2*>(vs + (t - t1)));
        } else {
            p.x = t < t1 ? src[t] : (t < t2 ? vs[t - t1] : 0.0);
            p.y = t + 1 < t1 ? src[t + 1] : (t + 1 < t2 ? vs[t + 1 - t1] : 0.0);
        }
        __stcs(reinterpret_cast<double2*>(dst + t), p);
    }
}

}  // namespace

void launch_pack_schur(Packed S, int64_t Ns, int r, const double* C, int64_t ldc, const double* T, int64_t ldt,
                       const double* V, int64_t ldv, cudaStream_t st) {
    schur_pack_kernel<<<dim3((unsigned)S.Np, (unsigned)((S.Np + 255) / 256)), 256, 0, st>>>(S, Ns, r, C, ldc, T, ldt,
                                                                                             V, ldv);
    g_launch_count++;
}

void launch_add_noise_dense(double* C, int64_t ld, int64_t n, double s2, const double* diag, const double* dense,
                            cudaStream_t st) {
    if (n <= 0 || (!dense && !diag && s2 == 0.0)) return;
    add_noise_kernel<<<dim3((unsigned)n, (unsigned)((n + 255) / 256)), 256, 0, st>>>(C, ld, n, s2, diag, dense);
    g_launch_count++;
}

void launch_append_relayout(Packed J, Packed O, int64_t N1, int64_t N2, const double* V, int64_t ldv, int64_t h,
                            cudaStream_t st) {
    if (h <= 0) return;
    append_relayout_kernel<<<(unsigned)h, 256, 0, st>>>(J, O, N1, N2, V, ldv);
    g_launch_count++;
}

}  // namespace sb
