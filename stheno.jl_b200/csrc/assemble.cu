// K1: block-structured covariance assembly.
//
// Replaces, in one pass per (row-block, col-block) of the BlockData grid, everything the
// reference does between `cov(f::GPPP, x)` and the dense matrix handed to `cholesky`:
//   KernelFunctions.kernelmatrix (pairwise distance + kappa map; SURVEY.md App. A),
//   the scale/sum broadcasts of src/affine_transformations/{addition,product}.jl,
//   the two mortar->Array copies of src/affine_transformations/cross.jl:59-62,
//   and `cov(f, x) + Sigma_y` of AbstractGPs.
// HBM-write bound: each element is produced once, in registers, and stored once with
// 16-byte vector stores (64 consecutive rows x 16 B = 1 KB contiguous per warp per column).
#include "sb_common.cuh"

namespace sb {

thread_local int64_t g_launch_count = 0;

namespace {

constexpr int TR = 128;  // tile rows   (2 per thread x 64 thread-rows)
constexpr int TC = 32;   // tile cols   (8 per thread x 4 thread-cols)

// Julia's max(d, 0): a NaN distance (NaN input) stays NaN, where fmax would return 0 and make a NaN input
// look like a coincident point.
__device__ __forceinline__ double clamp0(double d) { return d < 0.0 ? 0.0 : d; }

// Distances.jl SqEuclidean pairwise: max(|x|^2 + |y|^2 - 2 x.y, 0).  For dim == 1 every
// operation is a single correctly-rounded IEEE op in the reference's order (no FMA
// contraction), so the result is bit-identical to the CPU path.
__device__ __forceinline__ double sqdist_gemm_trick(const double* __restrict__ x,
                                                    const double* __restrict__ y, int dim) {
    if (dim == 1) {
        double a = x[0], b = y[0];
        double s = __dadd_rn(__dmul_rn(a, a), __dmul_rn(b, b));
        return clamp0(__dsub_rn(s, __dmul_rn(2.0, __dmul_rn(a, b))));
    }
    double sa = 0.0, sb_ = 0.0, dot = 0.0;
    for (int d = 0; d < dim; d++) {
        sa = __dadd_rn(sa, __dmul_rn(x[d], x[d]));
        sb_ = __dadd_rn(sb_, __dmul_rn(y[d], y[d]));
        dot = fma(x[d], y[d], dot);
    }
    return clamp0(__dsub_rn(__dadd_rn(sa, sb_), __dmul_rn(2.0, dot)));
}

// Distances.colwise(SqEuclidean): direct differences (kernelmatrix_diag path).
__device__ __forceinline__ double sqdist_direct(const double* __restrict__ x,
                                                const double* __restrict__ y, int dim) {
    double s = 0.0;
    for (int d = 0; d < dim; d++) {
        double t = __dsub_rn(x[d], y[d]);
        s = __dadd_rn(s, __dmul_rn(t, t));
    }
    return s;
}

__device__ __forceinline__ bool all_equal(const double* __restrict__ x,
                                          const double* __restrict__ y, int dim) {
    bool eq = true;
    for (int d = 0; d < dim; d++) eq = eq && (x[d] == y[d]);
    return eq;
}

__device__ __forceinline__ double kappa(int kernel, double d2, double param) {
    switch (kernel) {
        case SB_K_SE:
            return exp(-0.5 * d2);
        case SB_K_MATERN12:
            return exp(-sqrt(d2));
        case SB_K_MATERN32: {
            double s = 1.7320508075688772 * sqrt(d2);
            return (1.0 + s) * exp(-s);
        }
        case SB_K_MATERN52: {
            double d = sqrt(d2);
            double s = 2.23606797749979 * d;
            return (1.0 + s + 5.0 * d * d / 3.0) * exp(-s);
        }
        case SB_K_CONST:
            return param;
        default:
            return 0.0;
    }
}

template <bool GEMM_TRICK>
__device__ __forceinline__ double eval_term(const TermDev& t, int64_t li, int64_t lj) {
    const double* x = t.zl + li * t.dim;
    const double* y = t.zr + lj * t.dim;
    double k;
    if (t.kernel == SB_K_WHITE) {
        k = all_equal(x, y, t.dim) ? 1.0 : 0.0;
    } else if (t.kernel == SB_K_CONST) {
        k = t.param;
    } else {
        double d2 = GEMM_TRICK ? sqdist_gemm_trick(x, y, t.dim) : sqdist_direct(x, y, t.dim);
        k = kappa(t.kernel, d2, t.param);
    }
    double s = t.coeff;
    if (t.sl) s *= t.sl[li];
    if (t.sr) s *= t.sr[lj];
    return s * k;
}

__device__ __forceinline__ int64_t clampi(int64_t v, int64_t lo, int64_t hi) {
    return v < lo ? lo : (v > hi ? hi : v);
}

// kappa for one (row pair) x (8 columns) strip of a 1-D term; KERNEL is uniform per term so the
// dispatch happens once per term, not per element
template <int KERNEL>
__device__ __forceinline__ void strip_1d(const TermDev& t, double xa, double xb, double sa, double sb_,
                                         const double* __restrict__ zr, const double* __restrict__ sr,
                                         const int64_t (&lj)[8], double (&v)[8][2]) {
    const double xa2 = __dmul_rn(xa, xa), xb2 = __dmul_rn(xb, xb);
#pragma unroll
    for (int j = 0; j < 8; j++) {
        const double y = zr[lj[j]];
        const double scol = sr ? sr[lj[j]] : 1.0;
        double ka, kb;
        if (KERNEL == SB_K_WHITE) {
            ka = (xa == y) ? 1.0 : 0.0;
            kb = (xb == y) ? 1.0 : 0.0;
        } else if (KERNEL == SB_K_CONST) {
            ka = kb = t.param;
        } else {
            // Distances.jl GEMM-trick rounding sequence, op for op (no FMA contraction)
            const double y2 = __dmul_rn(y, y);
            const double da = clamp0(__dsub_rn(__dadd_rn(xa2, y2), __dmul_rn(2.0, __dmul_rn(xa, y))));
            const double db = clamp0(__dsub_rn(__dadd_rn(xb2, y2), __dmul_rn(2.0, __dmul_rn(xb, y))));
            ka = kappa(KERNEL, da, t.param);
            kb = kappa(KERNEL, db, t.param);
        }
        v[j][0] = fma(sa * scol, ka, v[j][0]);
        v[j][1] = fma(sb_ * scol, kb, v[j][1]);
    }
}

// PACKED = true : write into the packed-lower matrix (skip tiles above the block diagonal,
//                 add noise on the diagonal).
// PACKED = false: write into a dense column-major matrix.
// ALL1D: every term has 1-D inputs (the common case): clamped, branch-free loads and one kernel
//        dispatch per term; otherwise the generic per-element path.
template <bool PACKED, bool ALL1D>
__global__ void __launch_bounds__(256)
assemble_kernel(const __grid_constant__ BlockDev b, OutDense dense, Packed packed, int64_t N, double sigma2,
                const double* __restrict__ noise_diag, int rank, int world) {
    const int64_t r_tile0 = (b.row0 / TR) * TR + (int64_t)blockIdx.x * TR;
    const int64_t c_tile0 = (b.col0 / TC) * TC + (int64_t)blockIdx.y * TC;
    if (PACKED) {
        // tile lies in NB-block (I, J); nothing above the block diagonal is stored
        if (r_tile0 / NB < c_tile0 / NB) return;
        // multi-GPU: a rank generates exactly the block columns it owns under the Cholesky
        // distribution (1-D block-cyclic); foreign columns arrive later as broadcast panels
        if (world > 1 && (int)((c_tile0 / NB) % world) != rank) return;
    }
    const int tr = threadIdx.x & 63, tc = threadIdx.x >> 6;
    const int64_t r0 = r_tile0 + 2 * tr;
    const int64_t c0 = c_tile0 + 8 * tc;
    const int64_t rend = b.row0 + b.nrows, cend = b.col0 + b.ncols;

    double v[8][2];
#pragma unroll
    for (int j = 0; j < 8; j++) v[j][0] = v[j][1] = 0.0;

    if (ALL1D) {
        const int64_t la = clampi(r0 - b.row0, 0, b.nrows - 1), lb = clampi(r0 + 1 - b.row0, 0, b.nrows - 1);
        int64_t lj[8];
#pragma unroll
        for (int j = 0; j < 8; j++) lj[j] = clampi(c0 + j - b.col0, 0, b.ncols - 1);
        for (int ti = 0; ti < b.nterms; ti++) {
            const TermDev& t = b.t[ti];
            const double xa = t.zl[la], xb = t.zl[lb];
            const double sa = t.sl ? t.coeff * t.sl[la] : t.coeff;
            const double sb_ = t.sl ? t.coeff * t.sl[lb] : t.coeff;
            switch (t.kernel) {
                case SB_K_SE: strip_1d<SB_K_SE>(t, xa, xb, sa, sb_, t.zr, t.sr, lj, v); break;
                case SB_K_MATERN12: strip_1d<SB_K_MATERN12>(t, xa, xb, sa, sb_, t.zr, t.sr, lj, v); break;
                case SB_K_MATERN32: strip_1d<SB_K_MATERN32>(t, xa, xb, sa, sb_, t.zr, t.sr, lj, v); break;
                case SB_K_MATERN52: strip_1d<SB_K_MATERN52>(t, xa, xb, sa, sb_, t.zr, t.sr, lj, v); break;
                case SB_K_WHITE: strip_1d<SB_K_WHITE>(t, xa, xb, sa, sb_, t.zr, t.sr, lj, v); break;
                default: strip_1d<SB_K_CONST>(t, xa, xb, sa, sb_, t.zr, t.sr, lj, v); break;
            }
        }
    } else {
        for (int ti = 0; ti < b.nterms; ti++) {
            const TermDev& t = b.t[ti];
#pragma unroll
            for (int j = 0; j < 8; j++) {
                int64_t c = c0 + j;
                if (c < b.col0 || c >= cend) continue;
#pragma unroll
                for (int i = 0; i < 2; i++) {
                    int64_t r = r0 + i;
                    if (r < b.row0 || r >= rend) continue;
                    v[j][i] += eval_term<true>(t, r - b.row0, c - b.col0);
                }
            }
        }
    }

#pragma unroll
    for (int j = 0; j < 8; j++) {
        int64_t c = c0 + j;
        if (c < b.col0 || c >= cend) continue;
        double* dst;
        if (PACKED) {
            dst = packed.at(r0, c);
        } else {
            dst = dense.p + c * dense.ld + r0;
        }
        bool in0 = (r0 >= b.row0 && r0 < rend), in1 = (r0 + 1 >= b.row0 && r0 + 1 < rend);
        double a0 = v[j][0], a1 = v[j][1];
        if (PACKED && !b.accumulate) {
            if (r0 == c) a0 += noise_diag ? noise_diag[c] : sigma2;
            if (r0 + 1 == c) a1 += noise_diag ? noise_diag[c] : sigma2;
        }
        if (b.accumulate) {
            if (in0) dst[0] += a0;
            if (in1) dst[1] += a1;
        } else if (in0 && in1 && ((reinterpret_cast<uintptr_t>(dst) & 15) == 0)) {
            *reinterpret_cast<double2*>(dst) = make_double2(a0, a1);
        } else {
            if (in0) dst[0] = a0;
            if (in1) dst[1] = a1;
        }
    }
}

// rows/cols >= N of the padded packed matrix: identity (L = I there, log-pivot 0).
__global__ void fill_padding_kernel(Packed A, int64_t N) {
    int64_t Np = A.Np;
    int64_t npad = Np - N;
    if (npad == 0) return;
    // every column c, padded rows r in [N, Np)
    int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int64_t c = idx / npad, r = N + idx % npad;
    if (c >= Np) return;
    if (r / NB < c / NB) return;
    *A.at(r, c) = (r == c) ? 1.0 : 0.0;
}

__global__ void assemble_diag_kernel(BlockDev b, double* __restrict__ out) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= b.nrows) return;
    double v = 0.0;
    for (int ti = 0; ti < b.nterms; ti++) v += eval_term<false>(b.t[ti], i, i);
    if (b.accumulate)
        out[b.row0 + i] += v;
    else
        out[b.row0 + i] = v;
}

// d kappa / d log(s) for inputs z = s x (stationary kernels; d = |z_i - z_j|): the lengthscale
// derivative every example optimises (examples/getting_started/script.jl:154-213)
__device__ __forceinline__ void kappa_and_dlogs(int kernel, double d2, double param, double& k, double& dk) {
    switch (kernel) {
        case SB_K_SE: k = exp(-0.5 * d2); dk = -d2 * k; break;
        case SB_K_MATERN12: { double d = sqrt(d2); k = exp(-d); dk = -d * k; break; }
        case SB_K_MATERN32: { double s = 1.7320508075688772 * sqrt(d2); double e = exp(-s); k = (1.0 + s) * e; dk = -s * s * e; break; }
        case SB_K_MATERN52: {
            double s = 2.23606797749979 * sqrt(d2);
            double e = exp(-s);
            k = (1.0 + s + s * s / 3.0) * e;
            dk = -(s * s / 3.0) * (1.0 + s) * e;
            break;
        }
        case SB_K_CONST: k = param; dk = 0.0; break;
        default: k = 0.0; dk = 0.0; break;
    }
}

// weight Q_rc of the logpdf gradient: (alpha_r alpha_c - Kinv_rc) / 2
struct LogpdfWeight {
    const double* __restrict__ alpha;
    const double* __restrict__ Kinv;
    int64_t ld;
    __device__ __forceinline__ double row(int64_t r) const { return alpha[r]; }
    __device__ __forceinline__ double operator()(double ar, int64_t r, int64_t c) const {
        return 0.5 * (ar * alpha[c] - Kinv[c * ld + r]);
    }
};

// weight Q_rc = a u_r v_c + b G_rc of the elbo gradient (G dense column-major, ld)
struct OuterPlusDense {
    double a;
    const double* __restrict__ u;
    const double* __restrict__ v;
    double b;
    const double* __restrict__ G;
    int64_t ld;
    __device__ __forceinline__ double row(int64_t r) const { return a * u[r]; }
    __device__ __forceinline__ double operator()(double aur, int64_t r, int64_t c) const {
        return aur * v[c] + b * G[c * ld + r];
    }
};

template <class Weight>
__global__ void __launch_bounds__(256)
grad_reduce_kernel(const __grid_constant__ BlockDev b, const Weight wt, double w, double* __restrict__ g) {
    // tile 64 rows x 32 cols; thread: 1 row x 8 cols
    const int64_t r = b.row0 + (int64_t)blockIdx.x * 64 + (threadIdx.x & 63);
    const int64_t c0 = b.col0 + (int64_t)blockIdx.y * 32 + (threadIdx.x >> 6) * 8;
    double acc[MAX_TERMS][2];
#pragma unroll
    for (int t = 0; t < MAX_TERMS; t++) acc[t][0] = acc[t][1] = 0.0;
    if (r < b.row0 + b.nrows) {
        const double ar = wt.row(r);
        for (int j = 0; j < 8; j++) {
            const int64_t c = c0 + j;
            if (c >= b.col0 + b.ncols) break;
            const double q = wt(ar, r, c);
            for (int ti = 0; ti < b.nterms; ti++) {
                const TermDev& t = b.t[ti];
                const double* x = t.zl + (r - b.row0) * t.dim;
                const double* y = t.zr + (c - b.col0) * t.dim;
                double k, dk;
                if (t.kernel == SB_K_WHITE) { k = all_equal(x, y, t.dim) ? 1.0 : 0.0; dk = 0.0; }
                else kappa_and_dlogs(t.kernel, sqdist_direct(x, y, t.dim), t.param, k, dk);
                double sc = q;
                if (t.sl) sc *= t.sl[r - b.row0];
                if (t.sr) sc *= t.sr[c - b.col0];
                acc[ti][0] = fma(sc, k, acc[ti][0]);
                acc[ti][1] = fma(sc * t.coeff, dk, acc[ti][1]);
            }
        }
    }
    __shared__ double red[8][MAX_TERMS][2];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int ti = 0; ti < b.nterms; ti++)
        for (int h = 0; h < 2; h++) {
            double v = acc[ti][h];
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
            if (lane == 0) red[warp][ti][h] = v;
        }
    __syncthreads();
    if (threadIdx.x < 2 * b.nterms) {
        const int ti = threadIdx.x >> 1, h = threadIdx.x & 1;
        double v = 0.0;
        for (int wdx = 0; wdx < 8; wdx++) v += red[wdx][ti][h];
        atomicAdd(&g[2 * b.tix[ti] + h], w * v);
    }
}

// the same two sums over the paired points of a diag spec: point i of the block carries the weight
// wdiag[row0 + i] (elbo: d/d K_ff[i, i] = -1 / (2 sigma_i^2))
__global__ void __launch_bounds__(256)
grad_diag_kernel(const __grid_constant__ BlockDev b, const double* __restrict__ wdiag, double* __restrict__ g) {
    const int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x;
    double acc[MAX_TERMS][2];
#pragma unroll
    for (int t = 0; t < MAX_TERMS; t++) acc[t][0] = acc[t][1] = 0.0;
    if (i < b.nrows) {
        const double q = wdiag[b.row0 + i];
        for (int ti = 0; ti < b.nterms; ti++) {
            const TermDev& t = b.t[ti];
            const double* x = t.zl + i * t.dim;
            const double* y = t.zr + i * t.dim;
            double k, dk;
            if (t.kernel == SB_K_WHITE) { k = all_equal(x, y, t.dim) ? 1.0 : 0.0; dk = 0.0; }
            else kappa_and_dlogs(t.kernel, sqdist_direct(x, y, t.dim), t.param, k, dk);
            double sc = q;
            if (t.sl) sc *= t.sl[i];
            if (t.sr) sc *= t.sr[i];
            acc[ti][0] = fma(sc, k, acc[ti][0]);
            acc[ti][1] = fma(sc * t.coeff, dk, acc[ti][1]);
        }
    }
    __shared__ double red[8][MAX_TERMS][2];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int ti = 0; ti < b.nterms; ti++)
        for (int h = 0; h < 2; h++) {
            double v = acc[ti][h];
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
            if (lane == 0) red[warp][ti][h] = v;
        }
    __syncthreads();
    if (threadIdx.x < 2 * b.nterms) {
        const int ti = threadIdx.x >> 1, h = threadIdx.x & 1;
        double v = 0.0;
        for (int wdx = 0; wdx < 8; wdx++) v += red[wdx][ti][h];
        atomicAdd(&g[2 * b.tix[ti] + h], v);
    }
}

bool all_1d(const BlockDev& b) {
    for (int t = 0; t < b.nterms; t++)
        if (b.t[t].dim != 1) return false;
    return true;
}

dim3 tile_grid(const BlockDev& b) {
    int64_t r_first = (b.row0 / TR) * TR, c_first = (b.col0 / TC) * TC;
    int64_t nrt = (b.row0 + b.nrows - r_first + TR - 1) / TR;
    int64_t nct = (b.col0 + b.ncols - c_first + TC - 1) / TC;
    return dim3((unsigned)nrt, (unsigned)nct, 1);
}

}  // namespace

void launch_assemble_dense(const BlockDev& b, OutDense out, cudaStream_t s) {
    if (b.nrows == 0 || b.ncols == 0) return;
    if (all_1d(b))
        assemble_kernel<false, true><<<tile_grid(b), 256, 0, s>>>(b, out, Packed{nullptr, 0}, 0, 0.0, nullptr, 0, 1);
    else
        assemble_kernel<false, false><<<tile_grid(b), 256, 0, s>>>(b, out, Packed{nullptr, 0}, 0, 0.0, nullptr, 0, 1);
    g_launch_count++;
}

void launch_assemble_packed(const BlockDev& b, Packed out, int64_t N, double sigma2,
                            const double* noise_diag, cudaStream_t s, int rank, int world) {
    if (b.nrows == 0 || b.ncols == 0) return;
    if (all_1d(b))
        assemble_kernel<true, true><<<tile_grid(b), 256, 0, s>>>(b, OutDense{nullptr, 0}, out, N, sigma2, noise_diag, rank, world);
    else
        assemble_kernel<true, false><<<tile_grid(b), 256, 0, s>>>(b, OutDense{nullptr, 0}, out, N, sigma2, noise_diag, rank, world);
    g_launch_count++;
}

void launch_grad_reduce(const BlockDev& b, const double* alpha, const double* Kinv, int64_t ld, double w,
                        double* g, cudaStream_t s) {
    if (b.nrows == 0 || b.ncols == 0 || b.nterms == 0) return;
    dim3 grid((unsigned)((b.nrows + 63) / 64), (unsigned)((b.ncols + 31) / 32));
    grad_reduce_kernel<<<grid, 256, 0, s>>>(b, LogpdfWeight{alpha, Kinv, ld}, w, g);
    g_launch_count++;
}

void launch_grad_reduce_outer(const BlockDev& b, double a, const double* u, const double* v, double bw,
                              const double* G, int64_t ld, double w, double* g, cudaStream_t s) {
    if (b.nrows == 0 || b.ncols == 0 || b.nterms == 0) return;
    dim3 grid((unsigned)((b.nrows + 63) / 64), (unsigned)((b.ncols + 31) / 32));
    grad_reduce_kernel<<<grid, 256, 0, s>>>(b, OuterPlusDense{a, u, v, bw, G, ld}, w, g);
    g_launch_count++;
}

void launch_grad_diag(const BlockDev& b, const double* wdiag, double* g, cudaStream_t s) {
    if (b.nrows == 0 || b.nterms == 0) return;
    grad_diag_kernel<<<(unsigned)((b.nrows + 255) / 256), 256, 0, s>>>(b, wdiag, g);
    g_launch_count++;
}

void launch_fill_padding(Packed out, int64_t N, cudaStream_t s) {
    int64_t npad = out.Np - N;
    if (npad == 0) return;
    int64_t total = npad * out.Np;
    fill_padding_kernel<<<(unsigned)((total + 255) / 256), 256, 0, s>>>(out, N);
    g_launch_count++;
}

void launch_assemble_diag(const BlockDev& b, double* out, cudaStream_t s) {
    if (b.nrows == 0) return;
    assemble_diag_kernel<<<(unsigned)((b.nrows + 255) / 256), 256, 0, s>>>(b, out);
    g_launch_count++;
}

}  // namespace sb
