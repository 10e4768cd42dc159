// K3': fp64 trailing update on the int8 tensor cores (Hopper wgmma) by integer slicing.
//
// The Ozaki scheme on the s8 kind of wgmma: every row of an operand panel is scaled by a power of two
// and cut into S = 7 signed 8-bit digits
//      x_ik  ~=  2^(e_i - 55) * sum_{p=1..7} d_p[i,k] * 2^(8(7-p)),     d_p in [-128, 127]
// (the bytes of the 56-bit two's-complement fixed-point value, re-centred so every digit is
// balanced), and   sum_k x_ik x_jk = s_i s_j * sum_{t=2..8} 2^(8(8-t)) G_t,   s = 2^(e-31),
//      G_t[i,j] = sum_{p+q=t} sum_k d_p[i,k] d_q[j,k]
// is EXACT int32 arithmetic on the tensor cores (|G_t| <= 7 * 512 * 2^14 < 2^31).  Digit pairs with
// p+q > 8 are dropped: a zero-mean truncation of ~1e-15 relative to |row_i|_max |row_j|_max, i.e.
// fp64-level.  28 int8 MMAs replace one fp64 MMA.
//
// Kernel structure (persistent CTAs, 3 warpgroups, warp-specialised), one 128 x 64 tile of C at a time:
//   warps 8-11 producer warpgroup (registers handed to the consumers with setmaxnreg); one lane is the TMA: cp.async.bulk.tensor of the digit planes of a 64-byte k-chunk of A (128
//              rows) and B (64 rows), one plane per copy, into a 2-stage shared-memory ring in the
//              SWIZZLE_64B layout wgmma reads; completion on mbarriers.
//   warps 0-7  two consumer warpgroups, rows 0-63 / 64-127 of the tile: wgmma.m64n64k32.s32.s8.s8
//              with both operands in shared memory, int32 accumulators in registers.
// The seven 64x64 int32 accumulators of a warpgroup would take 224 registers per thread, so every tile
// is computed in two passes over K: pass 0 forms G_2..G_5 (digit planes 1..4 only), pass 1 G_6..G_8 (all
// planes).  After each pass the accumulators are weighted into fp64 registers in the order t = 2..8,
// then C -= s_i s_j acc on the packed fp64 matrix.
// Replaces the dsyrk/dgemm inside LAPACK dpotrf (AbstractGPs `cholesky(Symmetric(cov(fx)))`).
#include <cuda.h>
#include <float.h>
#include <math_constants.h>

#include "sb_common.cuh"

namespace sb {
namespace {

constexpr int OZ_S = 7;              // digit planes
constexpr int OZ_BM = 128, OZ_BN = 64;
constexpr int OZ_KMAX = 512;         // bytes of K per row in the digit planes (row pitch)
constexpr int OZ_KC = 64;            // bytes of K per pipeline stage: one SWIZZLE_64B row
constexpr int OZ_STAGES = 2;
constexpr int OZ_MMA_WARPS = 8;      // two consumer warpgroups
constexpr int OZ_THREADS = OZ_MMA_WARPS * 32 + 128;   // + one producer warpgroup (setmaxnreg works per warpgroup)
constexpr int OZ_PRODUCER_REGS = 40, OZ_CONSUMER_REGS = 232;   // 128 x 40 + 256 x 232 <= 64K registers
constexpr int OZ_A_PLANE = OZ_BM * OZ_KC;                        // 8 KB
constexpr int OZ_B_PLANE = OZ_BN * OZ_KC;                        // 4 KB
constexpr int OZ_A_STAGE = OZ_S * OZ_A_PLANE;
constexpr int OZ_STAGE_BYTES = OZ_S * (OZ_A_PLANE + OZ_B_PLANE);  // 84 KB
constexpr size_t OZ_SMEM = (size_t)OZ_STAGES * OZ_STAGE_BYTES + 1024 /*align*/ + 64 /*barriers*/;
constexpr int OZ_PASS0_GROUPS = 4;   // pass 0: G_2..G_5 from planes 1..4; pass 1: G_6..G_8 from all 7

struct OzArgs {
    int mode;         // 1: packed SYRK (A == B == the panel), 0: plain  C[M x Ncols] -= A B^T, dense C
    Packed Pk;
    int64_t J0, w;    // packed: first owned trailing block column, column stride (world)
    int64_t total_tiles;
    int64_t tile_lo, tile_hi;   // this launch covers tiles [tile_lo, tile_hi) of the list (a trailing update can be split)
    int tri;             // plain mode: B is block lower triangular (128-blocks): column block q only needs K <= 128 (q + 1)
    int tiles_per_cta;   // always 0 (persistent CTAs); read by the tile loop, see oz_t_begin
    int kchunks;      // K / OZ_KC
    const double* scaleA;  // row scales s_i = 2^(e_i - 31), indexed by plane row of A / B
    const double* scaleB;
    // plain mode: tile (rt, ct) = (t % mtiles, t / mtiles); plane rows rowA0 + 128 rt, rowB0 + 64 ct
    double* C;
    int64_t ldc, mtiles;
    int64_t rowA0, rowB0;
    // plain mode C addressing: tile (rt, ct) starts at C + rt*c_rt_stride + (ct/2)*c_pair_stride + (ct%2)*64*ldc
    int64_t c_rt_stride, c_pair_stride;
    // store instance (panel solve): C = + s_i s_j acc, no read, and column block q = ct / 2 of C has its
    // own base / leading dimension (the packed matrix's block columns)
    double* cb[4];
    int64_t cld[4];
};

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, int count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
// Spin with a watchdog: a protocol bug must trap (error returned to the caller), never hang the device.
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    uint32_t ok = 0;
    long long t0 = 0;
    for (uint32_t it = 0;; it++) {
        asm volatile(
            "{\n .reg .pred p;\n mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n selp.u32 %0, 1, 0, p;\n}"
            : "=r"(ok)
            : "r"(bar), "r"(parity)
            : "memory");
        if (ok) return;
        if ((it & 0xfff) == 0xfff) {
            long long now = clock64();
            if (t0 == 0) t0 = now;
            else if (now - t0 > 20000000000LL) __trap();  // ~10 s
        }
    }
}

__device__ __forceinline__ void tma_load_3d(uint32_t dst, const CUtensorMap* tm, int c0, int c1, int c2, uint32_t bar) {
    asm volatile(
        "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];"
        ::"r"(dst), "l"(tm), "r"(c0), "r"(c1), "r"(c2), "r"(bar)
        : "memory");
}

// wgmma shared-memory matrix descriptor of a K-major SWIZZLE_64B operand (the layout the TMA box writes):
// start address >> 4 at [0,14), leading byte offset (unused when swizzled: 1) at [16,30), stride byte
// offset 512 B (8 rows x 64 B) >> 4 at [32,46), layout type 2 = 64B swizzle at [62,64)
__device__ __forceinline__ uint64_t wg_desc(uint32_t saddr) {
    return (uint64_t)((saddr >> 4) & 0x3fff) | ((uint64_t)1 << 16) | ((uint64_t)32 << 32) | ((uint64_t)2 << 62);
}

__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }

// d[64 x 64] += A[64 x 32 B] * B[64 x 32 B]^T, int8 x int8 -> int32, one warpgroup
__device__ __forceinline__ void wgmma_s8(int (&d)[32], uint64_t da, uint64_t db) {
    asm volatile(
        "wgmma.mma_async.sync.aligned.m64n64k32.s32.s8.s8 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, 1;"
        : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]),
          "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]),
          "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]),
          "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31])
        : "l"(da), "l"(db)
        : "memory");
}

// Tile range of this CTA: persistent CTAs, tile t = tile_lo + blockIdx.x + i*gridDim.x.  The tiles_per_cta branch
// (CTA b owns tiles [b*tpc, (b+1)*tpc)) is never taken, but without it nvcc 12.9 schedules the consumer epilogue
// of ozaki_syrk_kernel<false> differently, which measured 0.6% slower on an H100 80GB at 400 W.  Remove it together
// with the K3' retune (DESIGN.md §8), which reschedules this kernel anyway.
__device__ __forceinline__ int64_t oz_t_begin(const OzArgs& g) {
    return g.tile_lo + (g.tiles_per_cta > 0 ? (int64_t)blockIdx.x * g.tiles_per_cta : (int64_t)blockIdx.x);
}
__device__ __forceinline__ int64_t oz_t_end(const OzArgs& g) {
    if (g.tiles_per_cta <= 0) return g.tile_hi;
    const int64_t e = g.tile_lo + ((int64_t)blockIdx.x + 1) * g.tiles_per_cta;
    return e < g.tile_hi ? e : g.tile_hi;
}
__device__ __forceinline__ int64_t oz_t_step(const OzArgs& g) { return g.tiles_per_cta > 0 ? 1 : (int64_t)gridDim.x; }

// K chunks of tile t: all of K, or -- triangular B -- only the blocks up to the tile's column block
__device__ __forceinline__ int oz_tile_kchunks(const OzArgs& g, int64_t t) {
    if (!g.tri) return g.kchunks;
    const int64_t ct = t / g.mtiles;
    return (int)((ct >> 1) + 1) * (NB / OZ_KC);
}

struct OzTile {
    int rowA, rowB;    // first plane row of the A (128 rows) / B (64 rows) operand
    double* C;         // top-left element of the 128 x 64 output tile
    int64_t ldc;
};

// same enumeration as gemm_nt.cu's packed-SYRK cursor: owned block columns J0, J0+w, ...; column J
// holds nblk-J row blocks, two 64-wide half tiles per block
struct OzCursor {
    int64_t t, J, s0;
    __device__ __forceinline__ void init(const OzArgs& g, int64_t t0) {
        t = t0; J = g.J0; s0 = 0;
        seek(g);
    }
    __device__ __forceinline__ void seek(const OzArgs& g) {
        if (g.mode != 1) return;
        const int64_t nblk = g.Pk.nblk();
        while (t < g.total_tiles && t - s0 >= 2 * (nblk - J)) {
            s0 += 2 * (nblk - J);
            J += g.w;
        }
    }
    __device__ __forceinline__ void advance(const OzArgs& g, int64_t step) {
        t += step;
        seek(g);
    }
    __device__ __forceinline__ OzTile tile(const OzArgs& g) const {
        OzTile o;
        if (g.mode == 1) {
            const int64_t loc = t - s0;
            const int64_t I = J + (loc >> 1);
            const int h = (int)(loc & 1);
            o.rowA = (int)(I * NB);
            o.rowB = (int)(J * NB + h * OZ_BN);
            o.ldc = g.Pk.ld(J);
            o.C = g.Pk.blk(I, J) + (int64_t)(h * OZ_BN) * o.ldc;
        } else {
            const int64_t rt = t % g.mtiles, ct = t / g.mtiles;
            o.rowA = (int)(g.rowA0 + rt * OZ_BM);
            o.rowB = (int)(g.rowB0 + ct * OZ_BN);
            o.ldc = g.ldc;
            o.C = g.C + (ct >> 1) * g.c_pair_stride + (ct & 1) * OZ_BN * g.ldc + rt * g.c_rt_stride;
        }
        return o;
    }
};

// One pass of a consumer warpgroup over the K chunks of a tile: the groups G_{2+G0} .. G_{1+G1} of its
// 64 x 64 quarter (digit planes 0 .. G1-1 of both operands), then acc += 2^(8(6-grp)) G_{grp+2} in group order.
template <int G0, int G1>
__device__ __forceinline__ void oz_pass(double (&acc)[32], int kch, uint32_t& n, uint32_t base, uint32_t full0,
                                        uint32_t empty0, int wg, int lane) {
    int d[G1 - G0][32];
#pragma unroll
    for (int i = 0; i < G1 - G0; i++)
#pragma unroll
        for (int c = 0; c < 32; c++) d[i][c] = 0;
    for (int kc = 0; kc < kch; kc++, n++) {
        const uint32_t st = n % OZ_STAGES, ph = (n / OZ_STAGES) & 1;
        mbar_wait(full0 + 8 * st, ph);
        const uint32_t sA = base + st * OZ_STAGE_BYTES + (uint32_t)wg * (64 * OZ_KC), sB = base + st * OZ_STAGE_BYTES + OZ_A_STAGE;
        wg_fence();
#pragma unroll
        for (int kk = 0; kk < OZ_KC / 32; kk++) {
#pragma unroll
            for (int grp = G0; grp < G1; grp++) {
#pragma unroll
                for (int p = 0; p <= grp; p++) {   // digit planes p (of A) and q = grp - p (of B)
                    const int q = grp - p;
                    wgmma_s8(d[grp - G0], wg_desc(sA + p * OZ_A_PLANE + kk * 32), wg_desc(sB + q * OZ_B_PLANE + kk * 32));
                }
            }
        }
        wg_commit();
        wg_wait_all();
        __syncwarp();
        if (lane == 0) mbar_arrive(empty0 + 8 * st);   // this warp no longer reads the stage
    }
#pragma unroll
    for (int grp = G0; grp < G1; grp++) {
        const double wt = (double)(1ull << (8 * (OZ_S - 1 - grp)));   // 2^(8(8 - t)), t = grp + 2
#pragma unroll
        for (int c = 0; c < 32; c++) acc[c] = fma((double)d[grp - G0][c], wt, acc[c]);
    }
}

template <bool STORE>
__global__ void __launch_bounds__(OZ_THREADS, 1)
ozaki_syrk_kernel(const __grid_constant__ OzArgs g, const __grid_constant__ CUtensorMap tmA,
                  const __grid_constant__ CUtensorMap tmB) {
    extern __shared__ unsigned char oz_smem_raw[];
    const uint32_t raw = smem_u32(oz_smem_raw);
    const uint32_t base = (raw + 1023u) & ~1023u;            // stage buffers: 1024-byte aligned
    const uint32_t full0 = base + OZ_STAGES * OZ_STAGE_BYTES, empty0 = full0 + 8 * OZ_STAGES;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;

    if (tid == 0) {
        for (int s = 0; s < OZ_STAGES; s++) {
            mbar_init(full0 + 8 * s, 1);
            mbar_init(empty0 + 8 * s, OZ_MMA_WARPS);
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    }
    __syncthreads();
    const int64_t t_end = oz_t_end(g), t_step = oz_t_step(g);

    if (warp >= OZ_MMA_WARPS) {
        // ===================== TMA producer =====================
        asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(OZ_PRODUCER_REGS));
        if (warp == OZ_MMA_WARPS && lane == 0) {
            OzCursor cur;
            cur.init(g, oz_t_begin(g));
            uint32_t n = 0;
            for (; cur.t < t_end; cur.advance(g, t_step)) {
                const OzTile tl = cur.tile(g);
                const int kch = oz_tile_kchunks(g, cur.t);
                for (int pass = 0; pass < 2; pass++) {
                    const int np = pass == 0 ? OZ_PASS0_GROUPS : OZ_S;   // digit planes the pass reads
                    for (int kc = 0; kc < kch; kc++, n++) {
                        const uint32_t st = n % OZ_STAGES, ph = (n / OZ_STAGES) & 1;
                        mbar_wait(empty0 + 8 * st, ph ^ 1);
                        const uint32_t fb = full0 + 8 * st;
                        mbar_expect_tx(fb, (uint32_t)np * (OZ_A_PLANE + OZ_B_PLANE));
                        const uint32_t dA = base + st * OZ_STAGE_BYTES, dB = dA + OZ_A_STAGE;
                        for (int p = 0; p < np; p++) {
                            tma_load_3d(dA + p * OZ_A_PLANE, &tmA, kc * OZ_KC, tl.rowA, p, fb);
                            tma_load_3d(dB + p * OZ_B_PLANE, &tmB, kc * OZ_KC, tl.rowB, p, fb);
                        }
                    }
                }
            }
        }
        return;
    }

    // ===================== consumer warpgroups =====================
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(OZ_CONSUMER_REGS));
    const int wg = warp >> 2, wq = warp & 3;
    // accumulator fragment of wgmma m64nN: d[j] is row 16 wq + lane/4 (+8 for j%4 >= 2), column 8 (j/4) + 2 (lane%4) + j%2
    const int row0 = wg * 64 + wq * 16 + (lane >> 2), col0 = 2 * (lane & 3);
    OzCursor cur;
    cur.init(g, oz_t_begin(g));
    uint32_t n = 0;
    for (; cur.t < t_end; cur.advance(g, t_step)) {
        const OzTile tl = cur.tile(g);
        const int kch = oz_tile_kchunks(g, cur.t);
        double acc[32];
#pragma unroll
        for (int c = 0; c < 32; c++) acc[c] = 0.0;
        oz_pass<0, OZ_PASS0_GROUPS>(acc, kch, n, base, full0, empty0, wg, lane);
        oz_pass<OZ_PASS0_GROUPS, OZ_S>(acc, kch, n, base, full0, empty0, wg, lane);
        const double si[2] = {g.scaleA[tl.rowA + row0], g.scaleA[tl.rowA + row0 + 8]};
        if constexpr (STORE) {   // panel solve X = A W^T written straight into the packed matrix: no read of C
            const int64_t rt = cur.t % g.mtiles, ct = cur.t / g.mtiles;
            const int64_t ldq = g.cld[ct >> 1];
            double* xp = g.cb[ct >> 1] + ((ct & 1) * OZ_BN) * ldq + rt * OZ_BM + row0;
#pragma unroll
            for (int j = 0; j < 32; j++) {
                const int r = (j & 2) ? 8 : 0, c = 8 * (j >> 2) + col0 + (j & 1);
                xp[(int64_t)c * ldq + r] = (si[r >> 3] * g.scaleB[tl.rowB + c]) * acc[j];
            }
        } else {
            double* cp = tl.C + row0;
            const int64_t ldc = tl.ldc;
#pragma unroll
            for (int j0 = 0; j0 < 32; j0 += 8) {
                double old[8];
#pragma unroll
                for (int j = j0; j < j0 + 8; j++) {
                    const int r = (j & 2) ? 8 : 0, c = 8 * (j >> 2) + col0 + (j & 1);
                    old[j - j0] = __ldcs(cp + (int64_t)c * ldc + r);
                }
#pragma unroll
                for (int j = j0; j < j0 + 8; j++) {
                    const int r = (j & 2) ? 8 : 0, c = 8 * (j >> 2) + col0 + (j & 1);
                    cp[(int64_t)c * ldc + r] = fma(-(si[r >> 3] * g.scaleB[tl.rowB + c]), acc[j], old[j - j0]);
                }
            }
        }
    }
}

// ---- digit planes of an operand panel ------------------------------------------------------------
// Source: up to 4 segments of 128 columns each (K = 128 * nseg), element (row block rb, column k, row r)
// of segment q at  base[q] + rb*rbs[q] + k*ld[q] + r  (column-major panels: rbs = 128, ld = ld).
// Output, for plane row i = out_row_base + rb*128 + r and byte kb = 128*q + k:
//   plane[p][i*512 + kb]  (K-major, 512-byte pitch: the 3-D tensor the TMA box walks),
//   scale[i] = 2^(e_i - 31),  expo[i] = e_i.
// x scaled by the power of two of its column (OzSrc column equilibration); the identity without it
template <bool COLSCALE>
__device__ __forceinline__ double oz_col(const OzSrc& src, int q, int k, double x) {
    if constexpr (COLSCALE) {
        const double d = src.diag[q][(int64_t)k * src.dld[q] + k];
        if (d > 0.0 && d <= DBL_MAX) x = scalbn(x, src.colsign * ilogb(d));   // exact: a power of two
    }
    return x;
}

template <bool COLSCALE>
__global__ void __launch_bounds__(512)
oz_rowscale_kernel(const OzSrc src, int64_t rb_lo, int64_t out_row_base, double* __restrict__ scale,
                   int* __restrict__ expo) {
    // one CTA per 128-row block; 512 threads = 128 rows x 4 column groups
    __shared__ double red[4][NB];
    const int64_t rb = rb_lo + blockIdx.x;
    const int r = threadIdx.x & 127, cg = threadIdx.x >> 7;
    double m = 0.0;
    for (int q = 0; q < src.nseg; q++) {
        const double* P = src.base[q] + rb * src.rbs[q] + r;
        const int64_t ld = src.ld[q];
        for (int k = cg; k < NB; k += 4) {
            const double a = fabs(oz_col<COLSCALE>(src, q, k, P[(int64_t)k * ld]));
            m = fmax(m, a);
            if (!(a <= DBL_MAX)) m = CUDART_INF;   // NaN or Inf: fmax would drop a NaN
        }
    }
    red[cg][r] = m;
    __syncthreads();
    if (cg == 0) {
        m = fmax(fmax(red[0][r], red[1][r]), fmax(red[2][r], red[3][r]));
        const int64_t i = out_row_base + rb * NB + r;
        // Rows with no entry above 1e-280 are zero rows: no digits, scale 0.  Rows with a NaN, an Inf or an entry of
        // 1e280 or more cannot be cut into digits: no digits either, but scale NaN, so every product that touches the
        // row is NaN (NaN * 0) and the pivot check reports the failure instead of factoring a zeroed row.
        const bool ok = m > 1e-280 && m < 1e280;
        const int e = ok ? ilogb(m) + 2 : 0;   // |x| * 2^-e < 0.5
        scale[i] = ok ? scalbn(1.0, e - 31) : (m >= 1e280 ? CUDART_NAN : 0.0);
        expo[i] = ok ? e : 0x7fffffff;
    }
}

template <bool COLSCALE>
__global__ void __launch_bounds__(256)
oz_slice_kernel(const OzSrc src, int64_t rb_lo, int64_t out_row_base, int64_t plane_rows,
                const int* __restrict__ expo, signed char* __restrict__ planes) {
    // grid: (row blocks, nseg * 4 column chunks of 32); 256 threads = 128 rows x 2 halves of 16 cols
    __shared__ __align__(16) signed char sd[OZ_S][NB][32];
    const int64_t rb = rb_lo + blockIdx.x;
    const int q = blockIdx.y >> 2, kc = blockIdx.y & 3;
    const int r = threadIdx.x & 127, kh = threadIdx.x >> 7;
    const int64_t row0 = out_row_base + rb * NB;
    const int e = expo[row0 + r];
    const int64_t ld = src.ld[q];
    const double* P = src.base[q] + rb * src.rbs[q] + (int64_t)(kc * 32 + kh * 16) * ld + r;
#pragma unroll 4
    for (int kk = 0; kk < 16; kk++) {
        const double x = oz_col<COLSCALE>(src, q, kc * 32 + kh * 16 + kk, P[(int64_t)kk * ld]);
        long long Z = 0x0000808080808080LL;
        if (e != 0x7fffffff) Z += __double2ll_rn(scalbn(x, 55 - e));
        const int kb = kh * 16 + kk;
        sd[0][r][kb] = (signed char)(Z >> 48);
#pragma unroll
        for (int p = 1; p < OZ_S; p++) sd[p][r][kb] = (signed char)(((Z >> (8 * (OZ_S - 1 - p))) & 0xff) ^ 0x80);
    }
    __syncthreads();
    // 7 planes x 128 rows x 32 bytes: 16-byte stores, two per row
    for (int idx = threadIdx.x; idx < OZ_S * NB * 2; idx += 256) {
        const int p = idx / (NB * 2), rr = (idx >> 1) & 127, hf = idx & 1;
        const int4 v = *reinterpret_cast<const int4*>(&sd[p][rr][hf * 16]);
        *reinterpret_cast<int4*>(planes + ((int64_t)p * plane_rows + row0 + rr) * OZ_KMAX + q * NB + kc * 32 + hf * 16) = v;
    }
}

typedef CUresult (*EncodeTiled_t)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiled_t g_encode = nullptr;
bool g_oz_attr = false;
int g_oz_sms = 0;

int oz_init() {
    if (!g_encode) {
        void* fn = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres) != cudaSuccess || !fn) return -1;
        g_encode = (EncodeTiled_t)fn;
    }
    if (!g_oz_attr) {
        if (cudaFuncSetAttribute(ozaki_syrk_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)OZ_SMEM) != cudaSuccess ||
            cudaFuncSetAttribute(ozaki_syrk_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)OZ_SMEM) != cudaSuccess)
            return -2;
        int dev = 0;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&g_oz_sms, cudaDevAttrMultiProcessorCount, dev);
        g_oz_attr = true;
    }
    return 0;
}

}  // namespace

size_t oz_planes_bytes(int64_t Np) { return (size_t)OZ_S * Np * OZ_KMAX; }

// The two tensor maps over the digit planes: one plane of a 64-byte k-chunk of 128 rows (A) / 64 rows (B)
// per copy, SWIZZLE_64B.
int oz_make_maps(signed char* planes, int64_t Np, OzMaps* out) {
    if (oz_init() != 0) return -1;
    static_assert(sizeof(out->a) >= sizeof(CUtensorMap), "OzMaps too small");
    cuuint64_t dims[3] = {(cuuint64_t)OZ_KMAX, (cuuint64_t)Np, (cuuint64_t)OZ_S};
    cuuint64_t strides[2] = {(cuuint64_t)OZ_KMAX, (cuuint64_t)Np * OZ_KMAX};
    cuuint32_t estr[3] = {1, 1, 1};
    cuuint32_t boxA[3] = {OZ_KC, OZ_BM, 1}, boxB[3] = {OZ_KC, OZ_BN, 1};
    const CUresult r1 = g_encode(reinterpret_cast<CUtensorMap*>(out->a), CU_TENSOR_MAP_DATA_TYPE_UINT8, 3, planes, dims,
                                 strides, boxA, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_64B,
                                 CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    const CUresult r2 = g_encode(reinterpret_cast<CUtensorMap*>(out->b), CU_TENSOR_MAP_DATA_TYPE_UINT8, 3, planes, dims,
                                 strides, boxB, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_64B,
                                 CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    return (r1 == CUDA_SUCCESS && r2 == CUDA_SUCCESS) ? 0 : -3;
}

// digit planes + row scales of row blocks [rb_lo, rb_lo + nrb) of the source panel
void launch_oz_slice(const OzSrc& src, int64_t rb_lo, int64_t nrb, int64_t out_row_base, int64_t plane_rows,
                     double* scale, int* expo, signed char* planes, cudaStream_t s) {
    if (nrb <= 0 || src.nseg <= 0) return;
    const dim3 grid((unsigned)nrb, (unsigned)(src.nseg * 4));
    if (src.colsign != 0) {
        oz_rowscale_kernel<true><<<(unsigned)nrb, 512, 0, s>>>(src, rb_lo, out_row_base, scale, expo);
        oz_slice_kernel<true><<<grid, 256, 0, s>>>(src, rb_lo, out_row_base, plane_rows, expo, planes);
    } else {
        oz_rowscale_kernel<false><<<(unsigned)nrb, 512, 0, s>>>(src, rb_lo, out_row_base, scale, expo);
        oz_slice_kernel<false><<<grid, 256, 0, s>>>(src, rb_lo, out_row_base, plane_rows, expo, planes);
    }
    g_launch_count += 2;
}

static int oz_launch(OzArgs& g, const OzMaps* mapsA, const OzMaps* mapsB, bool store, cudaStream_t s, int reserve_sms) {
    int64_t cap = g_oz_sms - reserve_sms;
    if (cap < 1) cap = 1;
    if (g.tile_hi <= 0 || g.tile_hi > g.total_tiles) g.tile_hi = g.total_tiles;
    if (g.tile_lo < 0) g.tile_lo = 0;
    const int64_t ntiles = g.tile_hi - g.tile_lo;
    if (ntiles <= 0) return 0;
    const int64_t grid = ntiles < cap ? ntiles : cap;
    const CUtensorMap* ma = reinterpret_cast<const CUtensorMap*>(mapsA->a);
    const CUtensorMap* mb = reinterpret_cast<const CUtensorMap*>(mapsB->b);
    if (store) ozaki_syrk_kernel<true><<<(unsigned)grid, OZ_THREADS, OZ_SMEM, s>>>(g, *ma, *mb);
    else ozaki_syrk_kernel<false><<<(unsigned)grid, OZ_THREADS, OZ_SMEM, s>>>(g, *ma, *mb);
    g_launch_count++;
    return 0;
}

// A[I, J] -= P_I P_J^T on the packed lower matrix for the owned block columns J in [jlo, jhi), with
// the digit planes / scales produced by launch_oz_slice.  K = 128 * nseg.
int launch_syrk_ozaki(Packed Apk, int64_t k, int nseg, int64_t jlo, int64_t jhi, int rank, int world,
                      const OzMaps* maps, const double* scale, cudaStream_t s, int reserve_sms, int64_t tile_lo,
                      int64_t tile_hi) {
    if (oz_init() != 0) return -1;
    const int64_t nblk = Apk.nblk();
    if (jlo < k + 1) jlo = k + 1;
    if (jhi > nblk) jhi = nblk;
    const int64_t J0 = jlo + ((rank - jlo % world) % world + world) % world;
    const int64_t tiles = syrk_packed_tiles(nblk, k, jlo, jhi, rank, world);
    if (tiles <= 0 || nseg <= 0) return 0;
    OzArgs g{};
    g.mode = 1;
    g.Pk = Apk; g.J0 = J0; g.w = world;
    g.total_tiles = tiles * 2;
    g.tile_lo = tile_lo; g.tile_hi = tile_hi;   // (0, 0): everything
    g.kchunks = nseg * NB / OZ_KC;
    g.scaleA = g.scaleB = scale;
    return oz_launch(g, maps, maps, false, s, reserve_sms);
}

// plain product  C[M x Ncols] -= A B^T  (C dense column-major, ldc; M % 128 == 0, Ncols % 64 == 0):
// A = plane rows [rowA0, rowA0 + M) of the (mapsA, scaleA) set, B = plane rows [rowB0, rowB0 + Ncols) of
// (mapsB, scaleB); K = 128 * nseg.  Used by the posterior / VFE matrix-TRSM sweeps.
int launch_gemm_ozaki(double* C, int64_t ldc, int64_t M, int64_t Ncols, int nseg, const OzMaps* mapsA,
                      const double* scaleA, int64_t rowA0, const OzMaps* mapsB, const double* scaleB, int64_t rowB0,
                      cudaStream_t s) {
    if (oz_init() != 0) return -1;
    if (M <= 0 || Ncols <= 0 || nseg <= 0) return 0;
    OzArgs g{};
    g.mode = 0;
    g.C = C; g.ldc = ldc; g.mtiles = M / OZ_BM;
    g.c_rt_stride = OZ_BM;
    g.c_pair_stride = 2 * OZ_BN * ldc;
    g.total_tiles = (M / OZ_BM) * (Ncols / OZ_BN);
    g.kchunks = nseg * NB / OZ_KC;
    g.scaleA = scaleA; g.scaleB = scaleB;
    g.rowA0 = rowA0; g.rowB0 = rowB0;
    return oz_launch(g, mapsA, mapsB, false, s, 0);
}

// Panel solve of the wide panel phase:  X[M x 512] = A W^T, W = inv(L_512) block lower triangular (K blocks above
// the diagonal are skipped), written over the four block columns Xcol[q] (leading dimensions ldx[q]) the planes of A
// were cut from.
int launch_panel_solve_ozaki(double* const* Xcol, const int64_t* ldx, int64_t M, const OzMaps* mapsA, const double* scaleA,
                             int64_t rowA0, const OzMaps* mapsW, const double* scaleW, cudaStream_t s) {
    if (oz_init() != 0) return -1;
    if (M <= 0) return 0;
    OzArgs g{};
    g.mode = 0;
    g.mtiles = M / OZ_BM;
    g.total_tiles = (M / OZ_BM) * (4 * NB / OZ_BN);
    g.kchunks = 4 * NB / OZ_KC;
    g.tri = 1;
    for (int q = 0; q < 4; q++) { g.cb[q] = Xcol[q]; g.cld[q] = ldx[q]; }
    g.C = Xcol[0]; g.ldc = ldx[0]; g.c_rt_stride = OZ_BM; g.c_pair_stride = 0;
    g.scaleA = scaleA; g.scaleB = scaleW;
    g.rowA0 = rowA0; g.rowB0 = 0;
    return oz_launch(g, mapsA, mapsW, true, s, 0);
}

}  // namespace sb
