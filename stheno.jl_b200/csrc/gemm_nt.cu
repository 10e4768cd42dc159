// K3: fp64 tensor-core NT contraction   C = beta*C + alpha * A * B^T   (all column-major).
//
// This one kernel is the whole O(N^3) of the path: the Cholesky trailing update (SYRK on the
// packed lower matrix), the panel TRSM (as a product with the explicit inverse of the
// diagonal block), the posterior matrix TRSM sweep and the posterior covariance downdate.
// It replaces LAPACK dpotrf's dsyrk/dgemm/dtrsm inside `cholesky(Symmetric(K + Sigma_y))` and
// the `C.U' \ K_fx` solves of AbstractGPs (SURVEY.md App. A).
//
// sm_90a notes.  wgmma has no fp64 kind, so fp64 tensor math is the DMMA path
// (mma.sync.m16n8k4.f64 -> SASS DMMA.16x8x4).  Operand k-slabs are staged global->shared by the
// TMA engine with 1-D bulk copies (cp.async.bulk ... mbarrier::complete_tx -> SASS UBLKCP) into a
// 4-stage ring; one mbarrier per stage.  Shared tiles are [k][row] with a 4-double pad so the
// fragment loads (8 rows x 4 k per LDS.64) are bank-conflict free.  The MMA is issued
// "transposed" (m <-> C columns, n <-> C rows) so each thread owns 2 consecutive rows of C and
// the epilogue uses 16-byte loads/stores.  CTA tile 128x64, 8 warps of 32x32, 2 CTAs per SM so
// one CTA's C read-modify-write epilogue overlaps the other's MMA main loop.  Two CTAs of 9 warps
// cap the kernel at 96 registers: each of the SM's 4 sub-partitions holds 16384 registers and
// some sub-partition gets 5 of the 18 warps (5 * 32 * 96 <= 16384 < 5 * 32 * 104).  At 112 registers
// only one CTA fits and the kernel is slower.  On H100 DMMA.8x8x4 (m8n8k4) issues at half the fp64
// tensor rate of the m16n8k{4,8,16} shapes (profiles/mb_dmma_loop_h100.txt); m16n8k4 is the one
// whose fragments fit the 96-register budget.
#include "sb_common.cuh"

namespace sb {
namespace {

constexpr int BM = 128;  // C rows per CTA
constexpr int BN = 64;   // C cols per CTA
constexpr int KC = 16;   // k-slab per pipeline stage
constexpr int STAGES = 4;
constexpr int LDA_S = BM + 4;
constexpr int LDB_S = BN + 4;
constexpr int SLAB = KC * LDA_S;           // doubles in one A k-slab image  [16][132]
constexpr int SLAB_BYTES = SLAB * 8;       // 16896
constexpr int SLAB_B = KC * LDB_S;         // B stage [16][68]
constexpr int MATH_WARPS = 8;
constexpr int THREADS = (MATH_WARPS + 1) * 32;  // + 1 TMA producer warp
constexpr size_t SMEM_BYTES = (size_t)STAGES * (SLAB + SLAB_B) * 8 + 2 * STAGES * 8 + 64;

constexpr int MAX_SEG = 4;

// Operands are K-segmented: k-chunks [seg*seg_chunks, (seg+1)*seg_chunks) of A (B) come from
// Aseg[seg] (Bseg[seg]) with leading dimension lda_seg[seg] (ldb_seg[seg]).  This is how one
// launch applies 2..4 panels at once (K = 256 / 512): each half panel / block column of L lives in
// its own buffer.  Tiled operands (see TilePtrs) ignore the leading dimensions.
struct GemmArgs {
    int mode;  // 0 plain, 1 packed SYRK
    int a_tiled, b_tiled, c_tiled;
    int seg_chunks;                 // k-chunks (of KC columns) per segment
    const double* Aseg[MAX_SEG];
    int64_t lda_seg[MAX_SEG];
    const double* Bseg[MAX_SEG];
    int64_t ldb_seg[MAX_SEG];
    double* C;
    int64_t ldc;
    int64_t mtiles;  // plain: number of row tiles
    int64_t total_tiles;
    int64_t K;
    double alpha, beta;
    // packed SYRK
    Packed Pk;
    int64_t k;      // first block column of the outer step (tiled row block 0 <-> block row k+1)
    int64_t J0;     // first owned block column >= jlo
    int64_t w;      // column stride (world)
};

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return (uint32_t)__cvta_generic_to_shared(p);
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, int count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)),
                 "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    do {
        asm volatile(
            "{\n .reg .pred p;\n mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
            " selp.u32 %0, 1, 0, p;\n}"
            : "=r"(ok)
            : "r"(smem_u32(bar)), "r"(parity)
            : "memory");
    } while (!ok);
}
// TMA 1-D bulk copy global -> shared, completion signalled on an mbarrier (SASS: UBLKCP).
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes,
                                         uint64_t* bar) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
        ::"r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar))
        : "memory");
}
// c[0..1] = C(m = gid, n = 2 tig + 0..1), c[2..3] = C(m = gid + 8, ...);
// a0 = A(m = gid, k = tig), a1 = A(m = gid + 8, k = tig), b = B(k = tig, n = gid)
__device__ __forceinline__ void dmma(double (&c)[4], double a0, double a1, double b) {
    asm volatile(
        "mma.sync.aligned.m16n8k4.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5}, {%6}, {%0,%1,%2,%3};"
        : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3])
        : "d"(a0), "d"(a1), "d"(b));
}

// TILED layout of a panel (written by the TRSM epilogue, read by the SYRK): for every 128-row
// block rb and panel column k (0..127) a padded column of 132 doubles; slab (rb, kc) = 16
// consecutive padded columns = exactly the shared-memory image [16][132] of a k-slab, so the
// TMA producer moves a whole operand slab with ONE bulk copy of 16896 bytes.
//   addr(rb, k, r) = ((rb * 128 + k) * 132 + r)
struct TilePtrs {
    double* C;
    int64_t ldc;
    int64_t a_off, b_off;  // column-major operands: row offset (elements) of this tile's rows
    int64_t a_blk, b_blk;  // tiled operands: 128-row block index
    int b_row_off;         // tiled B: 0 or 64 (which half of the 128-row block)
    int64_t c_rt;          // tiled C: row tile
    int c_ct;              // tiled C: column tile (0/1)
};

// Walks the tiles blockIdx.x, +gridDim.x, ... of one launch.  Packed SYRK tiles are enumerated
// block column by block column (columns J0, J0+w, ... ; column J holds nblk-J row blocks; two
// 64-wide half tiles per block), so advancing is a couple of integer compares -- no division,
// no square root.
struct TileCursor {
    int64_t t;     // linear tile index
    int64_t J;     // packed: current block column
    int64_t s0;    // packed: linear index of the first (half-)tile of column J
    __device__ __forceinline__ void init(const GemmArgs& g, int64_t t0) {
        t = t0;
        J = g.J0;
        s0 = 0;
        if (g.mode == 1) seek(g);
    }
    __device__ __forceinline__ void seek(const GemmArgs& g) {
        const int64_t nblk = g.Pk.nblk();
        while (t - s0 >= 2 * (nblk - J)) {
            s0 += 2 * (nblk - J);
            J += g.w;
        }
    }
    __device__ __forceinline__ void advance(const GemmArgs& g, int64_t step) {
        t += step;
        if (g.mode == 1 && t < g.total_tiles) seek(g);
    }
    __device__ __forceinline__ TilePtrs ptrs(const GemmArgs& g) const {
        TilePtrs p;
        if (g.mode == 0) {
            int64_t rt = t % g.mtiles, ct = t / g.mtiles;
            p.ldc = g.ldc;
            p.a_off = rt * BM;
            p.b_off = ct * BN;
            p.C = g.C + ct * BN * g.ldc + rt * BM;
            p.a_blk = rt; p.b_blk = ct >> 1; p.b_row_off = (int)(ct & 1) * BN;
            p.c_rt = rt; p.c_ct = (int)ct;
        } else {
            const int64_t loc = t - s0;
            const int64_t I = J + (loc >> 1);
            const int h = (int)(loc & 1);
            p.ldc = g.Pk.ld(J);
            p.C = g.Pk.blk(I, J) + (int64_t)h * BN * p.ldc;
            p.a_off = p.b_off = 0;
            p.a_blk = I - g.k - 1; p.b_blk = J - g.k - 1; p.b_row_off = h * BN;
            p.c_rt = 0; p.c_ct = 0;
        }
        return p;
    }
};

__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}

// Persistent CTAs (2 per SM): each walks tiles blockIdx.x, +gridDim.x, ...  Warp-specialised:
// warps 0..7 are math warps (LDS.64 fragments + DMMA + epilogue, no copy-issue code at all);
// warp 8 is the TMA producer: its lane 0 runs the whole refill loop (wait empty[] -> proxy fence
// -> arm full[] with the slab's byte count -> 32 bulk copies).  Issuing bulk copies from the math
// warps costs tensor-pipe issue slots: a bulk-copy issue stalls its warp.
// The ring is addressed by a chunk counter that runs ACROSS tiles, so the next tile's first
// k-slabs are already landing while the math warps are in the current tile's epilogue.  No
// CTA-wide barrier in steady state: full[] (tx-count) / empty[] (8 warp arrivals) mbarriers only.
__global__ void __launch_bounds__(THREADS, 2) gemm_nt_kernel(const __grid_constant__ GemmArgs g) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    double* sA = reinterpret_cast<double*>(smem_raw);
    double* sB = sA + STAGES * SLAB;
    uint64_t* full = reinterpret_cast<uint64_t*>(sB + STAGES * SLAB_B);
    uint64_t* empty = full + STAGES;

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int gid = lane >> 2, tig = lane & 3;
    const int nchunks = (int)(g.K / KC);

    if (tid == 0) {
#pragma unroll
        for (int s = 0; s < STAGES; s++) {
            mbar_init(&full[s], 1);
            mbar_init(&empty[s], MATH_WARPS);
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    }
    __syncthreads();

    if (warp == MATH_WARPS) {
        // ================= TMA producer warp =================
        // (SB_ABLATE_NO_TMA is a compile-time ablation used by tools/bench_gemm only -- wrong
        //  results, timing experiment: no bulk copies at all.  See DESIGN.md K3 and profiles/.
        //  The earlier "NO_WAIT" ablation (copies issued, nobody waits) belongs to the pre-
        //  warp-specialised kernel; here it would alias the empty[] parity and deadlock.)
#ifndef SB_ABLATE_NO_TMA
        if (lane == 0) {
            TileCursor pcur;
            pcur.init(g, blockIdx.x);
            int pslot = 0;
            uint32_t pphase = 0;
            bool pfirst = true;  // first pass over the ring: slots are fresh, nothing to wait for
            for (; pcur.t < g.total_tiles; pcur.advance(g, gridDim.x)) {
                const TilePtrs pp = pcur.ptrs(g);
                for (int pc = 0; pc < nchunks; pc++) {
                    if (!pfirst) {
                        mbar_wait(&empty[pslot], pphase);
                        // generic-proxy reads of the slot (math warps) -> async-proxy refill
                        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
                    }
                    const uint32_t abytes = g.a_tiled ? SLAB_BYTES : BM * KC * 8;
                    mbar_expect_tx(&full[pslot], abytes + BN * KC * 8);
                    double* dA = sA + pslot * SLAB;
                    double* dB = sB + pslot * SLAB_B;
                    const int seg = pc / g.seg_chunks, lc = pc - seg * g.seg_chunks;  // segment, chunk in it
                    if (g.a_tiled) {  // one bulk copy: the slab is stored as its shared-memory image
                        bulk_g2s(dA, g.Aseg[seg] + (pp.a_blk * 128 + lc * KC) * LDA_S, SLAB_BYTES, &full[pslot]);
                    } else {
                        const int64_t lda = g.lda_seg[seg];
                        const double* srcA = g.Aseg[seg] + pp.a_off + (int64_t)lc * KC * lda;
#pragma unroll
                        for (int kk = 0; kk < KC; kk++) bulk_g2s(dA + kk * LDA_S, srcA + kk * lda, BM * 8, &full[pslot]);
                    }
                    {   // B: 16 half-columns of 64 rows (from a column-major matrix, or strided out of
                        // the tiled panel: same bytes as needed, no over-fetch)
                        const int64_t ldb = g.b_tiled ? (int64_t)LDA_S : g.ldb_seg[seg];
                        const double* srcB = g.b_tiled
                            ? g.Bseg[seg] + (pp.b_blk * 128 + lc * KC) * LDA_S + pp.b_row_off
                            : g.Bseg[seg] + pp.b_off + (int64_t)lc * KC * ldb;
#pragma unroll
                        for (int kk = 0; kk < KC; kk++) bulk_g2s(dB + kk * LDB_S, srcB + kk * ldb, BN * 8, &full[pslot]);
                    }
                    if (++pslot == STAGES) {
                        pslot = 0;
                        if (pfirst) pfirst = false; else pphase ^= 1;
                    }
                }
            }
        }
#endif
        return;
    }

    // ================= math warps =================
    const int wr = warp & 3, wc = warp >> 2;  // 4 warps along rows, 2 along cols; 32x32 each
    const double alpha = g.alpha, beta = g.beta;
    const double* a_base = sA + wr * 32 + gid + tig * LDA_S;
    const double* b_base = sB + wc * 32 + gid + tig * LDB_S;
    int slot = 0;
    uint32_t phase = 0;
    TileCursor cur;
    cur.init(g, blockIdx.x);
    for (; cur.t < g.total_tiles; cur.advance(g, gridDim.x)) {
        // acc[jj][i][2h + e] = C(column wc*32 + (2jj + h)*8 + gid, row wr*32 + i*8 + 2tig + e)
        double acc[2][4][4];
#pragma unroll
        for (int jj = 0; jj < 2; jj++)
#pragma unroll
            for (int i = 0; i < 4; i++) acc[jj][i][0] = acc[jj][i][1] = acc[jj][i][2] = acc[jj][i][3] = 0.0;

        for (int c = 0; c < nchunks; c++) {
#ifndef SB_ABLATE_NO_TMA
            mbar_wait(&full[slot], phase);
#endif
            const double* a = a_base + slot * SLAB;
            const double* b = b_base + slot * SLAB_B;
#pragma unroll
            for (int k4 = 0; k4 < KC / 4; k4++) {
                double rf[4], cf[4];
#pragma unroll
                for (int i = 0; i < 4; i++) rf[i] = a[k4 * 4 * LDA_S + i * 8];
#pragma unroll
                for (int j = 0; j < 4; j++) cf[j] = b[k4 * 4 * LDB_S + j * 8];
#pragma unroll
                for (int jj = 0; jj < 2; jj++)
#pragma unroll
                    for (int i = 0; i < 4; i++) dmma(acc[jj][i], cf[2 * jj], cf[2 * jj + 1], rf[i]);
            }
            __syncwarp();
#ifndef SB_ABLATE_NO_TMA
            if (lane == 0) mbar_arrive(&empty[slot]);
#endif
            if (++slot == STAGES) { slot = 0; phase ^= 1; }
        }

        // (the tile's C pointers are formed only now: held across the main loop they cost registers)
        const TilePtrs tp = cur.ptrs(g);
        // epilogue: thread owns rows (2*tig, 2*tig+1) of column gid in each 8x8 quarter of a fragment
        // tiled output (TRSM -> panel in slab-image layout): column k of row tile rt is the padded
        // 132-double column ((rt*128 + k) * 132); this tile covers k = ct*64 .. ct*64+63
        double* cbase = g.c_tiled
            ? g.C + ((tp.c_rt * 128 + tp.c_ct * BN + wc * 32 + gid) * (int64_t)LDA_S) + wr * 32 + 2 * tig
            : tp.C + (int64_t)(wc * 32 + gid) * tp.ldc + wr * 32 + 2 * tig;
        const int64_t ldc = g.c_tiled ? (int64_t)LDA_S : tp.ldc;
        if (beta != 0.0) {
#pragma unroll
            for (int jh = 0; jh < 2; jh++) {  // 8 x 16-byte loads in flight per thread
                double2 old[2][4];
#pragma unroll
                for (int jj = 0; jj < 2; jj++)
#pragma unroll
                    for (int i = 0; i < 4; i++)
                        old[jj][i] = __ldcs(reinterpret_cast<const double2*>(
                            cbase + (int64_t)(jh * 2 + jj) * 8 * ldc + i * 8));
#pragma unroll
                for (int jj = 0; jj < 2; jj++)
#pragma unroll
                    for (int i = 0; i < 4; i++) {
                        const int j = jh * 2 + jj;
                        double2 o;
                        o.x = fma(alpha, acc[jh][i][2 * jj], beta * old[jj][i].x);
                        o.y = fma(alpha, acc[jh][i][2 * jj + 1], beta * old[jj][i].y);
                        *reinterpret_cast<double2*>(cbase + (int64_t)j * 8 * ldc + i * 8) = o;
                    }
            }
        } else {
#pragma unroll
            for (int j = 0; j < 4; j++)
#pragma unroll
                for (int i = 0; i < 4; i++) {
                    double2 o = make_double2(alpha * acc[j >> 1][i][2 * (j & 1)], alpha * acc[j >> 1][i][2 * (j & 1) + 1]);
                    *reinterpret_cast<double2*>(cbase + (int64_t)j * 8 * ldc + i * 8) = o;
                }
        }
    }
}

int g_num_sms = 0;
bool g_attr_set = false;
void ensure_attr() {
    if (!g_attr_set) {
        cudaFuncSetAttribute(gemm_nt_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                             (int)SMEM_BYTES);
        int dev = 0;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&g_num_sms, cudaDevAttrMultiProcessorCount, dev);
        g_attr_set = true;
    }
}

}  // namespace

static void launch_common(GemmArgs& g, cudaStream_t s, int reserve_sms = 0) {
    int64_t cap = 2 * (int64_t)(g_num_sms - reserve_sms);
    if (cap < 2) cap = 2;
    int64_t grid = g.total_tiles < cap ? g.total_tiles : cap;
    gemm_nt_kernel<<<(unsigned)grid, THREADS, SMEM_BYTES, s>>>(g);
    g_launch_count++;
}

void launch_gemm_nt(const double* A, int64_t lda, const double* B, int64_t ldb, double* C,
                    int64_t ldc, int64_t M, int64_t Ncols, int64_t K, double alpha, double beta,
                    cudaStream_t s) {
    if (M <= 0 || Ncols <= 0) return;
    ensure_attr();
    GemmArgs g{};
    g.mode = 0;
    g.Aseg[0] = A; g.lda_seg[0] = lda; g.Bseg[0] = B; g.ldb_seg[0] = ldb; g.C = C; g.ldc = ldc;
    g.seg_chunks = (int)(K / KC);
    g.mtiles = M / BM;
    g.K = K; g.alpha = alpha; g.beta = beta;
    g.total_tiles = (M / BM) * (Ncols / BN);
    launch_common(g, s);
}

// C (M x Ncols) = beta*C + alpha * [A_0 A_1 ...] [B_0 B_1 ...]^T, every segment 128 columns wide
void launch_gemm_nt_seg(int nseg, const double* const* A, const int64_t* lda, const double* const* B,
                        const int64_t* ldb, double* C, int64_t ldc, int64_t M, int64_t Ncols, double alpha,
                        double beta, cudaStream_t s) {
    if (M <= 0 || Ncols <= 0 || nseg <= 0) return;
    ensure_attr();
    GemmArgs g{};
    g.mode = 0;
    for (int i = 0; i < nseg; i++) { g.Aseg[i] = A[i]; g.lda_seg[i] = lda[i]; g.Bseg[i] = B[i]; g.ldb_seg[i] = ldb[i]; }
    g.C = C; g.ldc = ldc;
    g.seg_chunks = NB / KC;
    g.mtiles = M / BM;
    g.K = (int64_t)nseg * NB; g.alpha = alpha; g.beta = beta;
    g.total_tiles = (M / BM) * (Ncols / BN);
    launch_common(g, s);
}

// panel TRSM as a product with the explicit inverse: Pt (tiled, see TilePtrs) = A * invL^T,
// A = m x 128 column-major (lda), invL = 128 x 128 column-major (ld 128)
void launch_trsm_tiled(const double* A, int64_t lda, const double* invL, double* Pt, int64_t m,
                       cudaStream_t s) {
    if (m <= 0) return;
    ensure_attr();
    GemmArgs g{};
    g.mode = 0;
    g.Aseg[0] = A; g.lda_seg[0] = lda; g.Bseg[0] = invL; g.ldb_seg[0] = NB; g.C = Pt; g.ldc = 0; g.c_tiled = 1;
    g.seg_chunks = NB / KC;
    g.mtiles = m / BM;
    g.K = NB; g.alpha = 1.0; g.beta = 0.0;
    g.total_tiles = (m / BM) * (NB / BN);
    launch_common(g, s);
}

int64_t syrk_packed_tiles(int64_t nblk, int64_t k, int64_t jlo, int64_t jhi, int rank, int world) {
    if (jlo < k + 1) jlo = k + 1;
    if (jhi > nblk) jhi = nblk;
    int64_t J0 = jlo + ((rank - jlo % world) % world + world) % world;
    int64_t tiles = 0;
    for (int64_t J = J0; J < jhi; J += world) tiles += nblk - J;
    return tiles;
}

// Pt[0..nseg): the panels of one outer step in TILED layout; row block 0 <-> block row k+1 of
// the matrix (panel q's first q row blocks are unused).  K = 128 * nseg.
void launch_syrk_packed(Packed Apk, int64_t k, const double* const* Pt, int nseg, int64_t jlo, int64_t jhi,
                        int rank, int world, cudaStream_t s, int reserve_sms) {
    int64_t nblk = Apk.nblk();
    if (jlo < k + 1) jlo = k + 1;
    if (jhi > nblk) jhi = nblk;
    int64_t J0 = jlo + ((rank - jlo % world) % world + world) % world;
    int64_t tiles = syrk_packed_tiles(nblk, k, jlo, jhi, rank, world);
    if (tiles <= 0 || nseg <= 0) return;
    ensure_attr();
    GemmArgs g{};
    g.mode = 1;
    for (int i = 0; i < nseg; i++) { g.Aseg[i] = Pt[i]; g.Bseg[i] = Pt[i]; }
    g.a_tiled = 1; g.b_tiled = 1;
    g.seg_chunks = NB / KC;
    g.K = (int64_t)nseg * NB; g.alpha = -1.0; g.beta = 1.0;
    g.Pk = Apk; g.k = k; g.J0 = J0; g.w = world;
    g.total_tiles = tiles * 2;
    launch_common(g, s, reserve_sms);
}

}  // namespace sb
