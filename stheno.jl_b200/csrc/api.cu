// C ABI of libstheno_b200 (see include/stheno_b200.h): contexts, plan upload, the blocked
// right-looking Cholesky driver, logpdf / posterior / rand / VFE orchestration.
#include <dlfcn.h>
#include <math.h>
#include <nccl.h>
#include <stdlib.h>
#include <string.h>

#include <string>
#include <vector>

#include "sb_common.cuh"

namespace sb {

static thread_local std::string g_err;
void set_error(const std::string& msg) { g_err = msg; }
int32_t cuda_fail(cudaError_t e, const char* what, const char* file, int line) {
    g_err = std::string("CUDA error: ") + cudaGetErrorString(e) + " in " + what + " at " + file +
            ":" + std::to_string(line);
    if (e == cudaErrorMemoryAllocation) {
        cudaGetLastError();
        return SB_ERR_NOMEM;
    }
    return SB_ERR_CUDA;
}

}  // namespace sb

using namespace sb;

// NCCL is bound lazily with dlopen (only when world > 1): a single-GPU / Julia user never loads
// it, and inside a Python process that also imports torch the already-loaded libnccl.so.2
// (torch bundles its own) is reused instead of clashing with the system copy.
namespace nccl_dl {
typedef ncclResult_t (*GetUniqueId_t)(ncclUniqueId*);
typedef ncclResult_t (*CommInitRank_t)(ncclComm_t*, int, ncclUniqueId, int);
typedef ncclResult_t (*CommDestroy_t)(ncclComm_t);
typedef ncclResult_t (*Broadcast_t)(const void*, void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t);
typedef ncclResult_t (*AllReduce_t)(const void*, void*, size_t, ncclDataType_t, ncclRedOp_t, ncclComm_t, cudaStream_t);
typedef ncclResult_t (*AllGather_t)(const void*, void*, size_t, ncclDataType_t, ncclComm_t, cudaStream_t);
typedef ncclResult_t (*Group_t)(void);
typedef const char* (*ErrStr_t)(ncclResult_t);
static GetUniqueId_t GetUniqueId;
static CommInitRank_t CommInitRank;
static CommDestroy_t CommDestroy;
static Broadcast_t Broadcast;
static AllReduce_t AllReduce;
static AllGather_t AllGather;
static Group_t GroupStart, GroupEnd;
static ErrStr_t GetErrorString;
static bool loaded = false;
static bool load() {
    if (loaded) return true;
    void* h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
    if (!h) h = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
    if (!h) {
        sb::set_error(std::string("cannot dlopen libnccl.so.2: ") + dlerror());
        return false;
    }
#define SB_SYM(name) name = (name##_t)dlsym(h, "nccl" #name); if (!name) { sb::set_error("missing NCCL symbol nccl" #name); return false; }
    SB_SYM(GetUniqueId) SB_SYM(CommInitRank) SB_SYM(CommDestroy) SB_SYM(Broadcast) SB_SYM(AllReduce) SB_SYM(AllGather)
    GroupStart = (Group_t)dlsym(h, "ncclGroupStart");
    GroupEnd = (Group_t)dlsym(h, "ncclGroupEnd");
    GetErrorString = (ErrStr_t)dlsym(h, "ncclGetErrorString");
    if (!GroupStart || !GroupEnd || !GetErrorString) { sb::set_error("missing NCCL group symbols"); return false; }
#undef SB_SYM
    loaded = true;
    return true;
}
}  // namespace nccl_dl

#define SB_NCCL(call)                                                                   \
    do {                                                                                \
        ncclResult_t _r = (call);                                                       \
        if (_r != ncclSuccess) {                                                        \
            sb::set_error(std::string("NCCL error: ") + nccl_dl::GetErrorString(_r) + " in " #call); \
            return SB_ERR_NCCL;                                                         \
        }                                                                               \
    } while (0)

struct sb_ctx {
    int device = 0;
    int rank = 0, world = 1;
    ncclComm_t comm = nullptr;
    cudaStream_t stream = nullptr;
    cudaStream_t stream2 = nullptr;  // look-ahead panel stream (multi-GPU)
    cudaStream_t xstream[4] = {nullptr, nullptr, nullptr, nullptr};  // column-exchange streams, one per owner in flight
    sb_timings tm{};
    bool fine_timing = true;
    // 0: fp64 DMMA (mma.sync), the faster path on H100 and the default; 1: int8 Ozaki slices on wgmma (ozaki.cu)
    int trailing_mode = 0;
    int num_sms = 132;
    cudaEvent_t marks[8] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
    // peer-to-peer panel exchange over NVLink (multi-GPU, see "P2P panel exchange" below)
    struct P2PState {
        int state = 0;            // 0: not tried, 1: on, -1: unavailable (NCCL broadcast is used)
        char* arena = nullptr;    // counters | head slots | panel slots; IPC-exported to every peer
        size_t bytes = 0;
        char* peer[8] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
        uint32_t pub[8] = {0, 0, 0, 0, 0, 0, 0, 0};   // panels published so far by each owner (same on all ranks)
        void* xch = nullptr;      // handle-exchange staging
    } p2p;
    // caching device allocator: the factor (17 GB at N=65536) and the posterior workspace are
    // re-used across calls instead of paying cudaMalloc/cudaFree (both device-synchronising)
    struct PoolBlock { size_t bytes; void* p; };
    std::vector<PoolBlock> pool_free_list;
    size_t pool_cached_bytes = 0;
    cudaError_t pool_alloc(void** out, size_t bytes) {
        if (bytes == 0) bytes = 8;
        int best = -1;
        for (int i = 0; i < (int)pool_free_list.size(); i++) {
            size_t b = pool_free_list[i].bytes;
            if (b >= bytes && b <= bytes + bytes / 4 + 4096 && (best < 0 || b < pool_free_list[best].bytes)) best = i;
        }
        if (best >= 0) {
            *out = pool_free_list[best].p;
            pool_cached_bytes -= pool_free_list[best].bytes;
            pool_free_list.erase(pool_free_list.begin() + best);
            return cudaSuccess;
        }
        cudaError_t e = cudaMalloc(out, bytes);
        if (e == cudaErrorMemoryAllocation && !pool_free_list.empty()) {
            cudaGetLastError();
            pool_trim();
            e = cudaMalloc(out, bytes);
        }
        return e;
    }
    void pool_release(void* p, size_t bytes) {
        if (!p) return;
        if (bytes == 0) bytes = 8;
        pool_free_list.push_back({bytes, p});
        pool_cached_bytes += bytes;
    }
    void pool_trim() {
        for (auto& b : pool_free_list) cudaFree(b.p);
        pool_free_list.clear();
        pool_cached_bytes = 0;
    }
    std::vector<cudaEvent_t> ev;
    size_t ev_used = 0;
    cudaEvent_t next_event() {
        if (ev_used == ev.size()) {
            cudaEvent_t e;
            cudaEventCreate(&e);
            ev.push_back(e);
        }
        return ev[ev_used++];
    }
};

struct sb_factor {
    sb_ctx* ctx = nullptr;
    int64_t N = 0, Np = 0;
    Packed L{nullptr, 0};
    double* invL = nullptr;
    double* ldiag = nullptr;  // multi-GPU only: contiguous copies of the diagonal blocks L_kk (broadcast payload)
    double* logdet_blk = nullptr;
    long long* info_dev = nullptr;
    double* panel = nullptr;  // 2 x (Np x NB) panel buffers
    double* alpha = nullptr;  // Np
    bool has_alpha = false;
    double logdet = 0.0;
    size_t bytes_L = 0, bytes_invL = 0, bytes_ld = 0, bytes_panel = 0, bytes_alpha = 0, bytes_ldiag = 0;
    // int8 Ozaki trailing update (ozaki.cu): two sets (look-ahead) of int8 digit planes + row scales, and the
    // wide panel phase's buffers below; all allocated together
    bool oz = false;
    signed char* oz_planes[2] = {nullptr, nullptr};
    double* oz_scale[2] = {nullptr, nullptr};
    int* oz_expo[2] = {nullptr, nullptr};
    unsigned* sweep_flags = nullptr;     // 2*nblk flags of the persistent triangular sweep
    // logpdf(fx, y) followed by posterior(fx, y) is THE usage pattern (README.md:61-81): the forward
    // sweep v = L^{-1} delta of the last single-RHS logpdf is kept so posterior only adds the backward one
    double* vcache = nullptr;            // [2][Np]: delta, then v
    int* vcache_flag = nullptr;
    bool vcache_valid = false;
    OzMaps oz_maps[2];
    size_t bytes_oz_planes = 0;
    // wide panel phase (see wide_diag_phase): dense scratch of the step's 512 x 512 diagonal block stacked over an
    // identity (input and result copies), inv(L_512) and its digit planes
    double* wide_D = nullptr;        // [2][1024 x 512], ld 1024
    double* wide_W = nullptr;        // 512 x 512, column-major
    signed char* wide_wp = nullptr;  // digit planes of wide_W  [7][512][512]
    double* wide_wscale = nullptr;
    int* wide_wexpo = nullptr;
    OzMaps wide_wmaps;
};

namespace {

struct PhaseTimer {  // accumulates the stream time between start() and stop() into *acc
    sb_ctx* c;
    cudaEvent_t e0, e1;
    double* acc;
    PhaseTimer(sb_ctx* ctx, double* a) : c(ctx), acc(a) {
        e0 = c->next_event();
        e1 = c->next_event();
        cudaEventRecord(e0, c->stream);
    }
    void stop() { cudaEventRecord(e1, c->stream); }
    void collect() {
        float ms = 0;
        cudaEventElapsedTime(&ms, e0, e1);
        *acc += ms;
    }
};

struct DevBuf {
    void* p = nullptr;
    size_t bytes = 0;
    sb_ctx* ctx = nullptr;
    DevBuf() {}
    explicit DevBuf(sb_ctx* c) : ctx(c) {}
    ~DevBuf() {
        if (!p) return;
        if (ctx) ctx->pool_release(p, bytes); else cudaFree(p);
    }
    int32_t alloc(size_t nbytes) {
        bytes = nbytes ? nbytes : 8;
        if (ctx) SB_CUDA(ctx->pool_alloc(&p, bytes)); else SB_CUDA(cudaMalloc(&p, bytes));
        return SB_OK;
    }
    double* d() { return reinterpret_cast<double*>(p); }
};

// uploaded covariance plan
struct DevSpec {
    DevBuf pool;
    explicit DevSpec(sb_ctx* c) : pool(c) {}
    std::vector<double*> arr;
    std::vector<BlockDev> blocks;
    int64_t nrows = 0, ncols = 0;

    int32_t build(const sb_covspec* spec, cudaStream_t st, bool diag) {
        SB_CHECK(spec != nullptr, "null covspec");
        nrows = spec->nrows;
        ncols = spec->ncols;
        SB_CHECK(nrows >= 0 && ncols >= 0, "negative matrix size");
        SB_CHECK(spec->narrays >= 0 && spec->nterms >= 0 && spec->nblocks >= 0, "negative count");
        size_t total = 0;
        for (int a = 0; a < spec->narrays; a++) {
            const sb_array& A = spec->arrays[a];
            SB_CHECK(A.n >= 0 && A.dim >= 0 && A.dim <= MAX_DIM, "array: bad n/dim (dim <= 8)");
            SB_CHECK(A.n == 0 || A.data != nullptr, "array: null data");
            total += (size_t)A.n * (A.dim ? A.dim : 1);
            total = (total + 1) & ~(size_t)1;  // keep 16-byte alignment
        }
        SB_TRY(pool.alloc(total * sizeof(double)));
        arr.resize(spec->narrays);
        size_t off = 0;
        for (int a = 0; a < spec->narrays; a++) {
            const sb_array& A = spec->arrays[a];
            size_t cnt = (size_t)A.n * (A.dim ? A.dim : 1);
            arr[a] = pool.d() + off;
            if (cnt)
                SB_CUDA(cudaMemcpyAsync(arr[a], A.data, cnt * sizeof(double), cudaMemcpyDefault, st));
            off += cnt;
            off = (off + 1) & ~(size_t)1;
        }
        for (int bi = 0; bi < spec->nblocks; bi++) {
            const sb_block& B = spec->blocks[bi];
            SB_CHECK(B.row0 >= 0 && B.nrows >= 0 && B.row0 + B.nrows <= nrows, "block rows out of range");
            SB_CHECK(B.col0 >= 0 && B.ncols >= 0 && B.col0 + B.ncols <= ncols, "block cols out of range");
            SB_CHECK(B.term0 >= 0 && B.nterms >= 0 && B.term0 + B.nterms <= spec->nterms, "block terms out of range");
            if (diag) SB_CHECK(B.nrows == B.ncols, "diag spec: blocks must be square (paired points)");
            int done = 0;
            do {
                BlockDev d{};
                d.row0 = B.row0; d.nrows = B.nrows; d.col0 = B.col0; d.ncols = B.ncols;
                d.accumulate = done > 0;
                int n = B.nterms - done;
                if (n > MAX_TERMS) n = MAX_TERMS;
                d.nterms = n;
                for (int t = 0; t < n; t++) {
                    const sb_term& T = spec->terms[B.term0 + done + t];
                    SB_CHECK(T.kernel >= SB_K_SE && T.kernel <= SB_K_CONST, "unknown kernel id");
                    SB_CHECK(T.zl >= 0 && T.zl < spec->narrays && T.zr >= 0 && T.zr < spec->narrays, "term: bad input array index");
                    const sb_array& ZL = spec->arrays[T.zl];
                    const sb_array& ZR = spec->arrays[T.zr];
                    SB_CHECK(ZL.dim >= 1 && ZL.dim == ZR.dim, "term: zl/zr dimension mismatch");
                    SB_CHECK(ZL.n == B.nrows && ZR.n == B.ncols, "term: input length != block size");
                    TermDev& D = d.t[t];
                    d.tix[t] = B.term0 + done + t;
                    D.kernel = T.kernel; D.dim = ZL.dim; D.coeff = T.coeff; D.param = T.param;
                    D.zl = arr[T.zl]; D.zr = arr[T.zr];
                    D.sl = nullptr; D.sr = nullptr;
                    if (T.sl >= 0) {
                        SB_CHECK(T.sl < spec->narrays && spec->arrays[T.sl].n == B.nrows && spec->arrays[T.sl].dim == 0, "term: bad row scale vector");
                        D.sl = arr[T.sl];
                    }
                    if (T.sr >= 0) {
                        SB_CHECK(T.sr < spec->narrays && spec->arrays[T.sr].n == B.ncols && spec->arrays[T.sr].dim == 0, "term: bad col scale vector");
                        D.sr = arr[T.sr];
                    }
                }
                blocks.push_back(d);
                done += n;
            } while (done < B.nterms);
        }
        return SB_OK;
    }
};

// keep only rows [lo, hi) of every block (and, for paired/diag specs, the same range of columns);
// rows are re-based to lo.  Used to shard the posterior's test points across ranks.
void clip_rows(DevSpec& ds, int64_t lo, int64_t hi, bool diag) {
    std::vector<BlockDev> out;
    for (BlockDev b : ds.blocks) {
        int64_t r0 = b.row0 > lo ? b.row0 : lo;
        int64_t r1 = b.row0 + b.nrows < hi ? b.row0 + b.nrows : hi;
        if (r1 <= r0) continue;
        int64_t off = r0 - b.row0;
        for (int t = 0; t < b.nterms; t++) {
            b.t[t].zl += off * b.t[t].dim;
            if (b.t[t].sl) b.t[t].sl += off;
            if (diag) {
                b.t[t].zr += off * b.t[t].dim;
                if (b.t[t].sr) b.t[t].sr += off;
            }
        }
        b.row0 = r0 - lo;
        b.nrows = r1 - r0;
        if (diag) { b.col0 = b.row0; b.ncols = b.nrows; }
        out.push_back(b);
    }
    ds.blocks.swap(out);
    ds.nrows = hi - lo;
    if (diag) ds.ncols = hi - lo;
}

void begin_call(sb_ctx* c) {
    cudaSetDevice(c->device);
    c->ev_used = 0;
}

void count_launches(sb_ctx* c, int64_t before) { c->tm.kernel_launches += g_launch_count - before; }

// dense assembly of a (possibly padded) nrows x ncols matrix with leading dimension ld
int32_t assemble_dense(sb_ctx* c, DevSpec& ds, double* out, int64_t ld) {
    for (auto& b : ds.blocks) launch_assemble_dense(b, OutDense{out, ld}, c->stream);
    SB_CUDA(cudaGetLastError());
    return SB_OK;
}

int32_t assemble_diag(sb_ctx* c, DevSpec& ds, double* out) {
    for (auto& b : ds.blocks) launch_assemble_diag(b, out, c->stream);
    SB_CUDA(cudaGetLastError());
    return SB_OK;
}

// ---- blocked right-looking Cholesky on the packed matrix ----------------------------------
// Two-level blocking: the layout / diagonal-block size is NB = 128, but trailing updates are
// applied for TWO block columns at once (K = 256), which halves the C read-modify-write traffic
// and the per-tile prologue/epilogue share of the DMMA kernel.  Outer step (k0, k1 = k0+1):
//   L_00 = chol(A_00), Linv_00                         (potrf.cu, one CTA)
//   P1   = A[k0+1:, k0] * Linv_00^T                    (gemm_nt.cu)      -> Pc[:, 0:128]
//   A[:, k1] -= P1 * P1_k1^T                            (gemm_nt.cu, one block column, K = 128)
//   L_11 = chol(A_11), Linv_11 ; P2 = A[k1+1:, k1] * Linv_11^T          -> Pc[128:, 128:256]
//   A[I, J] -= Pc_I * Pc_J^T,  k1 < J <= I              (gemm_nt.cu, K = 256, owned columns)
// Multi-GPU: block column J is owned by rank J % world (1-D block-cyclic); each half panel is
// broadcast by its owner with ncclBroadcast, received panels are kept, so after the sweep every
// rank holds the complete factor and the solves need no communication.
struct CholEv { cudaEvent_t e[4]; };

// One grouped broadcast per panel: inverse of the diagonal block, the diagonal block itself, its
// logdet share and the tiled sub-diagonal panel.  Non-owners drop L_kk into their packed matrix, so
// after the sweep every rank holds the complete factor without any extra collective.
// ---------------------------------------------------------------------------------------------
// P2P panel exchange.  Next to the trailing update an NCCL panel broadcast is slow, because it is a
// kernel on BOTH sides: the receivers' copies spin on SMs until the owner has factored the panel and
// the trailing update has to give those SMs up (or the broadcast starves).  The panels are moved
// by the copy engines instead, with no SM on the receiving side waiting for data:
//   * every rank has one "arena" (cudaMalloc, IPC-mapped by all peers): 64 ready counters + 64 ack
//     counters + an error word | 8 head slots (inv(L_kk), L_kk, logdet) | 8 panel slots (2 look-ahead
//     sets x OUTER_BLOCKS tiled panels; these ARE the panel buffers the local kernels read and write);
//   * the owner of panel k factors it into its own slot k % 8, packs the head, and bumps ready[owner]
//     in every peer's arena (st.release.sys over NVLink);
//   * a receiver waits on its LOCAL counter (one thread), pulls the head with a small kernel (peer
//     loads) and the slab with cudaMemcpyAsync from the owner's mapped slot into its own slot (copy
//     engine, NVLink read), then bumps ack[me] in the owner's arena;
//   * before a rank overwrites slot k % 8 that last held a panel it OWNED (panel k - 8), it waits until
//     every peer has acknowledged that panel (flow control; almost always already true).
// Counters are absolute (never reset while the arena lives), compared wrap-safe.  A waiter gives up
// after 20 s and raises the arena's error word, which fails the factorisation instead of hanging.
// ---------------------------------------------------------------------------------------------
constexpr int P2P_SLOTS = 2 * OUTER_BLOCKS;
constexpr int64_t P2P_HEAD_ELEMS = 2 * (int64_t)NB * NB + 32;
constexpr size_t P2P_CTR_BYTES = 4096;
constexpr size_t P2P_HEAD_OFF = P2P_CTR_BYTES;
constexpr size_t P2P_PANEL_OFF = P2P_HEAD_OFF + (size_t)P2P_SLOTS * P2P_HEAD_ELEMS * sizeof(double);
constexpr int P2P_READY = 0, P2P_ACK = 64, P2P_ERR = 128;
static_assert(P2P_PANEL_OFF % 1024 == 0, "panel slots must stay 1 KB aligned");
struct P2PPeers { char* base[8]; };

__device__ __forceinline__ uint32_t ld_acquire_sys_u32(const uint32_t* p) {
    uint32_t v;
    asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_release_sys_u32(uint32_t* p, uint32_t v) {
    asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ unsigned long long p2p_now_ns() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}

// thread i < count waits until ctr[first + i] has reached `target` (thread `skip` does not wait)
__global__ void p2p_wait_kernel(const uint32_t* ctr, int first, int count, int skip, uint32_t target, uint32_t* err) {
    const int i = threadIdx.x;
    if (i >= count || i == skip) return;
    const uint32_t* p = ctr + first + i;
    const unsigned long long t0 = p2p_now_ns();
    unsigned spins = 0;
    while ((int)(ld_acquire_sys_u32(p) - target) < 0) {
        if (++spins > 256) __nanosleep(50);
        if ((spins & 4095u) == 0 && p2p_now_ns() - t0 > 20000000000ull) { atomicExch(err, 1u); return; }
    }
}

// thread r writes `value` to counter `index` in the arena of peer r (all peers, or only `only`)
__global__ void p2p_signal_kernel(P2PPeers peers, int world, int me, int index, uint32_t value, int only) {
    const int r = threadIdx.x;
    if (r >= world || r == me || (only >= 0 && r != only)) return;
    __threadfence_system();
    st_release_sys_u32(reinterpret_cast<uint32_t*>(peers.base[r]) + index, value);
}

__global__ void p2p_pack_head_kernel(const double* __restrict__ invL, const double* __restrict__ ldiag,
                                     const double* __restrict__ logdet, double* __restrict__ head) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < NB * NB) { head[i] = invL[i]; head[NB * NB + i] = ldiag[i]; }
    if (i == 0) head[2 * NB * NB] = logdet[0];
}

// reads the owner's head slot over NVLink (volatile loads: never served from a stale line) and
// scatters it: inv(L_kk), the contiguous copy of L_kk, L_kk inside the packed factor, logdet term
__global__ void p2p_pull_head_kernel(const double* head, double* __restrict__ invL, double* __restrict__ ldiag,
                                     double* __restrict__ Lkk, int64_t ldL, double* __restrict__ logdet) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < NB * NB) {
        invL[i] = __ldcv(head + i);
        const double v = __ldcv(head + NB * NB + i);
        ldiag[i] = v;
        Lkk[(int64_t)(i / NB) * ldL + (i % NB)] = v;
    }
    if (i == 0) logdet[0] = __ldcv(head + 2 * NB * NB);
}

static int32_t nccl_barrier(sb_ctx* c, void* scratch4) {
    SB_NCCL(nccl_dl::AllReduce(scratch4, scratch4, 1, ncclInt, ncclMin, c->comm, c->stream));
    SB_CUDA(cudaStreamSynchronize(c->stream));
    return SB_OK;
}

static void p2p_close(sb_ctx* c) {
    auto& P = c->p2p;
    for (int r = 0; r < 8; r++) {
        if (P.peer[r] && r != c->rank) cudaIpcCloseMemHandle(P.peer[r]);
        P.peer[r] = nullptr;
    }
    if (P.arena) cudaFree(P.arena);
    P.arena = nullptr;
    P.bytes = 0;
}

// Collective: make sure every rank has an arena with panel slots for order-Np factors, mapped by all.
// Falls back (state = -1, once, on every rank together) when CUDA IPC is not available.
static int32_t p2p_ensure(sb_ctx* c, int64_t Np) {
    auto& P = c->p2p;
    if (P.state == 0) {
        const char* e = getenv("SB_P2P");
        if ((e && e[0] == '0') || c->world > 8) P.state = -1;
    }
    if (P.state < 0) return SB_OK;
    const size_t need = P2P_PANEL_OFF + (size_t)P2P_SLOTS * tiled_panel_elems(Np) * sizeof(double);
    if (P.state == 1 && P.bytes >= need) return SB_OK;
    const int world = c->world, rank = c->rank;
    SB_CUDA(cudaStreamSynchronize(c->stream));
    SB_CUDA(cudaStreamSynchronize(c->stream2));
    if (!P.xch) SB_CUDA(cudaMalloc(&P.xch, 8 * sizeof(cudaIpcMemHandle_t) + 64));
    int* flag_dev = reinterpret_cast<int*>(static_cast<char*>(P.xch) + 8 * sizeof(cudaIpcMemHandle_t));
    int one = 1;
    SB_CUDA(cudaMemcpy(flag_dev, &one, sizeof(int), cudaMemcpyHostToDevice));
    if (P.arena) {                       // growing: nobody may still be pulling from the old arena
        SB_TRY(nccl_barrier(c, flag_dev));
        p2p_close(c);
    }
    int ok = 1;
    cudaIpcMemHandle_t mine;
    memset(&mine, 0, sizeof(mine));
    if (cudaMalloc((void**)&P.arena, need) != cudaSuccess) { cudaGetLastError(); P.arena = nullptr; ok = 0; }
    if (ok && cudaMemset(P.arena, 0, P2P_PANEL_OFF) != cudaSuccess) ok = 0;
    if (ok && cudaIpcGetMemHandle(&mine, P.arena) != cudaSuccess) { cudaGetLastError(); ok = 0; }
    SB_CUDA(cudaMemcpy(static_cast<char*>(P.xch) + rank * sizeof(mine), &mine, sizeof(mine), cudaMemcpyHostToDevice));
    SB_CUDA(cudaMemcpy(flag_dev, &ok, sizeof(int), cudaMemcpyHostToDevice));
    SB_NCCL(nccl_dl::AllGather(static_cast<char*>(P.xch) + rank * sizeof(mine), P.xch, sizeof(mine), ncclChar, c->comm, c->stream));
    SB_TRY(nccl_barrier(c, flag_dev));   // min over ranks of ok
    SB_CUDA(cudaMemcpy(&ok, flag_dev, sizeof(int), cudaMemcpyDeviceToHost));
    if (ok) {
        cudaIpcMemHandle_t all[8];
        SB_CUDA(cudaMemcpy(all, P.xch, world * sizeof(mine), cudaMemcpyDeviceToHost));
        for (int r = 0; r < world && ok; r++) {
            if (r == rank) { P.peer[r] = P.arena; continue; }
            void* q = nullptr;
            if (cudaIpcOpenMemHandle(&q, all[r], cudaIpcMemLazyEnablePeerAccess) != cudaSuccess) { cudaGetLastError(); ok = 0; }
            P.peer[r] = static_cast<char*>(q);
        }
        SB_CUDA(cudaMemcpy(flag_dev, &ok, sizeof(int), cudaMemcpyHostToDevice));
        SB_TRY(nccl_barrier(c, flag_dev));
        SB_CUDA(cudaMemcpy(&ok, flag_dev, sizeof(int), cudaMemcpyDeviceToHost));
    }
    if (!ok) {
        p2p_close(c);
        P.state = -1;
        if (rank == 0) fprintf(stderr, "[stheno_b200] CUDA IPC peer mapping unavailable: panels go through ncclBroadcast\n");
        return SB_OK;
    }
    P.bytes = need;
    P.state = 1;
    for (int r = 0; r < 8; r++) P.pub[r] = 0;
    return SB_OK;
}

struct P2PRun {                 // one factorisation's view of the arena
    bool on = false;
    P2PPeers peers{};
    int64_t slot_elems = 0;     // doubles per panel slot
    std::vector<uint32_t> ord;  // ord[k]: absolute ordinal (1-based) of panel k among its owner's panels
    uint32_t guarded = 0;       // acks up to this ordinal of MY panels have already been waited for on the panel stream
    uint32_t* ctr(sb_ctx* c) const { return reinterpret_cast<uint32_t*>(c->p2p.arena); }
    double* head(char* base, int64_t k) const {
        return reinterpret_cast<double*>(base + P2P_HEAD_OFF) + (k % P2P_SLOTS) * P2P_HEAD_ELEMS;
    }
    double* slot(char* base, int s) const { return reinterpret_cast<double*>(base + P2P_PANEL_OFF) + (int64_t)s * slot_elems; }
};

// Before anything is written into slot k % 8 (TRSM output, pulled slab, packed head): the last panel this
// rank OWNED in that slot (k - 8m) must have been pulled by every peer.  Acks are monotone per owner, so
// one wait per new high-water mark is enough.
static int32_t p2p_slot_guard(sb_ctx* c, P2PRun& R, int64_t k, cudaStream_t st) {
    for (int64_t kp = k - P2P_SLOTS; kp >= 0; kp -= P2P_SLOTS) {
        if ((int)(kp % c->world) != c->rank) continue;
        if ((int)(R.ord[kp] - R.guarded) > 0) {
            p2p_wait_kernel<<<1, 32, 0, st>>>(R.ctr(c), P2P_ACK, c->world, c->rank, R.ord[kp], R.ctr(c) + P2P_ERR);
            SB_CUDA(cudaGetLastError());
            R.guarded = R.ord[kp];
        }
        break;
    }
    return SB_OK;
}

static int32_t p2p_publish(sb_ctx* c, sb_factor* f, P2PRun& R, int64_t k, cudaStream_t st) {
    const int64_t bo = k * (int64_t)NB * NB;
    p2p_pack_head_kernel<<<NB * NB / 256, 256, 0, st>>>(f->invL + bo, f->ldiag + bo, f->logdet_blk + k, R.head(c->p2p.arena, k));
    p2p_signal_kernel<<<1, 32, 0, st>>>(R.peers, c->world, c->rank, P2P_READY + c->rank, R.ord[k], -1);
    SB_CUDA(cudaGetLastError());
    return SB_OK;
}

static int32_t p2p_pull(sb_ctx* c, sb_factor* f, P2PRun& R, int64_t k, int owner, int64_t slab_off, size_t slab_elems,
                        cudaStream_t st) {
    const int64_t bo = k * (int64_t)NB * NB;
    p2p_wait_kernel<<<1, 32, 0, st>>>(R.ctr(c), P2P_READY + owner, 1, -1, R.ord[k], R.ctr(c) + P2P_ERR);
    p2p_pull_head_kernel<<<NB * NB / 256, 256, 0, st>>>(R.head(c->p2p.peer[owner], k), f->invL + bo, f->ldiag + bo,
                                                          f->L.blk(k, k), f->L.ld(k), f->logdet_blk + k);
    SB_CUDA(cudaGetLastError());
    if (slab_elems) {
        const int s = (int)(k % P2P_SLOTS);
        SB_CUDA(cudaMemcpyAsync(R.slot(c->p2p.arena, s) + slab_off, R.slot(c->p2p.peer[owner], s) + slab_off,
                                slab_elems * sizeof(double), cudaMemcpyDeviceToDevice, st));
    }
    p2p_signal_kernel<<<1, 32, 0, st>>>(R.peers, c->world, c->rank, P2P_ACK + c->rank, R.ord[k], owner);
    SB_CUDA(cudaGetLastError());
    return SB_OK;
}

static int32_t bcast_panel(sb_ctx* c, sb_factor* f, int64_t k, double* Pslab, size_t slab_elems, int owner,
                           cudaStream_t st) {
    const int64_t bo = k * (int64_t)NB * NB;
    SB_NCCL(nccl_dl::GroupStart());
    SB_NCCL(nccl_dl::Broadcast(f->invL + bo, f->invL + bo, (size_t)NB * NB, ncclDouble, owner, c->comm, st));
    SB_NCCL(nccl_dl::Broadcast(f->ldiag + bo, f->ldiag + bo, (size_t)NB * NB, ncclDouble, owner, c->comm, st));
    SB_NCCL(nccl_dl::Broadcast(f->logdet_blk + k, f->logdet_blk + k, 1, ncclDouble, owner, c->comm, st));
    if (slab_elems) SB_NCCL(nccl_dl::Broadcast(Pslab, Pslab, slab_elems, ncclDouble, owner, c->comm, st));
    SB_NCCL(nccl_dl::GroupEnd());
    if (owner != c->rank)
        SB_CUDA(cudaMemcpy2DAsync(f->L.blk(k, k), f->L.ld(k) * sizeof(double), f->ldiag + bo, NB * sizeof(double),
                                  NB * sizeof(double), NB, cudaMemcpyDeviceToDevice, st));
    return SB_OK;
}

// Multi-GPU DMMA factorisation with look-ahead.  Stream 1 (c->stream) runs the trailing updates,
// stream 2 (c->stream2) the panel phases (column catch-up, potrf, TRSM, panel exchange, untile).
// The trailing update of outer step s is split into T^A (the 4 block columns that form the NEXT
// step's panels; full grid) and T^B (everything to the right; persistent grid minus
// LOOKAHEAD_SMS SMs).  Panel phase s+1 starts as soon as T^A_s is done and overlaps T^B_s, so the
// serial potrf/TRSM/broadcast chain leaves the critical path.  Two sets of tiled panel buffers.
constexpr int LOOKAHEAD_SMS = 8;

// How many SMs T^B leaves to the concurrent panel phase.  With a fixed 8 SMs the panel-phase GEMMs
// (catch-up SYRK, TRSM-as-GEMM: up to ~2000 DMMA half-tiles per outer step) crawl on 16 CTA slots and
// the panel chain, not the trailing update, can set the pace of the second half of the factorisation.
// Pick the reservation that balances  T^B * S/(S-r)  against  serial chain + panel GEMM work / r.
// Per-tile cost: time per SM of one 128 x 64 half-tile with K = 512 (2*128*64*512 flop) at the DMMA
// trailing-update rate bench.py measured at N = 65536 on one H100 80GB (700 W), 28.1 TFLOP/s over 132 SMs.
// The serial-chain latencies below have not been measured on H100.
constexpr double DMMA_HALF_TILE_US = 39.5;
static int pick_lookahead_sms(int num_sms, double tilesB_half, int nq_next, int64_t rows_next) {
    const double serial_us = nq_next * 230.0;   // potrf + exchange latency; unmeasured
    // DMMA half-tiles of the next panel phase: TRSM (nq panels) + catch-up (0 + 1 + 2 + 3 segments)
    const double gemm_tiles = (double)nq_next * (rows_next / 64.0) * (1.0 + 0.5 * (nq_next - 1) * 0.5);
    const int cand[] = {8, 12, 16, 24, 32, 48, 64};
    int best = LOOKAHEAD_SMS;
    double best_t = 1e30;
    for (int r : cand) {
        if (r >= num_sms / 2) break;
        const double tB = tilesB_half * DMMA_HALF_TILE_US / (num_sms - r);
        // (panel-phase GEMM tiles have K = 128: a quarter of a half-tile's work)
        const double tP = serial_us + gemm_tiles * (DMMA_HALF_TILE_US / 4.0) / r;
        const double t = tB > tP ? tB : tP;
        if (t < best_t - 1e-9) { best_t = t; best = r; }
    }
    return best;
}

struct CommEv { cudaEvent_t a, b; };

// Panels q0 .. q1-1 of the outer step at block column k0: column catch-up, potrf, TRSM, exchange, untile.
// comm_ev (fine timing): one interval per panel around its exchange (empty on one rank).
static int32_t panel_phase(sb_ctx* c, sb_factor* f, int64_t k0, int q0, int q1, double* const* Pw, const double* const* Pt,
                           int rank, int world, cudaStream_t st, std::vector<CommEv>* comm_ev, P2PRun* R = nullptr) {
    const bool p2p = R && R->on;
    const int64_t Np = f->Np;
    for (int q = q0; q < q1; q++) {
        const int64_t kq = k0 + q;
        const int64_t mq = Np - (kq + 1) * NB;
        const int owner = (int)(kq % world);
        double* Pq = Pw[q] + tiled_panel_elems((int64_t)q * NB);
        if (owner == rank) {
            if (q > 0) launch_syrk_packed(f->L, k0, Pt, q, kq, kq + 1, rank, world, st);
            launch_potrf_inv(f->L, kq, f->N, f->invL, f->logdet_blk, f->info_dev, st, world > 1 ? f->ldiag : nullptr);
            if (p2p) SB_TRY(p2p_slot_guard(c, *R, kq, st));
            if (mq > 0)
                launch_trsm_tiled(f->L.blk(kq + 1, kq), f->L.ld(kq), f->invL + kq * (int64_t)NB * NB, Pq, mq, st);
        }
        CommEv ce{nullptr, nullptr};
        if (comm_ev && c->fine_timing) {
            ce.a = c->next_event(); ce.b = c->next_event();
            SB_CUDA(cudaEventRecord(ce.a, st));
        }
        if (world > 1) {
            const size_t slab = mq > 0 ? (size_t)tiled_panel_elems(mq) : 0;
            if (!p2p) {
                SB_TRY(bcast_panel(c, f, kq, Pq, slab, owner, st));
            } else if (owner == rank) {
                SB_TRY(p2p_publish(c, f, *R, kq, st));
            } else {
                SB_TRY(p2p_slot_guard(c, *R, kq, st));
                SB_TRY(p2p_pull(c, f, *R, kq, owner, tiled_panel_elems((int64_t)q * NB), slab, st));
            }
        }
        if (ce.a) { SB_CUDA(cudaEventRecord(ce.b, st)); comm_ev->push_back(ce); }
        if (mq > 0) launch_untile_panel(Pt[q], q, mq / NB, f->L.blk(kq + 1, kq), f->L.ld(kq), st);
    }
    return SB_OK;
}

// ---------------------------------------------------------------------------------------------
// Wide panel phase (int8 Ozaki path).  The per-panel chain  catch-up -> potrf -> TRSM -> exchange  (x 512)
// keeps full-height DMMA products between the potrfs; on several GPUs that chain, squeezed onto the
// SMs the trailing update leaves free, can bound the factorisation.  Here the four block columns of an outer step are factored together:
//   (0) multi-GPU: every owner publishes its (already updated) block column, everyone pulls the other three
//       into its own packed matrix (copy engines, see "P2P panel exchange") -- all ranks then do the rest
//       redundantly, so nothing but the raw columns crosses NVLink;
//   (1) the 512 x 512 diagonal block is copied into a dense scratch stacked over an identity and factored
//       right-looking with 128-blocks (potrf_inv + small DMMA products).  The same column operations applied
//       to the identity rows leave inv(L_512)^T there, for free;
//   (2) ALL rows below are solved by ONE product  X = A inv(L_512)^T  on the tensor cores (int8 digit planes
//       of A and of inv(L_512), K = N = 512), written straight into the tiled panel buffers.
// The serial part per step is four potrfs + nine tiny products; the O(m 512^2) work is a single launch.
// ---------------------------------------------------------------------------------------------
constexpr int64_t WIDE = (int64_t)OUTER_BLOCKS * NB;   // 512
static_assert(OUTER_BLOCKS == 4 && NB == 128, "wide panel phase is written for 4 x 128");

__global__ void wide_load_kernel(Packed L, int64_t k0, int nq, double* __restrict__ D) {
    const int c = blockIdx.x;              // column inside the step
    const int64_t g0 = k0 * NB;
    for (int r = threadIdx.x; r < 2 * WIDE; r += blockDim.x) {
        double v = 0.0;
        if (r < nq * NB) {
            if (r / NB >= c / NB) v = *L.at(g0 + r, g0 + c);
        } else if (r >= WIDE && r - WIDE == c) {
            v = 1.0;
        }
        D[(int64_t)c * (2 * WIDE) + r] = v;
    }
}

// the sub-diagonal blocks of the factored diagonal block go back into the packed matrix
__global__ void wide_store_kernel(Packed L, int64_t k0, int nq, const double* __restrict__ X) {
    const int c = blockIdx.x;
    const int64_t g0 = k0 * NB;
    for (int r = threadIdx.x; r < nq * NB; r += blockDim.x)
        if (r / NB > c / NB) *L.at(g0 + r, g0 + c) = X[(int64_t)c * (2 * WIDE) + r];
}

static int32_t p2p_exchange_col(sb_ctx* c, sb_factor* f, P2PRun& R, int64_t k, cudaStream_t st) {
    const int owner = (int)(k % c->world), s = (int)(k % P2P_SLOTS);
    const size_t bytes = (size_t)f->L.ld(k) * NB * sizeof(double);   // the block column is one contiguous slab
    double* col = f->L.blk(k, k);
    if (owner == c->rank) {
        SB_TRY(p2p_slot_guard(c, R, k, st));
        SB_CUDA(cudaMemcpyAsync(R.slot(c->p2p.arena, s), col, bytes, cudaMemcpyDeviceToDevice, st));
        p2p_signal_kernel<<<1, 32, 0, st>>>(R.peers, c->world, c->rank, P2P_READY + c->rank, R.ord[k], -1);
    } else {
        p2p_wait_kernel<<<1, 32, 0, st>>>(R.ctr(c), P2P_READY + owner, 1, -1, R.ord[k], R.ctr(c) + P2P_ERR);
        SB_CUDA(cudaMemcpyAsync(col, R.slot(c->p2p.peer[owner], s), bytes, cudaMemcpyDeviceToDevice, st));
        p2p_signal_kernel<<<1, 32, 0, st>>>(R.peers, c->world, c->rank, P2P_ACK + c->rank, R.ord[k], owner);
    }
    SB_CUDA(cudaGetLastError());
    return SB_OK;
}

// Serial part of the wide panel phase (panel stream): column exchange, the 512 x 512 diagonal block, inv(L_512)
// and its digit planes.  Only small kernels: it runs on the few SMs the first part of T^B leaves free.
static int32_t wide_diag_phase(sb_ctx* c, sb_factor* f, int64_t k0, int nq, int rank, int world, cudaStream_t st,
                               std::vector<CommEv>* comm_ev, P2PRun* R) {
    const int64_t nblk = f->L.nblk();
    const bool bulk = nblk - (k0 + nq) > 0;            // rows under the step (then nq == OUTER_BLOCKS)
    if (world > 1) {
        if (!(R && R->on)) {
            sb::set_error("wide panel phase needs the peer-to-peer arena");
            return SB_ERR_UNSUPPORTED;
        }
        CommEv ce{nullptr, nullptr};
        if (comm_ev && c->fine_timing) {
            ce.a = c->next_event(); ce.b = c->next_event();
            SB_CUDA(cudaEventRecord(ce.a, st));
        }
        // The columns of a step come from different owners: their pulls run side by side, one stream per owner
        // (two columns of the same owner stay in order on one stream, which keeps its counters monotone).
        cudaEvent_t e0 = c->next_event();
        SB_CUDA(cudaEventRecord(e0, st));
        bool used[4] = {false, false, false, false};
        for (int q = 0; q < nq; q++) {
            const int xi = (int)((k0 + q) % world) % 4;
            if (!used[xi]) { SB_CUDA(cudaStreamWaitEvent(c->xstream[xi], e0, 0)); used[xi] = true; }
            SB_TRY(p2p_exchange_col(c, f, *R, k0 + q, c->xstream[xi]));
        }
        for (int xi = 0; xi < 4; xi++) {
            if (!used[xi]) continue;
            cudaEvent_t e1 = c->next_event();
            SB_CUDA(cudaEventRecord(e1, c->xstream[xi]));
            SB_CUDA(cudaStreamWaitEvent(st, e1, 0));
        }
        if (ce.a) { SB_CUDA(cudaEventRecord(ce.b, st)); comm_ev->push_back(ce); }
    }
    double* Din = f->wide_D;
    double* X = f->wide_D + 2 * WIDE * WIDE;
    const int64_t ldd = 2 * WIDE;
    wide_load_kernel<<<nq * NB, 256, 0, st>>>(f->L, k0, nq, Din);
    const int64_t rtot = bulk ? 2 * WIDE : (int64_t)nq * NB;     // rows of the scratch that take part
    for (int q = 0; q < nq; q++) {
        const int64_t kq = k0 + q;
        const int64_t dq = (int64_t)q * NB + (int64_t)q * NB * ldd;   // block (q, q)
        launch_potrf_inv(f->L, kq, f->N, f->invL, f->logdet_blk, f->info_dev, st, f->ldiag, Din + dq, ldd);
        const int64_t mq = rtot - (q + 1) * NB;
        if (mq > 0)
            launch_gemm_nt(Din + dq + NB, ldd, f->invL + kq * (int64_t)NB * NB, NB, X + dq + NB, ldd, mq, NB, NB, 1.0, 0.0, st);
        for (int q2 = q + 1; q2 < nq; q2++) {
            const int64_t xo = (int64_t)q2 * NB + (int64_t)q * NB * ldd;       // X rows from block q2 down, column q
            const int64_t co = (int64_t)q2 * NB + (int64_t)q2 * NB * ldd;      // block (q2, q2) and below
            launch_gemm_nt(X + xo, ldd, X + xo, ldd, Din + co, ldd, rtot - q2 * NB, NB, NB, -1.0, 1.0, st);
        }
    }
    wide_store_kernel<<<nq * NB, 256, 0, st>>>(f->L, k0, nq, X);
    SB_CUDA(cudaGetLastError());
    if (!bulk) return SB_OK;
    // inv(L_512)[n, k] = (identity rows of X)[k, n]
    launch_transpose(X + WIDE, ldd, WIDE, WIDE, f->wide_W, WIDE, st);
    OzSrc ws{};
    ws.nseg = OUTER_BLOCKS;
    for (int q = 0; q < OUTER_BLOCKS; q++) { ws.base[q] = f->wide_W + (int64_t)q * NB * WIDE; ws.ld[q] = WIDE; ws.rbs[q] = NB; }
    launch_oz_slice(ws, 0, OUTER_BLOCKS, 0, WIDE, f->wide_wscale, f->wide_wexpo, f->wide_wp, st);
    return SB_OK;
}

// Parallel part (trailing stream, whole GPU): digit planes of the un-normalised columns, the panel solve
// X = A inv(L_512)^T on the tensor cores (K blocks above the diagonal of inv(L_512) skipped) written over the
// columns in the packed matrix, digit planes of X for the trailing updates.  `set`: the digit-plane set of this
// step (it first holds the planes of A, then those of X).
static int32_t wide_bulk_phase(sb_ctx* c, sb_factor* f, int64_t k0, int nq, int set, cudaStream_t st) {
    const int64_t nblk = f->L.nblk(), Np = f->Np;
    const int64_t below = nblk - (k0 + nq);
    if (below <= 0) return SB_OK;
    OzSrc as{};
    as.nseg = OUTER_BLOCKS;
    const int64_t r0 = k0 + OUTER_BLOCKS;              // first block row under the step
    double* xcol[OUTER_BLOCKS];
    int64_t ldx[OUTER_BLOCKS];
    for (int q = 0; q < OUTER_BLOCKS; q++) {
        xcol[q] = f->L.blk(r0, k0 + q); ldx[q] = f->L.ld(k0 + q);
        as.base[q] = xcol[q]; as.ld[q] = ldx[q]; as.rbs[q] = NB;
    }
    launch_oz_slice(as, 0, below, r0 * NB, Np, f->oz_scale[set], f->oz_expo[set], f->oz_planes[set], st);
    if (launch_panel_solve_ozaki(xcol, ldx, below * NB, &f->oz_maps[set], f->oz_scale[set], r0 * NB, &f->wide_wmaps,
                                 f->wide_wscale, st) != 0) {
        sb::set_error("int8 Ozaki panel solve failed to launch");
        return SB_ERR_CUDA;
    }
    launch_oz_slice(as, 0, below, r0 * NB, Np, f->oz_scale[set], f->oz_expo[set], f->oz_planes[set], st);
    SB_CUDA(cudaGetLastError());
    return SB_OK;
}

// Start of a factorisation over the IPC-mapped arena: ordinal of every panel among its owner's panels, and (on
// stream st) a wait until every panel this rank published in earlier factorisations has been pulled by everyone.
static int32_t p2p_run_begin(sb_ctx* c, sb_factor* f, P2PRun& R, int world, int rank, cudaStream_t st) {
    const int64_t nblk = f->L.nblk();
    R.on = true;
    R.slot_elems = tiled_panel_elems(f->Np);
    for (int r = 0; r < 8; r++) R.peers.base[r] = c->p2p.peer[r];
    R.ord.resize(nblk);
    R.guarded = c->p2p.pub[rank];
    for (int64_t k = 0; k < nblk; k++) R.ord[k] = ++c->p2p.pub[k % world];
    p2p_wait_kernel<<<1, 32, 0, st>>>(R.ctr(c), P2P_ACK, world, rank, R.guarded, R.ctr(c) + P2P_ERR);
    SB_CUDA(cudaGetLastError());
    return SB_OK;
}

// End of a two-stream factorisation: the trailing stream waits for the panel stream and the host for both, a
// timed-out peer exchange fails the factorisation, and the exchange intervals and panel-stream phases (fine
// timing) are added to comm_ms and panel_chain_ms.
static int32_t finish_two_streams(sb_ctx* c, const P2PRun& R, const std::vector<CommEv>& comm_ev,
                                  const std::vector<CommEv>& chain_ev) {
    cudaEvent_t e_pend = c->next_event();
    SB_CUDA(cudaEventRecord(e_pend, c->stream2));
    SB_CUDA(cudaStreamWaitEvent(c->stream, e_pend, 0));
    SB_CUDA(cudaGetLastError());
    SB_CUDA(cudaStreamSynchronize(c->stream));
    if (R.on) {
        uint32_t err = 0;
        SB_CUDA(cudaMemcpy(&err, R.ctr(c) + P2P_ERR, sizeof(err), cudaMemcpyDeviceToHost));
        if (err) {
            sb::set_error("peer-to-peer panel exchange timed out (a peer rank stopped making progress)");
            return SB_ERR_NCCL;
        }
    }
    if (c->fine_timing) {
        // exchange time includes waiting for the owner's panel work on the other ranks
        for (auto& ce : comm_ev) {
            float ms = 0;
            cudaEventElapsedTime(&ms, ce.a, ce.b);
            c->tm.comm_ms += ms;
        }
        for (auto& ce : chain_ev) {
            float ms = 0;
            cudaEventElapsedTime(&ms, ce.a, ce.b);
            c->tm.panel_chain_ms += ms;
        }
    }
    return SB_OK;
}

// Look-ahead factorisation (see above).  Panels move by the P2P exchange when the arena is mapped, else by the
// NCCL broadcast.
static int32_t cholesky_lookahead(sb_ctx* c, sb_factor* f, int world, int rank) {
    const int64_t nblk = f->L.nblk(), Np = f->Np;
    std::vector<CommEv> comm_ev, chain_ev;
    cudaStream_t s1 = c->stream, s2 = c->stream2;
    const int64_t nsteps = (nblk + OUTER_BLOCKS - 1) / OUTER_BLOCKS;
    double* Pw[2][OUTER_BLOCKS];
    const double* Pt[2][OUTER_BLOCKS];
    for (int set = 0; set < 2; set++)
        for (int q = 0; q < OUTER_BLOCKS; q++)
            Pt[set][q] = Pw[set][q] = f->panel + (int64_t)(set * OUTER_BLOCKS + q) * tiled_panel_elems(Np);
    std::vector<cudaEvent_t> ev_p(nsteps), ev_a(nsteps), ev_t0(nsteps), ev_t1(nsteps);
    for (int64_t s = 0; s < nsteps; s++) {
        ev_p[s] = c->next_event(); ev_a[s] = c->next_event(); ev_t0[s] = c->next_event(); ev_t1[s] = c->next_event();
    }
    cudaEvent_t e_start = c->next_event();
    // stream 2 starts after everything already queued on stream 1 (assembly)
    SB_CUDA(cudaEventRecord(e_start, s1));
    SB_CUDA(cudaStreamWaitEvent(s2, e_start, 0));
    P2PRun R;
    if (c->p2p.state == 1) {
        SB_TRY(p2p_run_begin(c, f, R, world, rank, s2));
        for (int set = 0; set < 2; set++)   // the arena slots ARE the tiled panel buffers
            for (int q = 0; q < OUTER_BLOCKS; q++) Pt[set][q] = Pw[set][q] = R.slot(c->p2p.arena, set * OUTER_BLOCKS + q);
    }
    {
        const int nq0 = (int)(nblk < OUTER_BLOCKS ? nblk : OUTER_BLOCKS);
        SB_TRY(panel_phase(c, f, 0, 0, nq0, Pw[0], Pt[0], rank, world, s2, &comm_ev, &R));
        SB_CUDA(cudaEventRecord(ev_p[0], s2));
    }
    double flops = 0;
    int64_t nlaunch = 0;
    for (int64_t s = 0; s < nsteps; s++) {
        const int64_t k0 = s * OUTER_BLOCKS;
        const int nq = (int)(nblk - k0 < OUTER_BLOCKS ? nblk - k0 : OUTER_BLOCKS);
        const int set = (int)(s & 1);
        const int64_t jt = k0 + nq;
        SB_CUDA(cudaStreamWaitEvent(s1, ev_p[s], 0));
        SB_CUDA(cudaEventRecord(ev_t0[s], s1));
        if (jt < nblk) {
            const int64_t jA = jt + OUTER_BLOCKS < nblk ? jt + OUTER_BLOCKS : nblk;
            launch_syrk_packed(f->L, k0, Pt[set], nq, jt, jA, rank, world, s1);              // T^A: next panels' columns
            SB_CUDA(cudaEventRecord(ev_a[s], s1));
            if (s + 1 < nsteps) {
                const int nq1 = (int)(nblk - jt < OUTER_BLOCKS ? nblk - jt : OUTER_BLOCKS);
                SB_CUDA(cudaStreamWaitEvent(s2, ev_a[s], 0));
                CommEv ch{nullptr, nullptr};
                if (c->fine_timing) { ch.a = c->next_event(); ch.b = c->next_event(); SB_CUDA(cudaEventRecord(ch.a, s2)); }
                SB_TRY(panel_phase(c, f, jt, 0, nq1, Pw[set ^ 1], Pt[set ^ 1], rank, world, s2, &comm_ev, &R));
                SB_CUDA(cudaEventRecord(ev_p[s + 1], s2));
                if (ch.a) { SB_CUDA(cudaEventRecord(ch.b, s2)); chain_ev.push_back(ch); }
            }
            if (jA < nblk) {                                                                // T^B
                const double tilesB = 2.0 * (double)syrk_packed_tiles(nblk, k0, jA, nblk, rank, world);
                const int nq1 = (int)(nblk - jt < OUTER_BLOCKS ? nblk - jt : OUTER_BLOCKS);
                const int reserve = (s + 1 < nsteps)
                    ? pick_lookahead_sms(c->num_sms, tilesB, nq1, Np - (jt + 1) * NB) : 0;
                launch_syrk_packed(f->L, k0, Pt[set], nq, jA, nblk, rank, world, s1, reserve);
            }
            int64_t tiles = syrk_packed_tiles(nblk, k0, jt, nblk, rank, world);
            if (tiles > 0) { flops += (double)tiles * 2.0 * NB * NB * ((double)nq * NB); nlaunch++; }
        }
        SB_CUDA(cudaEventRecord(ev_t1[s], s1));
    }
    SB_TRY(finish_two_streams(c, R, comm_ev, chain_ev));
    if (c->fine_timing) {
        for (int64_t s = 0; s < nsteps; s++) {
            float ms = 0;
            cudaEventElapsedTime(&ms, ev_t0[s], ev_t1[s]);
            c->tm.trailing_ms += ms;
            c->tm.trailing_kernel_ms += ms;
        }
        float ms = 0;
        cudaEventElapsedTime(&ms, e_start, ev_p[0]);
        c->tm.panel_ms += ms;  // only the first, un-hidden panel phase is on the critical path
    }
    c->tm.trailing_flops += flops;
    c->tm.trailing_launches += nlaunch;
    return SB_OK;
}

// Factorisation with the wide panel phase (int8 Ozaki path).  Per outer step s, on the trailing stream:
//   T^A_s | T^B_s part 1 (leaves a few SMs free) | panel solve of step s+1 (whole GPU) | T^B_s part 2 (whole GPU)
// and on the panel stream, under T^B_s part 1: column exchange + diagonal block + inv(L_512) of step s+1.
// Part 1 is sized to the duration of that serial chain, so the SM reservation costs ~ 8 / 132 of the GPU for that long per step.
static int32_t cholesky_wide(sb_ctx* c, sb_factor* f, int world, int rank) {
    const int64_t nblk = f->L.nblk();
    std::vector<CommEv> comm_ev, chain_ev, bulk_ev;
    cudaStream_t s1 = c->stream, s2 = c->stream2;
    const int64_t nsteps = (nblk + OUTER_BLOCKS - 1) / OUTER_BLOCKS;
    std::vector<cudaEvent_t> ev_d(nsteps), ev_a(nsteps), ev_t0(nsteps), ev_t1(nsteps);
    for (int64_t s = 0; s < nsteps; s++) {
        ev_d[s] = c->next_event(); ev_a[s] = c->next_event(); ev_t0[s] = c->next_event(); ev_t1[s] = c->next_event();
    }
    cudaEvent_t e_start = c->next_event();
    SB_CUDA(cudaEventRecord(e_start, s1));
    SB_CUDA(cudaStreamWaitEvent(s2, e_start, 0));
    P2PRun R;
    if (world > 1) SB_TRY(p2p_run_begin(c, f, R, world, rank, s2));
    const int reserve_p1 = LOOKAHEAD_SMS;
    const double chain_us = world > 1 ? 2500.0 : 1200.0;
    const int64_t p1_tiles = (int64_t)(chain_us / 14.5 * (c->num_sms - reserve_p1));   // half-tiles T^B part 1 should last

    auto bulk = [&](int64_t s) -> int32_t {      // panel solve + digit planes of step s, trailing stream
        const int64_t k0 = s * OUTER_BLOCKS;
        const int nq = (int)(nblk - k0 < OUTER_BLOCKS ? nblk - k0 : OUTER_BLOCKS);
        const int set = (int)(s & 1);
        SB_CUDA(cudaStreamWaitEvent(s1, ev_d[s], 0));
        CommEv be{nullptr, nullptr};
        if (c->fine_timing) { be.a = c->next_event(); be.b = c->next_event(); SB_CUDA(cudaEventRecord(be.a, s1)); }
        SB_TRY(wide_bulk_phase(c, f, k0, nq, set, s1));
        if (be.a) { SB_CUDA(cudaEventRecord(be.b, s1)); bulk_ev.push_back(be); }
        return SB_OK;
    };
    auto diag = [&](int64_t s) -> int32_t {      // serial part of step s, panel stream
        const int64_t k0 = s * OUTER_BLOCKS;
        const int nq = (int)(nblk - k0 < OUTER_BLOCKS ? nblk - k0 : OUTER_BLOCKS);
        CommEv ch{nullptr, nullptr};
        if (c->fine_timing) { ch.a = c->next_event(); ch.b = c->next_event(); SB_CUDA(cudaEventRecord(ch.a, s2)); }
        SB_TRY(wide_diag_phase(c, f, k0, nq, rank, world, s2, &comm_ev, &R));
        SB_CUDA(cudaEventRecord(ev_d[s], s2));
        if (ch.a) { SB_CUDA(cudaEventRecord(ch.b, s2)); chain_ev.push_back(ch); }
        return SB_OK;
    };
    SB_TRY(diag(0));
    SB_TRY(bulk(0));
    double flops = 0;
    int64_t nlaunch = 0;
    for (int64_t s = 0; s < nsteps; s++) {
        const int64_t k0 = s * OUTER_BLOCKS;
        const int nq = (int)(nblk - k0 < OUTER_BLOCKS ? nblk - k0 : OUTER_BLOCKS);
        const int set = (int)(s & 1);
        const int64_t jt = k0 + nq;
        SB_CUDA(cudaEventRecord(ev_t0[s], s1));
        if (jt < nblk) {
            const int64_t jA = jt + OUTER_BLOCKS < nblk ? jt + OUTER_BLOCKS : nblk;
            auto trailing = [&](int64_t jlo, int64_t jhi, int reserve, int64_t lo, int64_t hi) -> int32_t {
                if (launch_syrk_ozaki(f->L, k0, nq, jlo, jhi, rank, world, &f->oz_maps[set], f->oz_scale[set],
                                      s1, reserve, lo, hi) != 0) {
                    sb::set_error("int8 Ozaki trailing kernel could not be launched");
                    return SB_ERR_CUDA;
                }
                return SB_OK;
            };
            SB_TRY(trailing(jt, jA, 0, 0, 0));                     // T^A: the next step's block columns
            SB_CUDA(cudaEventRecord(ev_a[s], s1));
            const bool next = s + 1 < nsteps;
            if (next) {
                SB_CUDA(cudaStreamWaitEvent(s2, ev_a[s], 0));
                SB_TRY(diag(s + 1));
            }
            const int64_t tilesB = jA < nblk ? 2 * syrk_packed_tiles(nblk, k0, jA, nblk, rank, world) : 0;
            const int64_t n1 = next ? (tilesB < p1_tiles + 2 * c->num_sms ? tilesB : p1_tiles) : tilesB;
            if (n1 > 0) SB_TRY(trailing(jA, nblk, next ? reserve_p1 : 0, 0, n1));          // T^B part 1
            if (next) SB_TRY(bulk(s + 1));
            if (tilesB > n1) SB_TRY(trailing(jA, nblk, 0, n1, tilesB));                      // T^B part 2
            const int64_t tiles = syrk_packed_tiles(nblk, k0, jt, nblk, rank, world);
            if (tiles > 0) { flops += (double)tiles * 2.0 * NB * NB * ((double)nq * NB); nlaunch++; }
        }
        SB_CUDA(cudaEventRecord(ev_t1[s], s1));
    }
    SB_TRY(finish_two_streams(c, R, comm_ev, chain_ev));
    if (c->fine_timing) {
        double tr = 0, bk = 0;
        for (int64_t s = 0; s < nsteps; s++) {
            float ms = 0;
            cudaEventElapsedTime(&ms, ev_t0[s], ev_t1[s]);
            tr += ms;
        }
        for (size_t i = 0; i < bulk_ev.size(); i++) {
            float ms = 0;
            cudaEventElapsedTime(&ms, bulk_ev[i].a, bulk_ev[i].b);
            if (i > 0) bk += ms;               // the first panel solve lies before ev_t0[0]
            c->tm.panel_ms += ms;              // panel solves are on the critical path (whole GPU)
        }
        c->tm.trailing_ms += tr - bk;
        c->tm.trailing_kernel_ms += tr - bk;
        float ms = 0;
        cudaEventElapsedTime(&ms, e_start, ev_d[0]);
        c->tm.panel_ms += ms;                  // the first serial phase is not hidden
    }
    c->tm.trailing_flops += flops;
    c->tm.trailing_launches += nlaunch;
    c->tm.trailing_int8_ops += 28.0 * flops;
    return SB_OK;
}

static int32_t sync_info(sb_ctx* c, sb_factor* f);

int32_t cholesky_packed(sb_ctx* c, sb_factor* f, bool force_local = false) {
    const int64_t nblk = f->L.nblk();
    const int world = force_local ? 1 : c->world, rank = force_local ? 0 : c->rank;
    // Overlapping the panel chain with the trailing update (two streams) pays for the int8 Ozaki path, and on
    // several GPUs, where the chain includes the panel exchange.  With the DMMA trailing kernel on ONE GPU the
    // 8 SMs the look-ahead reserves cost about as much as the hidden panel chain saves: the serial driver below.
    // int8 Ozaki (f->oz: nblk > 2 * OUTER_BLOCKS) uses the wide panel phase, which on several GPUs needs the
    // IPC-mapped arena; without it the DMMA look-ahead factors (P2P exchange or NCCL broadcast).
    if (world == 1 ? f->oz : nblk > OUTER_BLOCKS) {
        if (world > 1) SB_TRY(p2p_ensure(c, f->Np));
        if (f->oz && (world == 1 || c->p2p.state == 1)) SB_TRY(cholesky_wide(c, f, world, rank));
        else SB_TRY(cholesky_lookahead(c, f, world, rank));
        if (world > 1) {
            SB_TRY(sync_info(c, f));
            SB_CUDA(cudaStreamSynchronize(c->stream));  // callers read info / logdet with blocking copies
        }
        return SB_OK;
    }
    const int64_t Np = f->Np;
    cudaStream_t st = c->stream;
    const bool ft = c->fine_timing;
    std::vector<cudaEvent_t> ev;  // per outer step: t0, after panel work, after comm, after trailing ...
    auto mark = [&]() {
        if (ft) {
            cudaEvent_t e = c->next_event();
            cudaEventRecord(e, st);
            ev.push_back(e);
        }
    };
    std::vector<int> evkind;  // kind of the interval ENDING at event i: 0 panel, 1 comm, 2 trailing(big), 3 start
    auto markk = [&](int kind) { if (ft) { mark(); evkind.push_back(kind); } };
    std::vector<CommEv> comm_ev;
    double flops = 0;
    int64_t nlaunch = 0;
    // the OUTER_BLOCKS panels of an outer step, each in TILED layout (gemm_nt.cu); row block 0 <->
    // block row k0+1, panel q starts at row block q
    const double* Pt[OUTER_BLOCKS];
    double* Pw[OUTER_BLOCKS];
    for (int q = 0; q < OUTER_BLOCKS; q++) Pt[q] = Pw[q] = f->panel + (int64_t)q * tiled_panel_elems(Np);
    for (int64_t k0 = 0; k0 < nblk; k0 += OUTER_BLOCKS) {
        const int nq = (int)(nblk - k0 < OUTER_BLOCKS ? nblk - k0 : OUTER_BLOCKS);
        for (int q = 0; q < nq; q++) {   // one panel at a time: the panel work, exchange and untile are timed apart
            markk(3);
            SB_TRY(panel_phase(c, f, k0, q, q + 1, Pw, Pt, rank, world, st, &comm_ev));
            if (ft) {   // the interval ending before the exchange is panel work, the exchange itself comm
                ev.push_back(comm_ev.back().a); evkind.push_back(0);
                ev.push_back(comm_ev.back().b); evkind.push_back(1);
            }
        }
        const int64_t jt = k0 + nq;  // first trailing block column
        if (jt < nblk) {
            int64_t tiles = syrk_packed_tiles(nblk, k0, jt, nblk, rank, world);
            markk(0);
            launch_syrk_packed(f->L, k0, Pt, nq, jt, nblk, rank, world, st);
            markk(2);
            if (tiles > 0) {
                flops += (double)tiles * 2.0 * NB * NB * ((double)nq * NB);
                nlaunch++;
            }
        }
    }
    if (world > 1) SB_TRY(sync_info(c, f));
    SB_CUDA(cudaGetLastError());
    SB_CUDA(cudaStreamSynchronize(st));
    if (ft) {
        for (size_t i = 1; i < ev.size(); i++) {
            if (evkind[i] == 3) continue;
            float ms = 0;
            cudaEventElapsedTime(&ms, ev[i - 1], ev[i]);
            if (evkind[i] == 0) c->tm.panel_ms += ms;
            else if (evkind[i] == 1) c->tm.comm_ms += ms;
            else { c->tm.trailing_ms += ms; c->tm.trailing_kernel_ms += ms; }
        }
    }
    c->tm.trailing_flops += flops;
    c->tm.trailing_launches += nlaunch;
    return SB_OK;
}

__global__ void vec_differs_kernel(const double* a, const double* b, int64_t n, int* flag) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n && __double_as_longlong(a[i]) != __double_as_longlong(b[i])) *flag = 1;
}

// info = first failing pivot over all ranks (0 = ok): min over ranks of (info ? info : INT64_MAX),
// mapped on the device -- one tiny all-reduce, no host round trip.
__global__ void info_map_kernel(long long* info, int back) {
    const long long big = 0x7fffffffffffffffLL;
    if (back) { if (*info == big) *info = 0; }
    else      { if (*info == 0) *info = big; }
}

static int32_t sync_info(sb_ctx* c, sb_factor* f) {
    cudaStream_t st = c->stream;
    info_map_kernel<<<1, 1, 0, st>>>(f->info_dev, 0);
    SB_NCCL(nccl_dl::AllReduce(f->info_dev, f->info_dev, 1, ncclInt64, ncclMin, c->comm, st));
    info_map_kernel<<<1, 1, 0, st>>>(f->info_dev, 1);
    g_launch_count += 2;
    SB_CUDA(cudaGetLastError());
    return SB_OK;
}

// forward sweep  b <- L^{-1} b  for S right-hand sides (b: Np x S, ld Np)
void forward_solve(sb_ctx* c, sb_factor* f, double* b, int S) {
    for (int s0 = 0; s0 < S; s0 += 8) {
        int s = S - s0 < 8 ? S - s0 : 8;
        launch_sweep(f->L, f->invL, b + (int64_t)s0 * f->Np, s, false, f->sweep_flags, c->num_sms, c->stream);
    }
}

// backward sweep  b <- L^{-T} b
void backward_solve(sb_ctx* c, sb_factor* f, double* b, int S) {
    for (int s0 = 0; s0 < S; s0 += 8) {
        int s = S - s0 < 8 ? S - s0 : 8;
        launch_sweep(f->L, f->invL, b + (int64_t)s0 * f->Np, s, true, f->sweep_flags, c->num_sms, c->stream);
    }
}

// upload an N x S column-major host/device matrix into a zero-padded Np x S device buffer
int32_t upload_padded(sb_ctx* c, const void* src, int64_t N, int64_t Np, int S, double* dst) {
    SB_CUDA(cudaMemsetAsync(dst, 0, sizeof(double) * Np * S, c->stream));
    SB_CUDA(cudaMemcpy2DAsync(dst, Np * sizeof(double), src, N * sizeof(double), N * sizeof(double), S,
                              cudaMemcpyDefault, c->stream));
    return SB_OK;
}

}  // namespace

extern "C" {

int32_t sb_abi_version(void) { return SB_ABI_VERSION; }
const char* sb_last_error(void) { return sb::g_err.c_str(); }

int32_t sb_ctx_create(int32_t device, sb_ctx** out) {
    SB_CHECK(out != nullptr, "null out");
    int ndev = 0;
    SB_CUDA(cudaGetDeviceCount(&ndev));
    SB_CHECK(device >= 0 && device < ndev, "no such CUDA device");
    SB_CUDA(cudaSetDevice(device));
    cudaDeviceProp prop;
    SB_CUDA(cudaGetDeviceProperties(&prop, device));
    if (prop.major != 9 || prop.minor != 0) {   // the cubin is sm_90a only (wgmma / setmaxnreg have no later-arch form)
        sb::set_error("libstheno_b200 is built for sm_90a (H100) only; found sm_" +
                      std::to_string(prop.major) + std::to_string(prop.minor));
        return SB_ERR_UNSUPPORTED;
    }
    sb_ctx* c = new sb_ctx();
    c->device = device;
    SB_CUDA(cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking));
    {   // the panel stream outranks the trailing-update stream: its kernels sit on the critical path
        int prio_lo = 0, prio_hi = 0;
        SB_CUDA(cudaDeviceGetStreamPriorityRange(&prio_lo, &prio_hi));
        SB_CUDA(cudaStreamCreateWithPriority(&c->stream2, cudaStreamNonBlocking, prio_hi));
        for (int i = 0; i < 4; i++) SB_CUDA(cudaStreamCreateWithPriority(&c->xstream[i], cudaStreamNonBlocking, prio_hi));
    }
    const char* ft = getenv("SB_FINE_TIMING");
    if (ft && ft[0] == '0') c->fine_timing = false;
    SB_CUDA(cudaDeviceGetAttribute(&c->num_sms, cudaDevAttrMultiProcessorCount, device));
    const char* tr = getenv("SB_TRAILING");   // "dmma" | "ozaki"
    if (tr && !strcmp(tr, "dmma")) c->trailing_mode = 0;
    if (tr && !strcmp(tr, "ozaki")) c->trailing_mode = 1;
    *out = c;
    return SB_OK;
}

int32_t sb_nccl_unique_id(void* id128) {
    SB_CHECK(id128 != nullptr, "null id");
    static_assert(sizeof(ncclUniqueId) == 128, "ncclUniqueId size");
    ncclUniqueId id;
    if (!nccl_dl::load()) return SB_ERR_NCCL;
    SB_NCCL(nccl_dl::GetUniqueId(&id));
    memcpy(id128, &id, 128);
    return SB_OK;
}

int32_t sb_ctx_create_dist(int32_t device, int32_t rank, int32_t world, const void* nccl_id128,
                           sb_ctx** out) {
    SB_CHECK(world >= 1 && rank >= 0 && rank < world, "bad rank/world");
    SB_TRY(sb_ctx_create(device, out));
    sb_ctx* c = *out;
    c->rank = rank;
    c->world = world;
    if (world > 1) {
        SB_CHECK(nccl_id128 != nullptr, "null nccl id");
        ncclUniqueId id;
        memcpy(&id, nccl_id128, 128);
        if (!nccl_dl::load()) return SB_ERR_NCCL;
        SB_NCCL(nccl_dl::CommInitRank(&c->comm, world, id, rank));
    }
    return SB_OK;
}

int32_t sb_ctx_destroy(sb_ctx* c) {
    if (!c) return SB_OK;
    cudaSetDevice(c->device);
    if (c->p2p.arena) {   // collective, like the communicator: no peer may still be reading this arena
        cudaStreamSynchronize(c->stream);
        cudaStreamSynchronize(c->stream2);
        if (c->comm && c->p2p.xch) nccl_barrier(c, static_cast<char*>(c->p2p.xch) + 8 * sizeof(cudaIpcMemHandle_t));
        p2p_close(c);
    }
    if (c->p2p.xch) cudaFree(c->p2p.xch);
    if (c->comm) nccl_dl::CommDestroy(c->comm);
    c->pool_trim();
    for (auto e : c->ev) cudaEventDestroy(e);
    for (auto e : c->marks) if (e) cudaEventDestroy(e);
    if (c->stream) cudaStreamDestroy(c->stream);
    if (c->stream2) cudaStreamDestroy(c->stream2);
    for (int i = 0; i < 4; i++) if (c->xstream[i]) cudaStreamDestroy(c->xstream[i]);
    delete c;
    return SB_OK;
}

int32_t sb_ctx_timings(sb_ctx* c, sb_timings* out, int32_t reset) {
    SB_CHECK(c != nullptr, "null ctx");
    if (out) *out = c->tm;
    if (reset) c->tm = sb_timings{};
    return SB_OK;
}

int32_t sb_ctx_set_option(sb_ctx* c, const char* key, int64_t value) {
    SB_CHECK(c && key, "null argument");
    if (!strcmp(key, "trailing")) {
        SB_CHECK(value == 0 || value == 1, "trailing: 0 = fp64 DMMA, 1 = int8 Ozaki");
        c->trailing_mode = (int)value;
        return SB_OK;
    }
    if (!strcmp(key, "fine_timing")) { c->fine_timing = value != 0; return SB_OK; }
    sb::set_error(std::string("unknown option ") + key);
    return SB_ERR_INVALID;
}

int32_t sb_owner_of_block(int64_t J, int32_t world) { return world > 0 ? (int32_t)(J % world) : 0; }

int64_t sb_owned_trailing_tiles(int64_t nblk, int64_t k, int32_t rank, int32_t world) {
    if (world < 1 || rank < 0 || rank >= world) return -1;
    return syrk_packed_tiles(nblk, k, k + 1, nblk, rank, world);
}

int32_t sb_row_chunk(int64_t ns, int32_t rank, int32_t world, int64_t* lo, int64_t* hi) {
    SB_CHECK(lo && hi && world >= 1 && rank >= 0 && rank < world && ns >= 0, "bad argument");
    int64_t chunk = (ns + world - 1) / world;
    *lo = rank * chunk < ns ? rank * chunk : ns;
    *hi = *lo + chunk < ns ? *lo + chunk : ns;
    return SB_OK;
}

int32_t sb_ctx_mark(sb_ctx* c, int32_t slot) {
    SB_CHECK(c && slot >= 0 && slot < 8, "bad mark slot");
    cudaSetDevice(c->device);
    if (!c->marks[slot]) SB_CUDA(cudaEventCreate(&c->marks[slot]));
    SB_CUDA(cudaEventRecord(c->marks[slot], c->stream));
    return SB_OK;
}

int32_t sb_ctx_elapsed_ms(sb_ctx* c, int32_t a, int32_t b, double* ms) {
    SB_CHECK(c && ms && a >= 0 && a < 8 && b >= 0 && b < 8 && c->marks[a] && c->marks[b], "bad mark slot");
    SB_CUDA(cudaEventSynchronize(c->marks[b]));
    float f = 0;
    SB_CUDA(cudaEventElapsedTime(&f, c->marks[a], c->marks[b]));
    *ms = f;
    return SB_OK;
}

int32_t sb_cov_dense(sb_ctx* c, const sb_covspec* spec, void* K_out) {
    SB_CHECK(c && spec && K_out, "null argument");
    begin_call(c);
    int64_t before = g_launch_count;
    DevSpec ds(c);
    SB_TRY(ds.build(spec, c->stream, false));
    DevBuf K(c);
    size_t bytes = (size_t)ds.nrows * ds.ncols * sizeof(double);
    SB_TRY(K.alloc(bytes));
    SB_CUDA(cudaMemsetAsync(K.p, 0, bytes, c->stream));
    PhaseTimer t(c, &c->tm.assemble_ms);
    SB_TRY(assemble_dense(c, ds, K.d(), ds.nrows));
    t.stop();
    SB_CUDA(cudaMemcpyAsync(K_out, K.p, bytes, cudaMemcpyDefault, c->stream));
    SB_CUDA(cudaStreamSynchronize(c->stream));
    t.collect();
    count_launches(c, before);
    return SB_OK;
}

int32_t sb_cov_diag(sb_ctx* c, const sb_covspec* spec, void* out) {
    SB_CHECK(c && spec && out, "null argument");
    begin_call(c);
    int64_t before = g_launch_count;
    DevSpec ds(c);
    SB_TRY(ds.build(spec, c->stream, true));
    DevBuf v(c);
    SB_TRY(v.alloc(ds.nrows * sizeof(double)));
    SB_CUDA(cudaMemsetAsync(v.p, 0, ds.nrows * sizeof(double), c->stream));
    SB_TRY(assemble_diag(c, ds, v.d()));
    SB_CUDA(cudaMemcpyAsync(out, v.p, ds.nrows * sizeof(double), cudaMemcpyDefault, c->stream));
    SB_CUDA(cudaStreamSynchronize(c->stream));
    count_launches(c, before);
    return SB_OK;
}

int32_t sb_factor_destroy(sb_factor* f) {
    if (!f) return SB_OK;
    cudaSetDevice(f->ctx->device);
    sb_ctx* c = f->ctx;
    c->pool_release(f->L.base, f->bytes_L);
    c->pool_release(f->invL, f->bytes_invL);
    c->pool_release(f->ldiag, f->bytes_ldiag);
    c->pool_release(f->logdet_blk, f->bytes_ld);
    c->pool_release(f->info_dev, 8);
    c->pool_release(f->panel, f->bytes_panel);
    c->pool_release(f->alpha, f->bytes_alpha);
    for (int i = 0; i < 2; i++) {
        c->pool_release(f->oz_planes[i], f->bytes_oz_planes);
        c->pool_release(f->oz_scale[i], (size_t)f->Np * sizeof(double));
        c->pool_release(f->oz_expo[i], (size_t)f->Np * sizeof(int));
    }
    {
        constexpr int64_t WD = (int64_t)OUTER_BLOCKS * NB;
        c->pool_release(f->wide_D, (size_t)2 * 2 * WD * WD * sizeof(double));
        c->pool_release(f->wide_W, (size_t)WD * WD * sizeof(double));
        c->pool_release(f->wide_wp, oz_planes_bytes(WD));
        c->pool_release(f->wide_wscale, (size_t)WD * sizeof(double));
        c->pool_release(f->wide_wexpo, (size_t)WD * sizeof(int));
    }
    c->pool_release(f->sweep_flags, (size_t)2 * (f->Np / NB) * sizeof(unsigned));
    c->pool_release(f->vcache, (size_t)2 * f->Np * sizeof(double));
    c->pool_release(f->vcache_flag, sizeof(int));
    delete f;
    return SB_OK;
}

static int32_t factor_create_impl(sb_ctx* c, const sb_covspec* spec, const sb_noise* noise, sb_factor** out,
                                  int64_t* info, bool force_local);

int32_t sb_factor_create(sb_ctx* c, const sb_covspec* spec, const sb_noise* noise, sb_factor** out,
                         int64_t* info) {
    return factor_create_impl(c, spec, noise, out, info, false);
}

// allocate the buffers of a factor of order N from the context pool
static int32_t factor_alloc(sb_ctx* c, int64_t N, sb_factor** out) {
    sb_factor* f = new sb_factor();
    f->ctx = c;
    f->N = N;
    f->Np = round_up(N, NB);
    f->L.Np = f->Np;
    const int64_t nblk = f->L.nblk();
    f->bytes_L = (size_t)f->L.total() * sizeof(double);
    f->bytes_invL = (size_t)nblk * NB * NB * sizeof(double);
    f->bytes_ld = (size_t)nblk * sizeof(double);
    f->bytes_panel = (size_t)2 * OUTER_BLOCKS * tiled_panel_elems(f->Np) * sizeof(double);
    f->bytes_alpha = (size_t)f->Np * sizeof(double);
    f->bytes_ldiag = c->world > 1 ? f->bytes_invL : 0;
    cudaError_t e = cudaSuccess;
    if (e == cudaSuccess) e = c->pool_alloc((void**)&f->L.base, f->bytes_L);
    if (e == cudaSuccess) e = c->pool_alloc((void**)&f->invL, f->bytes_invL);
    if (e == cudaSuccess && f->bytes_ldiag) e = c->pool_alloc((void**)&f->ldiag, f->bytes_ldiag);
    if (e == cudaSuccess) e = c->pool_alloc((void**)&f->logdet_blk, f->bytes_ld);
    if (e == cudaSuccess) e = c->pool_alloc((void**)&f->info_dev, 8);
    if (e == cudaSuccess) e = c->pool_alloc((void**)&f->panel, f->bytes_panel);
    if (e == cudaSuccess) e = c->pool_alloc((void**)&f->alpha, f->bytes_alpha);
    if (e == cudaSuccess) e = c->pool_alloc((void**)&f->sweep_flags, (size_t)2 * nblk * sizeof(unsigned));
    if (e == cudaSuccess) e = c->pool_alloc((void**)&f->vcache, (size_t)2 * f->Np * sizeof(double));
    if (e == cudaSuccess) e = c->pool_alloc((void**)&f->vcache_flag, sizeof(int));
    if (e == cudaSuccess) e = cudaMemsetAsync(f->info_dev, 0, sizeof(long long), c->stream);
    if (e == cudaSuccess) e = cudaMemsetAsync(f->logdet_blk, 0, nblk * sizeof(double), c->stream);
    // int8 Ozaki path: worth it (and exercised) once the trailing matrix has a few hundred tiles
    if (e == cudaSuccess && c->trailing_mode == 1 && nblk > 2 * OUTER_BLOCKS) {
        f->bytes_oz_planes = oz_planes_bytes(f->Np);
        for (int i = 0; i < 2 && e == cudaSuccess; i++) {
            e = c->pool_alloc((void**)&f->oz_planes[i], f->bytes_oz_planes);
            if (e == cudaSuccess) e = c->pool_alloc((void**)&f->oz_scale[i], (size_t)f->Np * sizeof(double));
            if (e == cudaSuccess) e = c->pool_alloc((void**)&f->oz_expo[i], (size_t)f->Np * sizeof(int));
        }
        constexpr int64_t WD = (int64_t)OUTER_BLOCKS * NB;
        if (e == cudaSuccess) e = c->pool_alloc((void**)&f->wide_D, (size_t)2 * 2 * WD * WD * sizeof(double));
        if (e == cudaSuccess) e = c->pool_alloc((void**)&f->wide_W, (size_t)WD * WD * sizeof(double));
        if (e == cudaSuccess) e = c->pool_alloc((void**)&f->wide_wp, oz_planes_bytes(WD));
        if (e == cudaSuccess) e = c->pool_alloc((void**)&f->wide_wscale, (size_t)WD * sizeof(double));
        if (e == cudaSuccess) e = c->pool_alloc((void**)&f->wide_wexpo, (size_t)WD * sizeof(int));
        if (e == cudaSuccess) {
            if (oz_make_maps(f->oz_planes[0], f->Np, &f->oz_maps[0]) != 0 ||
                oz_make_maps(f->oz_planes[1], f->Np, &f->oz_maps[1]) != 0 ||
                oz_make_maps(f->wide_wp, WD, &f->wide_wmaps) != 0) {
                sb_factor_destroy(f);
                sb::set_error("cuTensorMapEncodeTiled failed for the int8 digit planes");
                return SB_ERR_CUDA;
            }
            f->oz = true;
        }
    }
    if (e != cudaSuccess) {
        sb_factor_destroy(f);
        return sb::cuda_fail(e, "factor_alloc", __FILE__, __LINE__);
    }
    *out = f;
    return SB_OK;
}

// run the Cholesky on an assembled packed matrix and collect info / logdet
static int32_t factor_finish(sb_ctx* c, sb_factor* f, int64_t* info, bool force_local) {
    SB_TRY(cholesky_packed(c, f, force_local));
    const int64_t nblk = f->L.nblk();
    long long h_info = 0;
    std::vector<double> ld(nblk);
    SB_CUDA(cudaMemcpy(&h_info, f->info_dev, sizeof(long long), cudaMemcpyDeviceToHost));
    SB_CUDA(cudaMemcpy(ld.data(), f->logdet_blk, nblk * sizeof(double), cudaMemcpyDeviceToHost));
    if (h_info != 0) {
        if (info) *info = (int64_t)h_info;
        sb::set_error("matrix is not positive definite; Cholesky factorization failed at pivot " +
                      std::to_string(h_info));
        return SB_ERR_NOT_POSDEF;
    }
    double sum = 0.0;
    for (double v : ld) sum += v;
    f->logdet = sum;
    return SB_OK;
}

static int32_t factor_create_impl(sb_ctx* c, const sb_covspec* spec, const sb_noise* noise, sb_factor** out,
                                  int64_t* info, bool force_local) {
    SB_CHECK(c && spec && out, "null argument");
    SB_CHECK(spec->symmetric == 1 && spec->nrows == spec->ncols, "factor needs a symmetric square spec");
    SB_CHECK(spec->nrows > 0, "empty matrix");
    begin_call(c);
    int64_t before = g_launch_count;
    if (info) *info = 0;
    *out = nullptr;
    cudaEvent_t t0 = c->next_event(), t1 = c->next_event();
    cudaEventRecord(t0, c->stream);

    DevSpec ds(c);
    SB_TRY(ds.build(spec, c->stream, false));
    sb_factor* f = nullptr;
    SB_TRY(factor_alloc(c, spec->nrows, &f));
    auto fail = [&](int32_t s) {
        sb_factor_destroy(f);
        return s;
    };
#define SB_CUDA_F(call)                                                        \
    do {                                                                       \
        cudaError_t _e = (call);                                               \
        if (_e != cudaSuccess) return fail(sb::cuda_fail(_e, #call, __FILE__, __LINE__)); \
    } while (0)
    const int a_rank = force_local ? 0 : c->rank, a_world = force_local ? 1 : c->world;
    DevBuf nd(c), ndense(c);
    const double* noise_diag = nullptr;
    double sigma2 = 0.0;
    if (noise && noise->dense) {
        if (ndense.alloc((size_t)f->N * f->N * sizeof(double)) != SB_OK) return fail(SB_ERR_NOMEM);
        SB_CUDA_F(cudaMemcpyAsync(ndense.p, noise->dense, (size_t)f->N * f->N * sizeof(double), cudaMemcpyDefault, c->stream));
    } else if (noise) {
        sigma2 = noise->sigma2;
        if (noise->diag) {
            if (nd.alloc(f->N * sizeof(double)) != SB_OK) return fail(SB_ERR_NOMEM);
            SB_CUDA_F(cudaMemcpyAsync(nd.p, noise->diag, f->N * sizeof(double), cudaMemcpyDefault, c->stream));
            noise_diag = nd.d();
        }
    }
    {
        PhaseTimer t(c, &c->tm.assemble_ms);
        // multi-GPU: every rank assembles only the block columns it owns under the Cholesky
        // distribution (the kernel skips foreign tiles); foreign columns arrive as broadcast panels
        for (auto& b : ds.blocks) launch_assemble_packed(b, f->L, f->N, sigma2, noise_diag, c->stream, a_rank, a_world);
        if (ndense.p) launch_add_dense_lower(f->L, ndense.d(), f->N, f->N, c->stream);
        launch_fill_padding(f->L, f->N, c->stream);
        t.stop();
        SB_CUDA_F(cudaGetLastError());
        int32_t s = factor_finish(c, f, info, force_local);
        if (s != SB_OK) return fail(s);
        t.collect();
    }
    cudaEventRecord(t1, c->stream);
    cudaEventSynchronize(t1);
    float ms = 0;
    cudaEventElapsedTime(&ms, t0, t1);
    c->tm.total_ms += ms;
    count_launches(c, before);
    *out = f;
    return SB_OK;
#undef SB_CUDA_F
}

// ---- factor checkpoint: export / import (SURVEY 8f.4) -------------------------------------------
// Blob = header | packed L (Np(Np+NB)/2 doubles) | inverses of the diagonal blocks | alpha (Np).
// PosteriorGP in the reference is a plain struct (alpha, C, x, delta) that Julia can serialise; the
// device-resident handle gets the same ability here.
struct FactorBlobHeader {
    char magic[8];        // "SBFACT01"
    int64_t N, Np;
    double logdet;
    int64_t has_alpha;
    int64_t reserved[3];
};

int32_t sb_factor_export_size(sb_ctx* c, sb_factor* f, int64_t* nbytes) {
    SB_CHECK(c && f && nbytes, "null argument");
    *nbytes = (int64_t)sizeof(FactorBlobHeader) + (int64_t)f->bytes_L + (int64_t)f->bytes_invL + (int64_t)f->bytes_alpha;
    return SB_OK;
}

int32_t sb_factor_export(sb_ctx* c, sb_factor* f, void* blob, int64_t nbytes) {
    SB_CHECK(c && f && blob, "null argument");
    int64_t need = 0;
    sb_factor_export_size(c, f, &need);
    SB_CHECK(nbytes >= need, "export buffer too small (see sb_factor_export_size)");
    begin_call(c);
    FactorBlobHeader h{};
    memcpy(h.magic, "SBFACT01", 8);
    h.N = f->N; h.Np = f->Np; h.logdet = f->logdet; h.has_alpha = f->has_alpha ? 1 : 0;
    char* p = static_cast<char*>(blob);
    SB_CUDA(cudaMemcpyAsync(p, &h, sizeof(h), cudaMemcpyDefault, c->stream));
    p += sizeof(h);
    SB_CUDA(cudaMemcpyAsync(p, f->L.base, f->bytes_L, cudaMemcpyDefault, c->stream));
    p += f->bytes_L;
    SB_CUDA(cudaMemcpyAsync(p, f->invL, f->bytes_invL, cudaMemcpyDefault, c->stream));
    p += f->bytes_invL;
    SB_CUDA(cudaMemcpyAsync(p, f->alpha, f->bytes_alpha, cudaMemcpyDefault, c->stream));
    SB_CUDA(cudaStreamSynchronize(c->stream));
    return SB_OK;
}

int32_t sb_factor_import(sb_ctx* c, const void* blob, int64_t nbytes, sb_factor** out) {
    SB_CHECK(c && blob && out, "null argument");
    SB_CHECK(nbytes >= (int64_t)sizeof(FactorBlobHeader), "blob too small");
    begin_call(c);
    *out = nullptr;
    FactorBlobHeader h{};
    SB_CUDA(cudaMemcpy(&h, blob, sizeof(h), cudaMemcpyDefault));
    SB_CHECK(memcmp(h.magic, "SBFACT01", 8) == 0, "not a libstheno_b200 factor blob");
    SB_CHECK(h.N > 0 && h.Np == round_up(h.N, NB), "corrupt factor blob header");
    sb_factor* f = nullptr;
    SB_TRY(factor_alloc(c, h.N, &f));
    const int64_t need = (int64_t)sizeof(h) + (int64_t)f->bytes_L + (int64_t)f->bytes_invL + (int64_t)f->bytes_alpha;
    if (nbytes < need) {
        sb_factor_destroy(f);
        sb::set_error("factor blob truncated");
        return SB_ERR_INVALID;
    }
    const char* p = static_cast<const char*>(blob) + sizeof(h);
    cudaError_t e = cudaMemcpyAsync(f->L.base, p, f->bytes_L, cudaMemcpyDefault, c->stream);
    p += f->bytes_L;
    if (e == cudaSuccess) e = cudaMemcpyAsync(f->invL, p, f->bytes_invL, cudaMemcpyDefault, c->stream);
    p += f->bytes_invL;
    if (e == cudaSuccess) e = cudaMemcpyAsync(f->alpha, p, f->bytes_alpha, cudaMemcpyDefault, c->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(c->stream);
    if (e != cudaSuccess) {
        sb_factor_destroy(f);
        return sb::cuda_fail(e, "sb_factor_import", __FILE__, __LINE__);
    }
    f->logdet = h.logdet;
    f->has_alpha = h.has_alpha != 0;
    *out = f;
    return SB_OK;
}

int32_t sb_factor_logdet(sb_ctx*, sb_factor* f, double* out) {
    SB_CHECK(f && out, "null argument");
    *out = f->logdet;
    return SB_OK;
}

int32_t sb_logpdf(sb_ctx* c, sb_factor* f, const void* delta, int32_t S, double* out) {
    SB_CHECK(c && f && delta && out && S >= 1, "bad argument");
    begin_call(c);
    int64_t before = g_launch_count;
    DevBuf b(c), q(c);
    SB_TRY(b.alloc((size_t)f->Np * S * sizeof(double)));
    SB_TRY(q.alloc(S * sizeof(double)));
    SB_TRY(upload_padded(c, delta, f->N, f->Np, S, b.d()));
    PhaseTimer t(c, &c->tm.solve_ms);
    if (S == 1) SB_CUDA(cudaMemcpyAsync(f->vcache, b.p, f->Np * sizeof(double), cudaMemcpyDeviceToDevice, c->stream));
    forward_solve(c, f, b.d(), S);
    if (S == 1) {
        SB_CUDA(cudaMemcpyAsync(f->vcache + f->Np, b.p, f->Np * sizeof(double), cudaMemcpyDeviceToDevice, c->stream));
        f->vcache_valid = true;
    }
    launch_colsumsq(b.d(), f->Np, f->Np, S, q.d(), c->stream);
    t.stop();
    SB_CUDA(cudaGetLastError());
    std::vector<double> hq(S);
    SB_CUDA(cudaMemcpyAsync(hq.data(), q.p, S * sizeof(double), cudaMemcpyDeviceToHost, c->stream));
    SB_CUDA(cudaStreamSynchronize(c->stream));
    t.collect();
    const double log2pi = 1.8378770664093454835606594728112;
    for (int s = 0; s < S; s++) out[s] = -((double)f->N * log2pi + f->logdet + hq[s]) / 2.0;
    count_launches(c, before);
    return SB_OK;
}

int32_t sb_factor_set_data(sb_ctx* c, sb_factor* f, const void* delta) {
    SB_CHECK(c && f && delta, "null argument");
    begin_call(c);
    int64_t before = g_launch_count;
    SB_TRY(upload_padded(c, delta, f->N, f->Np, 1, f->alpha));
    PhaseTimer t(c, &c->tm.solve_ms);
    bool reuse = false;
    if (f->vcache_valid) {   // same delta as the last logpdf call on this handle?  (bitwise, on device)
        int h = 1;
        SB_CUDA(cudaMemsetAsync(f->vcache_flag, 0, sizeof(int), c->stream));
        vec_differs_kernel<<<(unsigned)((f->Np + 255) / 256), 256, 0, c->stream>>>(f->alpha, f->vcache, f->Np, f->vcache_flag);
        g_launch_count++;
        SB_CUDA(cudaMemcpyAsync(&h, f->vcache_flag, sizeof(int), cudaMemcpyDeviceToHost, c->stream));
        SB_CUDA(cudaStreamSynchronize(c->stream));
        reuse = h == 0;
    }
    if (reuse) SB_CUDA(cudaMemcpyAsync(f->alpha, f->vcache + f->Np, f->Np * sizeof(double), cudaMemcpyDeviceToDevice, c->stream));
    else forward_solve(c, f, f->alpha, 1);
    backward_solve(c, f, f->alpha, 1);
    t.stop();
    SB_CUDA(cudaGetLastError());
    SB_CUDA(cudaStreamSynchronize(c->stream));
    t.collect();
    f->has_alpha = true;
    count_launches(c, before);
    return SB_OK;
}

// posterior(fx, y) is a pure function in the reference (AbstractGPs PosteriorGP holds its own
// alpha): a host object that shares the factor with other posteriors re-installs ITS alpha here
// before predicting.
int32_t sb_factor_set_alpha(sb_ctx* c, sb_factor* f, const void* alpha) {
    SB_CHECK(c && f && alpha, "null argument");
    begin_call(c);
    SB_TRY(upload_padded(c, alpha, f->N, f->Np, 1, f->alpha));
    SB_CUDA(cudaStreamSynchronize(c->stream));
    f->has_alpha = true;
    return SB_OK;
}

int32_t sb_factor_alpha(sb_ctx* c, sb_factor* f, void* alpha_out) {
    SB_CHECK(c && f && alpha_out, "null argument");
    SB_CHECK(f->has_alpha, "sb_factor_set_data has not been called");
    begin_call(c);
    SB_CUDA(cudaMemcpy(alpha_out, f->alpha, f->N * sizeof(double), cudaMemcpyDefault));
    return SB_OK;
}

// workspace of the int8 Ozaki matrix-TRSM sweep: digit planes / scales / tensor maps of the X panels
struct OzSweepWs {
    DevBuf planes, scale, expo;
    OzMaps maps;
    int64_t rows = 0;
    bool ready = false;
    explicit OzSweepWs(sb_ctx* c) : planes(c), scale(c), expo(c) {}
    int32_t init(int64_t rows_p) {
        rows = rows_p;
        SB_TRY(planes.alloc(oz_planes_bytes(rows_p)));
        SB_TRY(scale.alloc(rows_p * sizeof(double)));
        SB_TRY(expo.alloc(rows_p * sizeof(int)));
        if (oz_make_maps(reinterpret_cast<signed char*>(planes.p), rows_p, &maps) != 0) {
            sb::set_error("cuTensorMapEncodeTiled failed for the X digit planes");
            return SB_ERR_CUDA;
        }
        ready = true;
        return SB_OK;
    }
};
constexpr int SWEEP_COLS = OUTER_BLOCKS * NB;  // columns of the Xk workspace (rows_p x 512)

// W <- W L^{-T} (rows_p x Np, ld rows_p): right-looking block forward substitution, tensor-core
// products only.  keep: write the result back into W; acc != null: acc[r] += sum_c result[r,c]^2.
// Xk: rows_p x 512 workspace.  With a int8-Ozaki factor (f->oz) the big update of each outer
// step (4 block columns, K = 512) runs on the int8 Ozaki kernel; the small in-step products stay DMMA.
static int32_t trsm_sweep(sb_ctx* c, sb_factor* f, double* W, int64_t rows_p, double* Xk, bool keep, double* acc,
                          OzSweepWs* ws = nullptr) {
    const int64_t nblk = f->L.nblk(), Np = f->Np;
    if (f->oz && ws && ws->ready) {
        for (int64_t k0 = 0; k0 < nblk; k0 += OUTER_BLOCKS) {
            const int nq = (int)(nblk - k0 < OUTER_BLOCKS ? nblk - k0 : OUTER_BLOCKS);
            double* X[OUTER_BLOCKS];
            for (int q = 0; q < nq; q++) {
                const int64_t kq = k0 + q;
                double* Wq = W + kq * NB * rows_p;
                X[q] = Xk + (int64_t)q * NB * rows_p;
                if (q > 0) {  // bring block column kq up to date with the X panels of this outer step
                    const double* As[OUTER_BLOCKS]; int64_t las[OUTER_BLOCKS];
                    const double* Bs[OUTER_BLOCKS]; int64_t lbs[OUTER_BLOCKS];
                    for (int p = 0; p < q; p++) { As[p] = X[p]; las[p] = rows_p; Bs[p] = f->L.blk(kq, k0 + p); lbs[p] = f->L.ld(k0 + p); }
                    launch_gemm_nt_seg(q, As, las, Bs, lbs, Wq, rows_p, rows_p, NB, -1.0, 1.0, c->stream);
                }
                launch_gemm_nt(Wq, rows_p, f->invL + kq * (int64_t)NB * NB, NB, X[q], rows_p, rows_p, NB, NB, 1.0, 0.0, c->stream);
                if (keep) SB_CUDA(cudaMemcpyAsync(Wq, X[q], (size_t)rows_p * NB * sizeof(double), cudaMemcpyDeviceToDevice, c->stream));
                if (acc) launch_rowsumsq_acc(X[q], rows_p, rows_p, NB, acc, c->stream);
            }
            const int64_t jt = k0 + nq, m = Np - jt * NB;
            if (m <= 0) break;
            OzSrc sx{}, sl{};
            sx.nseg = sl.nseg = nq;
            for (int q = 0; q < nq; q++) {
                sx.base[q] = X[q]; sx.ld[q] = rows_p; sx.rbs[q] = NB;
                sl.base[q] = f->L.blk(jt, k0 + q); sl.ld[q] = f->L.ld(k0 + q); sl.rbs[q] = NB;
            }
            launch_oz_slice(sx, 0, rows_p / NB, 0, ws->rows, ws->scale.d(), reinterpret_cast<int*>(ws->expo.p),
                            reinterpret_cast<signed char*>(ws->planes.p), c->stream);
            launch_oz_slice(sl, 0, m / NB, jt * (int64_t)NB, Np, f->oz_scale[0], f->oz_expo[0], f->oz_planes[0], c->stream);
            if (launch_gemm_ozaki(W + jt * NB * rows_p, rows_p, rows_p, m, nq, &ws->maps, ws->scale.d(), 0, &f->oz_maps[0],
                                  f->oz_scale[0], jt * (int64_t)NB, c->stream) != 0) {
                sb::set_error("int8 Ozaki sweep kernel could not be launched");
                return SB_ERR_CUDA;
            }
        }
        SB_CUDA(cudaGetLastError());
        return SB_OK;
    }
    // DMMA path: two block columns per outer step so the big update runs at K = 256
    double* X0 = Xk;
    double* X1 = Xk + rows_p * NB;
    for (int64_t k0 = 0; k0 < nblk; k0 += 2) {
        const int64_t k1 = k0 + 1;
        double* W0 = W + k0 * NB * rows_p;
        launch_gemm_nt(W0, rows_p, f->invL + k0 * (int64_t)NB * NB, NB, X0, rows_p, rows_p, NB, NB, 1.0, 0.0, c->stream);
        if (keep) SB_CUDA(cudaMemcpyAsync(W0, X0, (size_t)rows_p * NB * sizeof(double), cudaMemcpyDeviceToDevice, c->stream));
        if (acc) launch_rowsumsq_acc(X0, rows_p, rows_p, NB, acc, c->stream);
        if (k1 >= nblk) break;
        double* W1 = W + k1 * NB * rows_p;
        launch_gemm_nt(X0, rows_p, f->L.blk(k1, k0), f->L.ld(k0), W1, rows_p, rows_p, NB, NB, -1.0, 1.0, c->stream);
        launch_gemm_nt(W1, rows_p, f->invL + k1 * (int64_t)NB * NB, NB, X1, rows_p, rows_p, NB, NB, 1.0, 0.0, c->stream);
        if (keep) SB_CUDA(cudaMemcpyAsync(W1, X1, (size_t)rows_p * NB * sizeof(double), cudaMemcpyDeviceToDevice, c->stream));
        if (acc) launch_rowsumsq_acc(X1, rows_p, rows_p, NB, acc, c->stream);
        const int64_t m = Np - (k1 + 1) * NB;
        if (m > 0) {
            const double* As[2] = {X0, X1};
            const int64_t las[2] = {rows_p, rows_p};
            const double* Bs[2] = {f->L.blk(k1 + 1, k0), f->L.blk(k1 + 1, k1)};
            const int64_t lbs[2] = {f->L.ld(k0), f->L.ld(k1)};
            launch_gemm_nt_seg(2, As, las, Bs, lbs, W + (k1 + 1) * NB * rows_p, rows_p, rows_p, m, -1.0, 1.0, c->stream);
        }
    }
    SB_CUDA(cudaGetLastError());
    return SB_OK;
}

// shared body of sb_predict / sb_predict_cov
static int32_t predict_impl(sb_ctx* c, sb_factor* f, const sb_covspec* cross,
                            const sb_covspec* prior, bool full_cov, void* mean_out, void* var_out,
                            void* cov_out, const sb_noise* post_noise = nullptr, sb_factor** fac_out = nullptr,
                            int64_t* info = nullptr) {
    begin_call(c);
    int64_t before = g_launch_count;
    SB_CHECK(cross->ncols == f->N, "cross spec must be N* x N");
    const int64_t Ns_all = cross->nrows;
    if (Ns_all == 0) return SB_OK;
    // multi-GPU: every rank holds the complete factor, so the test points are sharded by rows
    // (contiguous chunks) with no communication until the final all-gather of mean / var.
    const bool shard = c->world > 1 && !full_cov;
    const int64_t chunk = shard ? (Ns_all + c->world - 1) / c->world : Ns_all;
    const int64_t lo = shard ? (c->rank * chunk < Ns_all ? c->rank * chunk : Ns_all) : 0;
    const int64_t hi = shard ? (lo + chunk < Ns_all ? lo + chunk : Ns_all) : Ns_all;
    const int64_t Ns = hi - lo, Nsp = round_up(Ns > 0 ? Ns : 1, NB), Np = f->Np;
    const int64_t nblk = f->L.nblk();
    const bool need_var = var_out != nullptr || full_cov;
    SB_CHECK(!mean_out || f->has_alpha, "posterior mean requested before sb_factor_set_data");
    cudaEvent_t t0 = c->next_event(), t1 = c->next_event();
    cudaEventRecord(t0, c->stream);

    DevSpec dc(c), dp(c);
    SB_TRY(dc.build(cross, c->stream, false));
    if (need_var) {
        SB_CHECK(prior != nullptr, "prior spec required for var/cov");
        SB_CHECK(prior->nrows == Ns_all, "prior spec size mismatch");
        SB_TRY(dp.build(prior, c->stream, !full_cov));
    }
    if (shard) {
        clip_rows(dc, lo, hi, false);
        if (need_var) clip_rows(dp, lo, hi, true);
    }
    DevBuf gath(c);  // [2][world][chunk] gather buffer (mean, var) when sharded
    if (shard) SB_TRY(gath.alloc((size_t)2 * (c->world + 1) * chunk * sizeof(double)));
    double* g_send_m = shard ? gath.d() : nullptr;                       // chunk
    double* g_send_v = shard ? gath.d() + chunk : nullptr;               // chunk
    double* g_recv_m = shard ? gath.d() + 2 * chunk : nullptr;           // world*chunk
    double* g_recv_v = shard ? gath.d() + 2 * chunk + (size_t)c->world * chunk : nullptr;
    if (shard) SB_CUDA(cudaMemsetAsync(gath.p, 0, (size_t)2 * (c->world + 1) * chunk * sizeof(double), c->stream));
    DevBuf W(c), Xk(c), mean(c), acc(c), pd(c);
    SB_TRY(W.alloc((size_t)Nsp * Np * sizeof(double)));
    SB_CUDA(cudaMemsetAsync(W.p, 0, (size_t)Nsp * Np * sizeof(double), c->stream));
    SB_TRY(assemble_dense(c, dc, W.d(), Nsp));
    if (mean_out) {
        SB_TRY(mean.alloc(Nsp * sizeof(double)));
        launch_gemv_n(W.d(), Nsp, Nsp, Np, f->alpha, mean.d(), c->stream);
        if (shard) {
            if (Ns > 0) SB_CUDA(cudaMemcpyAsync(g_send_m, mean.p, Ns * sizeof(double), cudaMemcpyDeviceToDevice, c->stream));
        } else {
            SB_CUDA(cudaMemcpyAsync(mean_out, mean.p, Ns * sizeof(double), cudaMemcpyDefault, c->stream));
        }
    }
    if (need_var) {
        SB_TRY(Xk.alloc((size_t)Nsp * SWEEP_COLS * sizeof(double)));
        SB_TRY(acc.alloc(Nsp * sizeof(double)));
        SB_CUDA(cudaMemsetAsync(acc.p, 0, Nsp * sizeof(double), c->stream));
        // V^T = W L^{-T}: block forward substitution from the right, tensor-core products only
        OzSweepWs ws(c);
        if (f->oz) SB_TRY(ws.init(Nsp));
        SB_TRY(trsm_sweep(c, f, W.d(), Nsp, Xk.d(), /*keep=*/full_cov, full_cov ? nullptr : acc.d(), &ws));
        if (!full_cov) {
            SB_TRY(pd.alloc(Nsp * sizeof(double)));
            SB_CUDA(cudaMemsetAsync(pd.p, 0, Nsp * sizeof(double), c->stream));
            SB_TRY(assemble_diag(c, dp, pd.d()));
            launch_sub(pd.d(), pd.d(), acc.d(), Ns, c->stream);
            if (var_out && shard) {
                if (Ns > 0) SB_CUDA(cudaMemcpyAsync(g_send_v, pd.p, Ns * sizeof(double), cudaMemcpyDeviceToDevice, c->stream));
            } else if (var_out) {
                SB_CUDA(cudaMemcpyAsync(var_out, pd.p, Ns * sizeof(double), cudaMemcpyDefault, c->stream));
            }
        } else {
            // cov = prior_full - V^T V  = prior_full - W W^T   (W now holds V^T, Nsp x Np)
            DevBuf Cm(c);
            SB_TRY(Cm.alloc((size_t)Nsp * Nsp * sizeof(double)));
            SB_CUDA(cudaMemsetAsync(Cm.p, 0, (size_t)Nsp * Nsp * sizeof(double), c->stream));
            SB_TRY(assemble_dense(c, dp, Cm.d(), Nsp));
            launch_gemm_nt(W.d(), Nsp, W.d(), Nsp, Cm.d(), Nsp, Nsp, Nsp, Np, -1.0, 1.0, c->stream);
            if (cov_out)
                SB_CUDA(cudaMemcpy2DAsync(cov_out, Ns * sizeof(double), Cm.p, Nsp * sizeof(double),
                                          Ns * sizeof(double), Ns, cudaMemcpyDefault, c->stream));
            if (fac_out) {
                // posterior covariance (+ noise) -> packed layout -> Cholesky, all on device
                sb_factor* fn = nullptr;
                SB_TRY(factor_alloc(c, Ns, &fn));
                DevBuf nd(c), ndn(c);
                double s2 = post_noise ? post_noise->sigma2 : 0.0;
                const bool pn_dense = post_noise && post_noise->dense;
                launch_pack_lower(fn->L, Cm.d(), Nsp, (pn_dense || (post_noise && post_noise->diag)) ? 0.0 : s2, c->stream);
                if (pn_dense) {  // f_post(x*, Sigma_dense): add the lower triangle of the full noise matrix
                    int32_t st2 = ndn.alloc((size_t)Ns * Ns * sizeof(double));
                    if (st2 != SB_OK) { sb_factor_destroy(fn); return st2; }
                    cudaMemcpyAsync(ndn.p, post_noise->dense, (size_t)Ns * Ns * sizeof(double), cudaMemcpyDefault, c->stream);
                    launch_add_dense_lower(fn->L, ndn.d(), Ns, Ns, c->stream);
                } else if (post_noise && post_noise->diag) {
                    int32_t st2 = nd.alloc(Ns * sizeof(double));
                    if (st2 != SB_OK) { sb_factor_destroy(fn); return st2; }
                    cudaMemcpyAsync(nd.p, post_noise->diag, Ns * sizeof(double), cudaMemcpyDefault, c->stream);
                    launch_add_diag(fn->L, nd.d(), Ns, c->stream);
                }
                launch_fill_padding(fn->L, Ns, c->stream);
                int32_t st2 = factor_finish(c, fn, info, /*force_local=*/true);
                if (st2 != SB_OK) { sb_factor_destroy(fn); return st2; }
                *fac_out = fn;
            }
            SB_CUDA(cudaStreamSynchronize(c->stream));
        }
    }
    SB_CUDA(cudaGetLastError());
    if (shard) {
        if (mean_out) {
            SB_NCCL(nccl_dl::AllGather(g_send_m, g_recv_m, (size_t)chunk, ncclDouble, c->comm, c->stream));
            SB_CUDA(cudaMemcpyAsync(mean_out, g_recv_m, Ns_all * sizeof(double), cudaMemcpyDefault, c->stream));
        }
        if (var_out) {
            SB_NCCL(nccl_dl::AllGather(g_send_v, g_recv_v, (size_t)chunk, ncclDouble, c->comm, c->stream));
            SB_CUDA(cudaMemcpyAsync(var_out, g_recv_v, Ns_all * sizeof(double), cudaMemcpyDefault, c->stream));
        }
    }
    cudaEventRecord(t1, c->stream);
    SB_CUDA(cudaStreamSynchronize(c->stream));
    float ms = 0;
    cudaEventElapsedTime(&ms, t0, t1);
    c->tm.predict_ms += ms;
    c->tm.total_ms += ms;
    count_launches(c, before);
    return SB_OK;
}

int32_t sb_predict(sb_ctx* c, sb_factor* f, const sb_covspec* cross, const sb_covspec* prior_diag,
                   void* mean_out, void* var_out) {
    SB_CHECK(c && f && cross, "null argument");
    return predict_impl(c, f, cross, prior_diag, false, mean_out, var_out, nullptr);
}

int32_t sb_predict_cov(sb_ctx* c, sb_factor* f, const sb_covspec* cross,
                       const sb_covspec* prior_full, void* cov_out) {
    SB_CHECK(c && f && cross && prior_full && cov_out, "null argument");
    return predict_impl(c, f, cross, prior_full, true, nullptr, nullptr, cov_out);
}

int32_t sb_predict_factor(sb_ctx* c, sb_factor* f, const sb_covspec* cross, const sb_covspec* prior_full,
                          const sb_noise* noise, sb_factor** out, int64_t* info) {
    SB_CHECK(c && f && cross && prior_full && out, "null argument");
    *out = nullptr;
    if (info) *info = 0;
    return predict_impl(c, f, cross, prior_full, true, nullptr, nullptr, nullptr, noise, out, info);
}

// ---- gradients of logpdf (SURVEY 8f.1) ------------------------------------------------------------
// dlogpdf/dtheta = 1/2 tr((alpha alpha' - K^{-1}) dK/dtheta)  -- what Zygote + the ChainRules glue of
// src/affine_transformations/cross.jl:8-22 deliver in the reference (examples/getting_started/
// script.jl:154-213).  K^{-1} = L^{-T} L^{-1} is formed once with the tensor-core sweep (I L^{-T}, then
// one NT product), after which every term costs one fused O(N^2) reduction.
static __global__ void set_identity_kernel(double* W, int64_t n) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) W[i * n + i] = 1.0;
}
static __global__ void qdiag_kernel(const double* alpha, const double* Kinv, int64_t ld, int64_t n, double* out) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = 0.5 * (alpha[i] * alpha[i] - Kinv[i * ld + i]);
}

int32_t sb_logpdf_grad(sb_ctx* c, sb_factor* f, const sb_covspec* spec, double* g_terms, void* g_noise_diag) {
    SB_CHECK(c && f && spec && g_terms && g_noise_diag, "null argument");
    SB_CHECK(f->has_alpha, "sb_logpdf_grad needs alpha: call sb_factor_set_data(delta) first");
    SB_CHECK(spec->symmetric == 1 && spec->nrows == f->N && spec->ncols == f->N, "spec must be the symmetric N x N spec of the factor");
    begin_call(c);
    int64_t before = g_launch_count;
    const int64_t N = f->N, Np = f->Np;
    DevSpec ds(c);
    SB_TRY(ds.build(spec, c->stream, false));
    DevBuf W(c), Kinv(c), Xk(c), g(c), qd(c);
    SB_TRY(W.alloc((size_t)Np * Np * sizeof(double)));
    SB_TRY(Kinv.alloc((size_t)Np * Np * sizeof(double)));
    SB_TRY(Xk.alloc((size_t)Np * SWEEP_COLS * sizeof(double)));
    SB_TRY(g.alloc((size_t)2 * (spec->nterms > 0 ? spec->nterms : 1) * sizeof(double)));
    SB_TRY(qd.alloc((size_t)N * sizeof(double)));
    SB_CUDA(cudaMemsetAsync(W.p, 0, (size_t)Np * Np * sizeof(double), c->stream));
    SB_CUDA(cudaMemsetAsync(g.p, 0, (size_t)2 * (spec->nterms > 0 ? spec->nterms : 1) * sizeof(double), c->stream));
    set_identity_kernel<<<(unsigned)((Np + 255) / 256), 256, 0, c->stream>>>(W.d(), Np);
    OzSweepWs ws(c);
    if (f->oz) SB_TRY(ws.init(Np));
    SB_TRY(trsm_sweep(c, f, W.d(), Np, Xk.d(), /*keep=*/true, nullptr, &ws));              // W = L^{-T}
    launch_gemm_nt(W.d(), Np, W.d(), Np, Kinv.d(), Np, Np, Np, Np, 1.0, 0.0, c->stream);  // K^{-1} = W W'
    for (auto& b : ds.blocks) {
        const bool offdiag = b.row0 != b.col0;   // symmetric spec: blocks (i, j), j <= i; (i, i) is the full square
        launch_grad_reduce(b, f->alpha, Kinv.d(), Np, offdiag ? 2.0 : 1.0, g.d(), c->stream);
    }
    qdiag_kernel<<<(unsigned)((N + 255) / 256), 256, 0, c->stream>>>(f->alpha, Kinv.d(), Np, N, qd.d());
    g_launch_count += 2;
    SB_CUDA(cudaGetLastError());
    if (spec->nterms > 0)
        SB_CUDA(cudaMemcpyAsync(g_terms, g.p, (size_t)2 * spec->nterms * sizeof(double), cudaMemcpyDefault, c->stream));
    SB_CUDA(cudaMemcpyAsync(g_noise_diag, qd.p, (size_t)N * sizeof(double), cudaMemcpyDefault, c->stream));
    SB_CUDA(cudaStreamSynchronize(c->stream));
    count_launches(c, before);
    return SB_OK;
}

int32_t sb_rand(sb_ctx* c, sb_factor* f, const void* z, int32_t S, void* out) {
    SB_CHECK(c && f && z && out && S >= 1, "bad argument");
    begin_call(c);
    int64_t before = g_launch_count;
    DevBuf zb(c), ob(c);
    SB_TRY(zb.alloc((size_t)f->Np * S * sizeof(double)));
    SB_TRY(ob.alloc((size_t)f->Np * S * sizeof(double)));
    SB_TRY(upload_padded(c, z, f->N, f->Np, S, zb.d()));
    launch_trmv_lower(f->L, f->N, zb.d(), ob.d(), S, c->stream);
    SB_CUDA(cudaGetLastError());
    SB_CUDA(cudaMemcpy2DAsync(out, f->N * sizeof(double), ob.p, f->Np * sizeof(double), f->N * sizeof(double),
                              S, cudaMemcpyDefault, c->stream));
    SB_CUDA(cudaStreamSynchronize(c->stream));
    count_launches(c, before);
    return SB_OK;
}

int32_t sb_factor_get_L(sb_ctx* c, sb_factor* f, void* L_out) {
    SB_CHECK(c && f && L_out, "null argument");
    SB_CHECK(f->N <= 65535, "sb_factor_get_L is a debug path (N <= 65535)");
    begin_call(c);
    DevBuf d(c);
    SB_TRY(d.alloc((size_t)f->N * f->N * sizeof(double)));
    launch_unpack_lower(f->L, f->N, d.d(), c->stream);
    SB_CUDA(cudaGetLastError());
    SB_CUDA(cudaMemcpyAsync(L_out, d.p, (size_t)f->N * f->N * sizeof(double), cudaMemcpyDefault, c->stream));
    SB_CUDA(cudaStreamSynchronize(c->stream));
    return SB_OK;
}

struct sb_vfe {
    sb_ctx* ctx = nullptr;
    sb_factor* fu = nullptr;  // chol(K_uu + jitter)
    sb_factor* fl = nullptr;  // chol(A A^T + I)
    double* alpha = nullptr;  // Mp, K_*u alpha = posterior mean
    size_t bytes_alpha = 0;
    int64_t M = 0, Mp = 0;
};

int32_t sb_vfe_destroy(sb_vfe* v) {
    if (!v) return SB_OK;
    if (v->fu) sb_factor_destroy(v->fu);
    if (v->fl) sb_factor_destroy(v->fl);
    if (v->alpha) v->ctx->pool_release(v->alpha, v->bytes_alpha);
    delete v;
    return SB_OK;
}

// Titsias VFE (AbstractGPs `_compute_intermediates`, SURVEY App. A), streamed over row chunks of
// the observations so K_fu is never held whole:  per chunk  W = Sigma^{-1/2} K_fu  ->  W L_u^{-T}
// (= A^T rows)  ->  D += A A^T,  v += A delta~,  |A|_F^2.   Multi-GPU: chunks are sharded over
// ranks and D, v, |A|_F^2 are all-reduced (the only collective); the two M x M Choleskys are
// replicated.
int32_t sb_vfe_create(sb_ctx* c, const sb_covspec* uu, const sb_noise* noise_u, const sb_covspec* xu,
                      const sb_covspec* ff_diag, const sb_noise* noise_f, const void* delta, sb_vfe** out,
                      double* out2, int64_t* info) {
    SB_CHECK(c && uu && xu && ff_diag && noise_f && delta && out && out2, "null argument");
    begin_call(c);
    int64_t before = g_launch_count;
    *out = nullptr;
    if (info) *info = 0;
    const int64_t N = xu->nrows, M = xu->ncols;
    SB_CHECK(uu->nrows == M && uu->symmetric == 1, "uu must be the symmetric M x M spec of cov(fz)");
    SB_CHECK(ff_diag->nrows == N, "ff_diag must have N rows");
    SB_CHECK(N > 0 && M > 0, "empty problem");
    SB_CHECK(noise_f->dense == nullptr, "VFE needs diagonal observation noise");
    cudaEvent_t t0 = c->next_event(), t1 = c->next_event();
    cudaEventRecord(t0, c->stream);

    sb_vfe* v = new sb_vfe();
    v->ctx = c;
    auto fail = [&](int32_t st) { sb_vfe_destroy(v); return st; };
    int32_t st = factor_create_impl(c, uu, noise_u, &v->fu, info, /*force_local=*/true);
    if (st != SB_OK) return fail(st);
    begin_call(c);  // factor_create_impl reset the event pool; keep our own markers valid
    t0 = c->next_event(); t1 = c->next_event();
    cudaEventRecord(t0, c->stream);
    v->M = M;
    v->Mp = v->fu->Np;
    const int64_t Mp = v->Mp;

    // host O(N) prep: sigma^{-1}, delta~ = delta / sigma, log det Sigma_y, |delta~|^2
    std::vector<double> hd(N), sinv(N), hnoise(N);
    if (cudaMemcpy(hd.data(), delta, N * sizeof(double), cudaMemcpyDefault) != cudaSuccess) return fail(SB_ERR_CUDA);
    if (noise_f->diag) {
        if (cudaMemcpy(hnoise.data(), noise_f->diag, N * sizeof(double), cudaMemcpyDefault) != cudaSuccess) return fail(SB_ERR_CUDA);
    } else {
        for (int64_t i = 0; i < N; i++) hnoise[i] = noise_f->sigma2;
    }
    double logdet_sy = 0.0, dd = 0.0;
    for (int64_t i = 0; i < N; i++) {
        if (!(hnoise[i] > 0.0)) { sb::set_error("VFE needs positive observation noise"); return fail(SB_ERR_INVALID); }
        sinv[i] = 1.0 / sqrt(hnoise[i]);
        logdet_sy += log(hnoise[i]);
        hd[i] *= sinv[i];
        dd += hd[i] * hd[i];
    }

    DevSpec dxu(c), dff(c);
    if ((st = dxu.build(xu, c->stream, false)) != SB_OK) return fail(st);
    if ((st = dff.build(ff_diag, c->stream, true)) != SB_OK) return fail(st);
    const std::vector<BlockDev> all_blocks = dxu.blocks;

    const int64_t NC = 16384;  // observation rows per chunk
    DevBuf dsinv(c), ddt(c), W(c), T(c), Xk(c), D(c), vv(c), fro(c), varf(c);
    const int64_t nchunks_total = (N + NC - 1) / NC;
#define VFE_TRY(expr) do { int32_t _s = (expr); if (_s != SB_OK) return fail(_s); } while (0)
#define VFE_CUDA(call) do { cudaError_t _e = (call); if (_e != cudaSuccess) return fail(sb::cuda_fail(_e, #call, __FILE__, __LINE__)); } while (0)
    VFE_TRY(dsinv.alloc(N * sizeof(double)));
    VFE_TRY(ddt.alloc(round_up(N, NC) * sizeof(double)));
    VFE_TRY(W.alloc((size_t)NC * Mp * sizeof(double)));
    VFE_TRY(T.alloc((size_t)NC * Mp * sizeof(double)));
    VFE_TRY(Xk.alloc((size_t)NC * SWEEP_COLS * sizeof(double)));
    VFE_TRY(D.alloc((size_t)Mp * Mp * sizeof(double)));
    VFE_TRY(vv.alloc((size_t)(Mp + 8) * sizeof(double)));
    VFE_TRY(fro.alloc((size_t)(nchunks_total + 1) * sizeof(double)));
    VFE_TRY(varf.alloc(N * sizeof(double)));
    VFE_CUDA(cudaMemcpyAsync(dsinv.p, sinv.data(), N * sizeof(double), cudaMemcpyHostToDevice, c->stream));
    VFE_CUDA(cudaMemsetAsync(ddt.p, 0, round_up(N, NC) * sizeof(double), c->stream));
    VFE_CUDA(cudaMemcpyAsync(ddt.p, hd.data(), N * sizeof(double), cudaMemcpyHostToDevice, c->stream));
    VFE_CUDA(cudaMemsetAsync(D.p, 0, (size_t)Mp * Mp * sizeof(double), c->stream));
    VFE_CUDA(cudaMemsetAsync(vv.p, 0, (size_t)(Mp + 8) * sizeof(double), c->stream));
    VFE_CUDA(cudaMemsetAsync(fro.p, 0, (size_t)(nchunks_total + 1) * sizeof(double), c->stream));

    OzSweepWs ws(c);
    if (v->fu->oz) VFE_TRY(ws.init(NC));
    for (int64_t ci = c->rank; ci < nchunks_total; ci += c->world) {  // chunks round-robin over ranks
        const int64_t r0 = ci * NC, r1 = r0 + NC < N ? r0 + NC : N;
        const int64_t rows = r1 - r0, rows_p = round_up(rows, NB);
        dxu.blocks = all_blocks;
        dxu.nrows = N;
        clip_rows(dxu, r0, r1, false);
        VFE_CUDA(cudaMemsetAsync(W.p, 0, (size_t)rows_p * Mp * sizeof(double), c->stream));
        VFE_TRY(assemble_dense(c, dxu, W.d(), rows_p));
        launch_rowscale(W.d(), rows_p, rows, Mp, dsinv.d() + r0, c->stream);
        VFE_TRY(trsm_sweep(c, v->fu, W.d(), rows_p, Xk.d(), /*keep=*/true, nullptr, &ws));
        launch_colsumsq(W.d(), rows_p * Mp, 0, 1, fro.d() + ci, c->stream);
        launch_gemv_t(W.d(), rows_p, rows, Mp, ddt.d() + r0, vv.d(), c->stream);
        launch_transpose(W.d(), rows_p, rows_p, Mp, T.d(), Mp, c->stream);
        launch_gemm_nt(T.d(), Mp, T.d(), Mp, D.d(), Mp, Mp, Mp, rows_p, 1.0, 1.0, c->stream);
    }
    VFE_CUDA(cudaGetLastError());
    if (c->world > 1) {
        auto nc = [&](ncclResult_t r) { if (r != ncclSuccess) { sb::set_error("NCCL all-reduce failed in VFE"); return false; } return true; };
        if (!nc(nccl_dl::AllReduce(D.p, D.p, (size_t)Mp * Mp, ncclDouble, ncclSum, c->comm, c->stream))) return fail(SB_ERR_NCCL);
        if (!nc(nccl_dl::AllReduce(vv.p, vv.p, (size_t)Mp, ncclDouble, ncclSum, c->comm, c->stream))) return fail(SB_ERR_NCCL);
        if (!nc(nccl_dl::AllReduce(fro.p, fro.p, (size_t)nchunks_total, ncclDouble, ncclSum, c->comm, c->stream))) return fail(SB_ERR_NCCL);
    }
    // Lambda = chol(D + I)
    VFE_TRY(factor_alloc(c, M, &v->fl));
    launch_pack_lower(v->fl->L, D.d(), Mp, 1.0, c->stream);
    // (padding rows/cols of D are zero: +1 on the diagonal makes them identity)
    VFE_CUDA(cudaGetLastError());
    st = factor_finish(c, v->fl, info, /*force_local=*/true);
    if (st != SB_OK) return fail(st);
    // w = L_Lambda^{-1} (A delta~)
    DevBuf q(c);
    VFE_TRY(q.alloc(sizeof(double)));
    forward_solve(c, v->fl, vv.d(), 1);
    launch_colsumsq(vv.d(), Mp, Mp, 1, q.d(), c->stream);
    // var(f, x) for the trace term
    VFE_CUDA(cudaMemsetAsync(varf.p, 0, N * sizeof(double), c->stream));
    VFE_TRY(assemble_diag(c, dff, varf.d()));
    std::vector<double> hvar(N), hfro(nchunks_total);
    double hq = 0.0;
    VFE_CUDA(cudaMemcpyAsync(hvar.data(), varf.p, N * sizeof(double), cudaMemcpyDeviceToHost, c->stream));
    VFE_CUDA(cudaMemcpyAsync(hfro.data(), fro.p, nchunks_total * sizeof(double), cudaMemcpyDeviceToHost, c->stream));
    VFE_CUDA(cudaMemcpyAsync(&hq, q.p, sizeof(double), cudaMemcpyDeviceToHost, c->stream));
    // posterior weights: m_eps = L_Lambda^{-T} w ; alpha = L_u^{-T} m_eps
    backward_solve(c, v->fl, vv.d(), 1);
    backward_solve(c, v->fu, vv.d(), 1);
    v->bytes_alpha = (size_t)Mp * sizeof(double);
    VFE_CUDA(c->pool_alloc((void**)&v->alpha, v->bytes_alpha));
    VFE_CUDA(cudaMemcpyAsync(v->alpha, vv.p, v->bytes_alpha, cudaMemcpyDeviceToDevice, c->stream));
    VFE_CUDA(cudaGetLastError());
    cudaEventRecord(t1, c->stream);
    VFE_CUDA(cudaStreamSynchronize(c->stream));
    double tr = 0.0, fro_sum = 0.0;
    for (int64_t i = 0; i < N; i++) tr += hvar[i] / hnoise[i];
    for (double x : hfro) fro_sum += x;
    const double log2pi = 1.8378770664093454835606594728112;
    const double dtc = -((double)N * log2pi + logdet_sy + v->fl->logdet + dd - hq) / 2.0;
    out2[0] = dtc - (tr - fro_sum) / 2.0;  // elbo
    out2[1] = dtc;
    float ms = 0;
    cudaEventElapsedTime(&ms, t0, t1);
    c->tm.total_ms += ms;
    count_launches(c, before);
    *out = v;
    return SB_OK;
#undef VFE_TRY
#undef VFE_CUDA
}

// cov(f_approx_post(x*)) = K** - B'B + (L_Lambda^{-1} B)'(L_Lambda^{-1} B),  B = L_u^{-1} K_u*
// (AbstractGPs approx posterior, SURVEY App. A).  cross: N* x M dense spec, prior_full: N* x N*.
int32_t sb_vfe_predict_cov(sb_ctx* c, sb_vfe* v, const sb_covspec* cross, const sb_covspec* prior_full,
                           void* cov_out) {
    SB_CHECK(c && v && cross && prior_full && cov_out, "null argument");
    SB_CHECK(cross->ncols == v->M, "cross spec must be N* x M");
    SB_CHECK(prior_full->nrows == cross->nrows && prior_full->ncols == cross->nrows, "prior spec must be N* x N*");
    begin_call(c);
    int64_t before = g_launch_count;
    const int64_t Ns = cross->nrows, Nsp = round_up(Ns > 0 ? Ns : 1, NB), Mp = v->Mp;
    if (Ns == 0) return SB_OK;
    DevSpec dc(c), dp(c);
    SB_TRY(dc.build(cross, c->stream, false));
    SB_TRY(dp.build(prior_full, c->stream, false));
    DevBuf W(c), Xk(c), Cm(c);
    SB_TRY(W.alloc((size_t)Nsp * Mp * sizeof(double)));
    SB_TRY(Xk.alloc((size_t)Nsp * SWEEP_COLS * sizeof(double)));
    SB_TRY(Cm.alloc((size_t)Nsp * Nsp * sizeof(double)));
    SB_CUDA(cudaMemsetAsync(W.p, 0, (size_t)Nsp * Mp * sizeof(double), c->stream));
    SB_CUDA(cudaMemsetAsync(Cm.p, 0, (size_t)Nsp * Nsp * sizeof(double), c->stream));
    SB_TRY(assemble_dense(c, dc, W.d(), Nsp));
    SB_TRY(assemble_dense(c, dp, Cm.d(), Nsp));
    OzSweepWs ws(c);
    if (v->fu->oz || v->fl->oz) SB_TRY(ws.init(Nsp));
    SB_TRY(trsm_sweep(c, v->fu, W.d(), Nsp, Xk.d(), true, nullptr, &ws));      // W = B'
    launch_gemm_nt(W.d(), Nsp, W.d(), Nsp, Cm.d(), Nsp, Nsp, Nsp, Mp, -1.0, 1.0, c->stream);
    SB_TRY(trsm_sweep(c, v->fl, W.d(), Nsp, Xk.d(), true, nullptr, &ws));      // W = (L_Lambda^{-1} B)'
    launch_gemm_nt(W.d(), Nsp, W.d(), Nsp, Cm.d(), Nsp, Nsp, Nsp, Mp, 1.0, 1.0, c->stream);
    SB_CUDA(cudaGetLastError());
    SB_CUDA(cudaMemcpy2DAsync(cov_out, Ns * sizeof(double), Cm.p, Nsp * sizeof(double), Ns * sizeof(double), Ns,
                              cudaMemcpyDefault, c->stream));
    SB_CUDA(cudaStreamSynchronize(c->stream));
    count_launches(c, before);
    return SB_OK;
}

int32_t sb_vfe_predict(sb_ctx* c, sb_vfe* v, const sb_covspec* cross, const sb_covspec* prior_diag,
                       void* mean_out, void* var_out) {
    SB_CHECK(c && v && cross, "null argument");
    SB_CHECK(cross->ncols == v->M, "cross spec must be N* x M");
    begin_call(c);
    int64_t before = g_launch_count;
    const int64_t Ns = cross->nrows, Nsp = round_up(Ns > 0 ? Ns : 1, NB), Mp = v->Mp;
    if (Ns == 0) return SB_OK;
    DevSpec dc(c), dp(c);
    SB_TRY(dc.build(cross, c->stream, false));
    DevBuf W(c), Xk(c), mean(c), acc1(c), acc2(c), pd(c);
    SB_TRY(W.alloc((size_t)Nsp * Mp * sizeof(double)));
    SB_CUDA(cudaMemsetAsync(W.p, 0, (size_t)Nsp * Mp * sizeof(double), c->stream));
    SB_TRY(assemble_dense(c, dc, W.d(), Nsp));
    if (mean_out) {
        SB_TRY(mean.alloc(Nsp * sizeof(double)));
        launch_gemv_n(W.d(), Nsp, Nsp, Mp, v->alpha, mean.d(), c->stream);
        SB_CUDA(cudaMemcpyAsync(mean_out, mean.p, Ns * sizeof(double), cudaMemcpyDefault, c->stream));
    }
    if (var_out) {
        SB_CHECK(prior_diag && prior_diag->nrows == Ns, "prior diag spec required for var");
        SB_TRY(dp.build(prior_diag, c->stream, true));
        SB_TRY(Xk.alloc((size_t)Nsp * SWEEP_COLS * sizeof(double)));
        SB_TRY(acc1.alloc(Nsp * sizeof(double)));
        SB_TRY(acc2.alloc(Nsp * sizeof(double)));
        SB_TRY(pd.alloc(Nsp * sizeof(double)));
        SB_CUDA(cudaMemsetAsync(acc1.p, 0, Nsp * sizeof(double), c->stream));
        SB_CUDA(cudaMemsetAsync(acc2.p, 0, Nsp * sizeof(double), c->stream));
        SB_CUDA(cudaMemsetAsync(pd.p, 0, Nsp * sizeof(double), c->stream));
        // B^T = K_*u L_u^{-T} (kept), then (L_Lambda^{-1} B)^T = B^T L_Lambda^{-T}
        OzSweepWs ws(c);
        if (v->fu->oz || v->fl->oz) SB_TRY(ws.init(Nsp));
        SB_TRY(trsm_sweep(c, v->fu, W.d(), Nsp, Xk.d(), true, acc1.d(), &ws));
        SB_TRY(trsm_sweep(c, v->fl, W.d(), Nsp, Xk.d(), false, acc2.d(), &ws));
        SB_TRY(assemble_diag(c, dp, pd.d()));
        launch_sub(pd.d(), pd.d(), acc1.d(), Ns, c->stream);    // k** - |B|^2
        launch_axpy1(pd.d(), acc2.d(), Ns, c->stream);          //     + |L_Lambda^{-1} B|^2
        SB_CUDA(cudaMemcpyAsync(var_out, pd.p, Ns * sizeof(double), cudaMemcpyDefault, c->stream));
    }
    SB_CUDA(cudaGetLastError());
    SB_CUDA(cudaStreamSynchronize(c->stream));
    count_launches(c, before);
    return SB_OK;
}

}  // extern "C"
