// Host-side internals shared by api.cu (ABI entry points), cholesky.cu (factorisation drivers) and p2p.cu
// (peer-to-peer panel exchange): the context, the factor, pooled device buffers, event timing, NCCL.
#pragma once
#include <nccl.h>

#include <string>
#include <vector>

#include "sb_common.cuh"

// NCCL entry points, bound with dlopen by nccl_dl::load() (api.cu)
namespace nccl_dl {
typedef ncclResult_t (*GetUniqueId_t)(ncclUniqueId*);
typedef ncclResult_t (*CommInitRank_t)(ncclComm_t*, int, ncclUniqueId, int);
typedef ncclResult_t (*CommDestroy_t)(ncclComm_t);
typedef ncclResult_t (*Broadcast_t)(const void*, void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t);
typedef ncclResult_t (*AllReduce_t)(const void*, void*, size_t, ncclDataType_t, ncclRedOp_t, ncclComm_t, cudaStream_t);
typedef ncclResult_t (*AllGather_t)(const void*, void*, size_t, ncclDataType_t, ncclComm_t, cudaStream_t);
typedef ncclResult_t (*Group_t)(void);
typedef const char* (*ErrStr_t)(ncclResult_t);
extern GetUniqueId_t GetUniqueId;
extern CommInitRank_t CommInitRank;
extern CommDestroy_t CommDestroy;
extern Broadcast_t Broadcast;
extern AllReduce_t AllReduce;
extern AllGather_t AllGather;
extern Group_t GroupStart, GroupEnd;
extern ErrStr_t GetErrorString;
bool load();
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
    // peer-to-peer panel exchange over NVLink (multi-GPU, see p2p.cu)
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

// One allocation from the context's pool; it goes back to the pool, with the size it was taken with, when the
// buffer is destroyed.
struct DevBuf {
    void* p = nullptr;
    size_t bytes = 0;
    sb_ctx* ctx;
    explicit DevBuf(sb_ctx* c) : ctx(c) {}
    DevBuf(const DevBuf&) = delete;
    DevBuf& operator=(const DevBuf&) = delete;
    DevBuf(DevBuf&& o) noexcept : p(o.p), bytes(o.bytes), ctx(o.ctx) { o.p = nullptr; }
    ~DevBuf() { ctx->pool_release(p, bytes); }
    int32_t alloc(size_t nbytes) {
        bytes = nbytes ? nbytes : 8;
        SB_CUDA(ctx->pool_alloc(&p, bytes));
        return SB_OK;
    }
    double* d() const { return reinterpret_cast<double*>(p); }
};

// A DevBuf of T elements that converts to T*, so it is passed and indexed like the pointer it holds
template <class T>
struct DevArray : DevBuf {
    using DevBuf::DevBuf;
    operator T*() const { return static_cast<T*>(p); }
};

struct sb_factor {
    sb_ctx* ctx;
    int64_t N = 0, Np = 0;
    DevArray<double> L_buf{ctx};
    sb::Packed L{nullptr, 0};        // view of L_buf
    DevArray<double> invL{ctx};
    DevArray<double> ldiag{ctx};     // multi-GPU only: contiguous copies of the diagonal blocks L_kk (broadcast payload)
    DevArray<double> logdet_blk{ctx};
    DevArray<long long> info_dev{ctx};
    DevArray<double> panel{ctx};     // 2 x (Np x NB) panel buffers
    DevArray<double> alpha{ctx};     // Np
    bool has_alpha = false;
    double logdet = 0.0;
    // int8 Ozaki trailing update (ozaki.cu): two sets (look-ahead) of int8 digit planes + row scales, and the
    // wide panel phase's buffers below; all allocated together
    bool oz = false;
    DevArray<signed char> oz_planes[2]{DevArray<signed char>(ctx), DevArray<signed char>(ctx)};
    DevArray<double> oz_scale[2]{DevArray<double>(ctx), DevArray<double>(ctx)};
    DevArray<int> oz_expo[2]{DevArray<int>(ctx), DevArray<int>(ctx)};
    DevArray<unsigned> sweep_flags{ctx};  // 2*nblk flags of the persistent triangular sweep
    // logpdf(fx, y) followed by posterior(fx, y) is THE usage pattern (README.md:61-81): the forward
    // sweep v = L^{-1} delta of the last single-RHS logpdf is kept so posterior only adds the backward one
    DevArray<double> vcache{ctx};         // [2][Np]: delta, then v
    DevArray<int> vcache_flag{ctx};
    bool vcache_valid = false;
    sb::OzMaps oz_maps[2];
    // wide panel phase (see wide_diag_phase): dense scratch of the step's 512 x 512 diagonal block stacked over an
    // identity (input and result copies), inv(L_512) and its digit planes
    DevArray<double> wide_D{ctx};         // [2][1024 x 512], ld 1024
    DevArray<double> wide_W{ctx};         // 512 x 512, column-major
    DevArray<signed char> wide_wp{ctx};   // digit planes of wide_W  [7][512][512]
    DevArray<double> wide_wscale{ctx};
    DevArray<int> wide_wexpo{ctx};
    sb::OzMaps wide_wmaps;

    explicit sb_factor(sb_ctx* c) : ctx(c) {}
    // The pool's best fit breaks ties by free-list position, so the release order decides which buffer of a later
    // factor gets which block: it is kept fixed here.
    ~sb_factor() {
        DevBuf* order[] = {&L_buf, &invL, &ldiag, &logdet_blk, &info_dev, &panel, &alpha,
                           &oz_planes[0], &oz_scale[0], &oz_expo[0], &oz_planes[1], &oz_scale[1], &oz_expo[1],
                           &wide_D, &wide_W, &wide_wp, &wide_wscale, &wide_wexpo, &sweep_flags, &vcache, &vcache_flag};
        for (DevBuf* b : order) {
            ctx->pool_release(b->p, b->bytes);
            b->p = nullptr;
        }
    }
};

// Stream time between pairs of recorded events, added to sb_timings fields by collect() once the streams have
// synchronised.  A timer that is off records nothing (the drivers' intervals without fine timing).
struct Timer {
    struct Span { cudaEvent_t a, b; double* to; double* to2; double sign; };
    sb_ctx* c;
    bool on;
    std::vector<Span> spans;
    Timer(sb_ctx* ctx, bool enabled) : c(ctx), on(enabled) {}
    cudaEvent_t mark(cudaStream_t st) {  // a new event recorded on st (nullptr when off)
        if (!on) return nullptr;
        cudaEvent_t e = c->next_event();
        cudaEventRecord(e, st);
        return e;
    }
    // the time from a to b counts in *to (and *to2); sign -1 takes it off again
    void add(cudaEvent_t a, cudaEvent_t b, double* to, double* to2 = nullptr, double sign = 1.0) {
        if (on) spans.push_back({a, b, to, to2, sign});
    }
    void add_trailing(cudaEvent_t a, cudaEvent_t b, double sign = 1.0) {
        add(a, b, &c->tm.trailing_ms, &c->tm.trailing_kernel_ms, sign);
    }
    void collect() {
        for (const Span& s : spans) {
            float ms = 0;
            cudaEventElapsedTime(&ms, s.a, s.b);
            *s.to += s.sign * ms;
            if (s.to2) *s.to2 += s.sign * ms;
        }
        spans.clear();
    }
};

// block columns in the outer step that starts at block column k0
inline int outer_width(int64_t nblk, int64_t k0) {
    return (int)(nblk - k0 < sb::OUTER_BLOCKS ? nblk - k0 : sb::OUTER_BLOCKS);
}

// ---- P2P panel exchange (p2p.cu) --------------------------------------------------------------
struct P2PPeers { char* base[8]; };

struct P2PRun {                 // one factorisation's view of the arena
    bool on = false;
    P2PPeers peers{};
    int64_t slot_elems = 0;     // doubles per panel slot
    std::vector<uint32_t> ord;  // ord[k]: absolute ordinal (1-based) of panel k among its owner's panels
    uint32_t guarded = 0;       // acks up to this ordinal of MY panels have already been waited for on the panel stream
    uint32_t* ctr(sb_ctx* c) const;
    double* head(char* base, int64_t k) const;
    double* slot(char* base, int s) const;
};

int32_t p2p_ensure(sb_ctx* c, int64_t Np);
int32_t p2p_run_begin(sb_ctx* c, sb_factor* f, P2PRun& R, int world, int rank, cudaStream_t st);
double* p2p_panel_slot(sb_ctx* c, const P2PRun& R, int s);
int32_t p2p_check(sb_ctx* c, const P2PRun& R);
void p2p_shutdown(sb_ctx* c);
int32_t p2p_slot_guard(sb_ctx* c, P2PRun& R, int64_t k, cudaStream_t st);
int32_t p2p_publish(sb_ctx* c, sb_factor* f, P2PRun& R, int64_t k, cudaStream_t st);
int32_t p2p_pull(sb_ctx* c, sb_factor* f, P2PRun& R, int64_t k, int owner, int64_t slab_off, size_t slab_elems,
                 cudaStream_t st);
int32_t bcast_panel(sb_ctx* c, sb_factor* f, int64_t k, double* Pslab, size_t slab_elems, int owner, cudaStream_t st);
int32_t p2p_exchange_col(sb_ctx* c, sb_factor* f, P2PRun& R, int64_t k, cudaStream_t st);

// ---- Cholesky drivers (cholesky.cu) -----------------------------------------------------------
// factors the assembled packed matrix of f in place (force_local: this rank alone, whatever the world size)
int32_t cholesky_packed(sb_ctx* c, sb_factor* f, bool force_local = false);
