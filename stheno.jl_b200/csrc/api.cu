// C ABI of libstheno_b200 (see include/stheno_b200.h): contexts, plan upload, factor allocation,
// logpdf / posterior / rand / VFE orchestration.  The Cholesky drivers are in cholesky.cu.
#include <dlfcn.h>
#include <math.h>
#include <stdlib.h>
#include <string.h>

#include <memory>
#include <string>
#include <vector>

#include "sb_host.cuh"

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
GetUniqueId_t GetUniqueId;
CommInitRank_t CommInitRank;
CommDestroy_t CommDestroy;
Broadcast_t Broadcast;
AllReduce_t AllReduce;
AllGather_t AllGather;
Group_t GroupStart, GroupEnd;
ErrStr_t GetErrorString;
static bool loaded = false;
bool load() {
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

namespace {

// uploaded covariance plan
struct DevSpec {
    DevBuf pool;
    explicit DevSpec(sb_ctx* c) : pool(c) {}
    std::vector<double*> arr;
    std::vector<BlockDev> blocks;
    int64_t nrows = 0, ncols = 0;
    bool diag = false;  // paired points: every block is square and evaluated on its diagonal only

    int32_t build(const sb_covspec* spec, cudaStream_t st, bool paired) {
        SB_CHECK(spec != nullptr, "null covspec");
        diag = paired;
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

// the blocks of rows [lo, hi) of a plan (and, for paired/diag specs, the same range of columns), re-based to
// row lo.  Used for the row chunks of the VFE stream and to shard the posterior's test points across ranks.
std::vector<BlockDev> clip_rows(const DevSpec& ds, int64_t lo, int64_t hi) {
    std::vector<BlockDev> out;
    for (BlockDev b : ds.blocks) {
        int64_t r0 = b.row0 > lo ? b.row0 : lo;
        int64_t r1 = b.row0 + b.nrows < hi ? b.row0 + b.nrows : hi;
        if (r1 <= r0) continue;
        int64_t off = r0 - b.row0;
        for (int t = 0; t < b.nterms; t++) {
            b.t[t].zl += off * b.t[t].dim;
            if (b.t[t].sl) b.t[t].sl += off;
            if (ds.diag) {
                b.t[t].zr += off * b.t[t].dim;
                if (b.t[t].sr) b.t[t].sr += off;
            }
        }
        b.row0 = r0 - lo;
        b.nrows = r1 - r0;
        if (ds.diag) { b.col0 = b.row0; b.ncols = b.nrows; }
        out.push_back(b);
    }
    return out;
}

// rank's contiguous share [lo, hi) of ns rows split over world ranks in chunks of `chunk` rows
struct RowChunk { int64_t lo, hi, chunk; };
RowChunk row_chunk(int64_t ns, int rank, int world) {
    const int64_t chunk = (ns + world - 1) / world;
    const int64_t lo = rank * chunk < ns ? rank * chunk : ns;
    return {lo, lo + chunk < ns ? lo + chunk : ns, chunk};
}

void begin_call(sb_ctx* c) {
    cudaSetDevice(c->device);
    c->ev_used = 0;
}

// The sb_timings fields an ABI call's stream time adds to: none, total_ms, or predict_ms and total_ms
enum class Timed { no, total, predict };

// Bracket of an ABI call that launches kernels: it starts the call (begin_call) and, on the success path, end()
// adds the call's kernel launches to kernel_launches and its stream time to the fields `timed` names.  Helpers
// inside a call do neither, so every launch is counted once.
struct Call {
    sb_ctx* c;
    Timed timed;
    int64_t before = g_launch_count;
    cudaEvent_t t0 = nullptr;
    Call(sb_ctx* ctx, Timed t = Timed::no) : c(ctx), timed(t) {
        begin_call(c);
        if (timed != Timed::no) {
            t0 = c->next_event();
            cudaEventRecord(t0, c->stream);
        }
    }
    int32_t end() {
        if (timed != Timed::no) {
            cudaEvent_t t1 = c->next_event();
            cudaEventRecord(t1, c->stream);
            SB_CUDA(cudaEventSynchronize(t1));
            float ms = 0;
            cudaEventElapsedTime(&ms, t0, t1);
            if (timed == Timed::predict) c->tm.predict_ms += ms;
            c->tm.total_ms += ms;
        }
        c->tm.kernel_launches += g_launch_count - before;
        return SB_OK;
    }
};

// zero the padded matrix out (ld x ncols) and assemble blocks into it
int32_t assemble_dense(sb_ctx* c, const std::vector<BlockDev>& blocks, double* out, int64_t ld, int64_t ncols) {
    SB_CUDA(cudaMemsetAsync(out, 0, (size_t)ld * ncols * sizeof(double), c->stream));
    for (auto& b : blocks) launch_assemble_dense(b, OutDense{out, ld}, c->stream);
    SB_CUDA(cudaGetLastError());
    return SB_OK;
}

// zero the vector out (n entries) and assemble the diagonal of the paired blocks into it
int32_t assemble_diag(sb_ctx* c, const std::vector<BlockDev>& blocks, double* out, int64_t n) {
    SB_CUDA(cudaMemsetAsync(out, 0, n * sizeof(double), c->stream));
    for (auto& b : blocks) launch_assemble_diag(b, out, c->stream);
    SB_CUDA(cudaGetLastError());
    return SB_OK;
}

__global__ void vec_differs_kernel(const double* a, const double* b, int64_t n, int* flag) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n && __double_as_longlong(a[i]) != __double_as_longlong(b[i])) *flag = 1;
}

// triangular sweep for S right-hand sides (b: Np x S, ld Np):  b <- L^{-1} b,  or  b <- L^{-T} b  when backward
void tri_solve(sb_ctx* c, sb_factor* f, double* b, int S, bool backward) {
    for (int s0 = 0; s0 < S; s0 += 8) {
        int s = S - s0 < 8 ? S - s0 : 8;
        launch_sweep(f->L, f->invL, b + (int64_t)s0 * f->Np, s, backward, f->sweep_flags, c->num_sms, c->stream);
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
    p2p_shutdown(c);
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
    const RowChunk rc = row_chunk(ns, rank, world);
    *lo = rc.lo;
    *hi = rc.hi;
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
    Call call(c);
    DevSpec ds(c);
    SB_TRY(ds.build(spec, c->stream, false));
    DevBuf K(c);
    size_t bytes = (size_t)ds.nrows * ds.ncols * sizeof(double);
    SB_TRY(K.alloc(bytes));
    Timer t(c, true);
    cudaEvent_t t0 = t.mark(c->stream);
    SB_TRY(assemble_dense(c, ds.blocks, K.d(), ds.nrows, ds.ncols));
    t.add(t0, t.mark(c->stream), &c->tm.assemble_ms);
    SB_CUDA(cudaMemcpyAsync(K_out, K.p, bytes, cudaMemcpyDefault, c->stream));
    SB_CUDA(cudaStreamSynchronize(c->stream));
    t.collect();
    return call.end();
}

int32_t sb_cov_diag(sb_ctx* c, const sb_covspec* spec, void* out) {
    SB_CHECK(c && spec && out, "null argument");
    Call call(c);
    DevSpec ds(c);
    SB_TRY(ds.build(spec, c->stream, true));
    DevBuf v(c);
    SB_TRY(v.alloc(ds.nrows * sizeof(double)));
    SB_TRY(assemble_diag(c, ds.blocks, v.d(), ds.nrows));
    SB_CUDA(cudaMemcpyAsync(out, v.p, ds.nrows * sizeof(double), cudaMemcpyDefault, c->stream));
    SB_CUDA(cudaStreamSynchronize(c->stream));
    return call.end();
}

int32_t sb_factor_destroy(sb_factor* f) {
    if (!f) return SB_OK;
    cudaSetDevice(f->ctx->device);
    delete f;
    return SB_OK;
}

// allocate the buffers of a factor of order N from the context pool
static int32_t factor_alloc(sb_ctx* c, int64_t N, std::unique_ptr<sb_factor>& out) {
    std::unique_ptr<sb_factor> f(new sb_factor(c));
    f->N = N;
    f->Np = round_up(N, NB);
    f->L.Np = f->Np;
    const int64_t nblk = f->L.nblk();
    SB_TRY(f->L_buf.alloc((size_t)f->L.total() * sizeof(double)));
    f->L.base = f->L_buf;
    SB_TRY(f->invL.alloc((size_t)nblk * NB * NB * sizeof(double)));
    if (c->world > 1) SB_TRY(f->ldiag.alloc(f->invL.bytes));
    SB_TRY(f->logdet_blk.alloc((size_t)nblk * sizeof(double)));
    SB_TRY(f->info_dev.alloc(8));
    SB_TRY(f->panel.alloc((size_t)2 * OUTER_BLOCKS * tiled_panel_elems(f->Np) * sizeof(double)));
    SB_TRY(f->alpha.alloc((size_t)f->Np * sizeof(double)));
    SB_TRY(f->sweep_flags.alloc((size_t)2 * nblk * sizeof(unsigned)));
    SB_TRY(f->vcache.alloc((size_t)2 * f->Np * sizeof(double)));
    SB_TRY(f->vcache_flag.alloc(sizeof(int)));
    SB_CUDA(cudaMemsetAsync(f->info_dev, 0, sizeof(long long), c->stream));
    SB_CUDA(cudaMemsetAsync(f->logdet_blk, 0, nblk * sizeof(double), c->stream));
    // int8 Ozaki path: worth it (and exercised) once the trailing matrix has a few hundred tiles
    if (c->trailing_mode == 1 && nblk > 2 * OUTER_BLOCKS) {
        for (int i = 0; i < 2; i++) {
            SB_TRY(f->oz_planes[i].alloc(oz_planes_bytes(f->Np)));
            SB_TRY(f->oz_scale[i].alloc((size_t)f->Np * sizeof(double)));
            SB_TRY(f->oz_expo[i].alloc((size_t)f->Np * sizeof(int)));
        }
        constexpr int64_t WD = (int64_t)OUTER_BLOCKS * NB;
        SB_TRY(f->wide_D.alloc((size_t)2 * 2 * WD * WD * sizeof(double)));
        SB_TRY(f->wide_W.alloc((size_t)WD * WD * sizeof(double)));
        SB_TRY(f->wide_wp.alloc(oz_planes_bytes(WD)));
        SB_TRY(f->wide_wscale.alloc((size_t)WD * sizeof(double)));
        SB_TRY(f->wide_wexpo.alloc((size_t)WD * sizeof(int)));
        if (oz_make_maps(f->oz_planes[0], f->Np, &f->oz_maps[0]) != 0 ||
            oz_make_maps(f->oz_planes[1], f->Np, &f->oz_maps[1]) != 0 ||
            oz_make_maps(f->wide_wp, WD, &f->wide_wmaps) != 0) {
            sb::set_error("cuTensorMapEncodeTiled failed for the int8 digit planes");
            return SB_ERR_CUDA;
        }
        f->oz = true;
    }
    out = std::move(f);
    return SB_OK;
}

// f->logdet from the per-block log-pivots, summed on the host in block order
static int32_t sum_logdet(sb_ctx* c, sb_factor* f) {
    std::vector<double> ld(f->L.nblk());
    SB_CUDA(cudaMemcpyAsync(ld.data(), f->logdet_blk, ld.size() * sizeof(double), cudaMemcpyDeviceToHost, c->stream));
    SB_CUDA(cudaStreamSynchronize(c->stream));
    double sum = 0.0;
    for (double v : ld) sum += v;
    f->logdet = sum;
    return SB_OK;
}

// run the Cholesky on an assembled packed matrix and collect info / logdet
static int32_t factor_finish(sb_ctx* c, sb_factor* f, int64_t* info, bool force_local) {
    SB_TRY(cholesky_packed(c, f, force_local));
    long long h_info = 0;
    SB_CUDA(cudaMemcpy(&h_info, f->info_dev, sizeof(long long), cudaMemcpyDeviceToHost));
    if (h_info != 0) {
        if (info) *info = (int64_t)h_info;
        sb::set_error("matrix is not positive definite; Cholesky factorization failed at pivot " +
                      std::to_string(h_info));
        return SB_ERR_NOT_POSDEF;
    }
    return sum_logdet(c, f);
}

static int32_t factor_create_impl(sb_ctx* c, const sb_covspec* spec, const sb_noise* noise,
                                  std::unique_ptr<sb_factor>& out, int64_t* info, bool force_local) {
    SB_CHECK(spec->symmetric == 1 && spec->nrows == spec->ncols, "factor needs a symmetric square spec");
    SB_CHECK(spec->nrows > 0, "empty matrix");
    if (info) *info = 0;

    DevSpec ds(c);
    SB_TRY(ds.build(spec, c->stream, false));
    DevBuf nd(c), ndense(c);
    std::unique_ptr<sb_factor> f;
    SB_TRY(factor_alloc(c, spec->nrows, f));
    const int a_rank = force_local ? 0 : c->rank, a_world = force_local ? 1 : c->world;
    const double* noise_diag = nullptr;
    double sigma2 = 0.0;
    if (noise && noise->dense) {
        if (ndense.alloc((size_t)f->N * f->N * sizeof(double)) != SB_OK) return SB_ERR_NOMEM;
        SB_CUDA(cudaMemcpyAsync(ndense.p, noise->dense, (size_t)f->N * f->N * sizeof(double), cudaMemcpyDefault, c->stream));
    } else if (noise) {
        sigma2 = noise->sigma2;
        if (noise->diag) {
            if (nd.alloc(f->N * sizeof(double)) != SB_OK) return SB_ERR_NOMEM;
            SB_CUDA(cudaMemcpyAsync(nd.p, noise->diag, f->N * sizeof(double), cudaMemcpyDefault, c->stream));
            noise_diag = nd.d();
        }
    }
    Timer t(c, true);
    cudaEvent_t a0 = t.mark(c->stream);
    // multi-GPU: every rank assembles only the block columns it owns under the Cholesky
    // distribution (the kernel skips foreign tiles); foreign columns arrive as broadcast panels
    for (auto& b : ds.blocks) launch_assemble_packed(b, f->L, f->N, sigma2, noise_diag, c->stream, a_rank, a_world);
    if (ndense.p) launch_add_dense_lower(f->L, ndense.d(), f->N, f->N, c->stream);
    launch_fill_padding(f->L, f->N, c->stream);
    t.add(a0, t.mark(c->stream), &c->tm.assemble_ms);
    SB_CUDA(cudaGetLastError());
    SB_TRY(factor_finish(c, f.get(), info, force_local));
    t.collect();
    out = std::move(f);
    return SB_OK;
}

int32_t sb_factor_create(sb_ctx* c, const sb_covspec* spec, const sb_noise* noise, sb_factor** out,
                         int64_t* info) {
    SB_CHECK(c && spec && out, "null argument");
    Call call(c, Timed::total);
    std::unique_ptr<sb_factor> f;
    *out = nullptr;
    SB_TRY(factor_create_impl(c, spec, noise, f, info, false));
    *out = f.release();
    return call.end();
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
    *nbytes = (int64_t)sizeof(FactorBlobHeader) + (int64_t)f->L_buf.bytes + (int64_t)f->invL.bytes + (int64_t)f->alpha.bytes;
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
    SB_CUDA(cudaMemcpyAsync(p, f->L_buf, f->L_buf.bytes, cudaMemcpyDefault, c->stream));
    p += f->L_buf.bytes;
    SB_CUDA(cudaMemcpyAsync(p, f->invL, f->invL.bytes, cudaMemcpyDefault, c->stream));
    p += f->invL.bytes;
    SB_CUDA(cudaMemcpyAsync(p, f->alpha, f->alpha.bytes, cudaMemcpyDefault, c->stream));
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
    std::unique_ptr<sb_factor> f;
    SB_TRY(factor_alloc(c, h.N, f));
    const int64_t need = (int64_t)sizeof(h) + (int64_t)f->L_buf.bytes + (int64_t)f->invL.bytes + (int64_t)f->alpha.bytes;
    SB_CHECK(nbytes >= need, "factor blob truncated");
    const char* p = static_cast<const char*>(blob) + sizeof(h);
    SB_CUDA(cudaMemcpyAsync(f->L_buf, p, f->L_buf.bytes, cudaMemcpyDefault, c->stream));
    p += f->L_buf.bytes;
    SB_CUDA(cudaMemcpyAsync(f->invL, p, f->invL.bytes, cudaMemcpyDefault, c->stream));
    p += f->invL.bytes;
    SB_CUDA(cudaMemcpyAsync(f->alpha, p, f->alpha.bytes, cudaMemcpyDefault, c->stream));
    SB_CUDA(cudaStreamSynchronize(c->stream));
    f->logdet = h.logdet;
    f->has_alpha = h.has_alpha != 0;
    *out = f.release();
    return SB_OK;
}

int32_t sb_factor_logdet(sb_ctx*, sb_factor* f, double* out) {
    SB_CHECK(f && out, "null argument");
    *out = f->logdet;
    return SB_OK;
}

int32_t sb_logpdf(sb_ctx* c, sb_factor* f, const void* delta, int32_t S, double* out) {
    SB_CHECK(c && f && delta && out && S >= 1, "bad argument");
    Call call(c);
    DevBuf b(c), q(c);
    SB_TRY(b.alloc((size_t)f->Np * S * sizeof(double)));
    SB_TRY(q.alloc(S * sizeof(double)));
    SB_TRY(upload_padded(c, delta, f->N, f->Np, S, b.d()));
    Timer t(c, true);
    cudaEvent_t t0 = t.mark(c->stream);
    if (S == 1) SB_CUDA(cudaMemcpyAsync(f->vcache, b.p, f->Np * sizeof(double), cudaMemcpyDeviceToDevice, c->stream));
    tri_solve(c, f, b.d(), S, false);
    if (S == 1) {
        SB_CUDA(cudaMemcpyAsync(f->vcache + f->Np, b.p, f->Np * sizeof(double), cudaMemcpyDeviceToDevice, c->stream));
        f->vcache_valid = true;
    }
    launch_colsumsq(b.d(), f->Np, f->Np, S, q.d(), c->stream);
    t.add(t0, t.mark(c->stream), &c->tm.solve_ms);
    SB_CUDA(cudaGetLastError());
    std::vector<double> hq(S);
    SB_CUDA(cudaMemcpyAsync(hq.data(), q.p, S * sizeof(double), cudaMemcpyDeviceToHost, c->stream));
    SB_CUDA(cudaStreamSynchronize(c->stream));
    t.collect();
    const double log2pi = 1.8378770664093454835606594728112;
    for (int s = 0; s < S; s++) out[s] = -((double)f->N * log2pi + f->logdet + hq[s]) / 2.0;
    return call.end();
}

int32_t sb_factor_set_data(sb_ctx* c, sb_factor* f, const void* delta) {
    SB_CHECK(c && f && delta, "null argument");
    Call call(c);
    SB_TRY(upload_padded(c, delta, f->N, f->Np, 1, f->alpha));
    Timer t(c, true);
    cudaEvent_t t0 = t.mark(c->stream);
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
    else tri_solve(c, f, f->alpha, 1, false);
    tri_solve(c, f, f->alpha, 1, true);
    t.add(t0, t.mark(c->stream), &c->tm.solve_ms);
    SB_CUDA(cudaGetLastError());
    SB_CUDA(cudaStreamSynchronize(c->stream));
    t.collect();
    f->has_alpha = true;
    return call.end();
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

// Workspace of trsm_sweep for sweeps of up to `rows` rows: the X panels (rows x 512) and, only when asked for, the
// int8 digit planes, scales and tensor maps of X that the int8 Ozaki update reads
struct SweepWs {
    DevBuf X, planes, scale, expo;
    OzMaps maps;
    int64_t plane_rows = 0;  // 0: no planes, every sweep runs its big update on DMMA
    explicit SweepWs(sb_ctx* c) : X(c), planes(c), scale(c), expo(c) {}
    int32_t init(int64_t rows, bool int8) {
        SB_TRY(X.alloc((size_t)rows * OUTER_BLOCKS * NB * sizeof(double)));
        return int8 ? add_planes(rows) : SB_OK;
    }
    int32_t add_planes(int64_t rows) {
        plane_rows = rows;
        SB_TRY(planes.alloc(oz_planes_bytes(rows)));
        SB_TRY(scale.alloc(rows * sizeof(double)));
        SB_TRY(expo.alloc(rows * sizeof(int)));
        if (oz_make_maps(reinterpret_cast<signed char*>(planes.p), rows, &maps) != 0) {
            sb::set_error("cuTensorMapEncodeTiled failed for the X digit planes");
            return SB_ERR_CUDA;
        }
        return SB_OK;
    }
};

// W <- W L^{-T} (rows_p x Np, ld rows_p): right-looking block forward substitution, tensor-core
// products only.  keep: write the result back into W; acc != null: acc[r] += sum_c result[r,c]^2.
// Each outer step solves 4 block columns into ws.X (small in-step DMMA products) and then applies
// them to the rest of W in one big update with K = 512, which reads and writes the remaining columns
// of W once per 4 block columns.  That update runs on the int8 Ozaki kernel for an int8-Ozaki factor
// (f->oz) when ws has digit planes, and on DMMA otherwise.
static int32_t trsm_sweep(sb_ctx* c, sb_factor* f, double* W, int64_t rows_p, SweepWs& ws, bool keep, double* acc) {
    const int64_t nblk = f->L.nblk(), Np = f->Np;
    const bool oz = f->oz && ws.plane_rows > 0;
    const int64_t las[OUTER_BLOCKS] = {rows_p, rows_p, rows_p, rows_p};
    for (int64_t k0 = 0; k0 < nblk; k0 += OUTER_BLOCKS) {
        const int nq = outer_width(nblk, k0);
        const double* X[OUTER_BLOCKS];
        for (int q = 0; q < nq; q++) {
            const int64_t kq = k0 + q;
            double* Wq = W + kq * NB * rows_p;
            double* Xq = ws.X.d() + (int64_t)q * NB * rows_p;
            X[q] = Xq;
            if (q > 0) {  // bring block column kq up to date with the X panels of this outer step
                const double* Bs[OUTER_BLOCKS]; int64_t lbs[OUTER_BLOCKS];
                for (int p = 0; p < q; p++) { Bs[p] = f->L.blk(kq, k0 + p); lbs[p] = f->L.ld(k0 + p); }
                launch_gemm_nt_seg(q, X, las, Bs, lbs, Wq, rows_p, rows_p, NB, -1.0, 1.0, c->stream);
            }
            launch_gemm_nt(Wq, rows_p, f->invL + kq * (int64_t)NB * NB, NB, Xq, rows_p, rows_p, NB, NB, 1.0, 0.0, c->stream);
            if (keep) SB_CUDA(cudaMemcpyAsync(Wq, Xq, (size_t)rows_p * NB * sizeof(double), cudaMemcpyDeviceToDevice, c->stream));
            if (acc) launch_rowsumsq_acc(Xq, rows_p, rows_p, NB, acc, c->stream);
        }
        const int64_t jt = k0 + nq, m = Np - jt * NB;
        if (m <= 0) break;
        if (!oz) {  // W[:, jt..] -= [X_0 .. X_nq-1] [L(jt.., k0) .. L(jt.., k0+nq-1)]^T
            const double* Ls[OUTER_BLOCKS]; int64_t lls[OUTER_BLOCKS];
            for (int q = 0; q < nq; q++) { Ls[q] = f->L.blk(jt, k0 + q); lls[q] = f->L.ld(k0 + q); }
            launch_gemm_nt_seg(nq, X, las, Ls, lls, W + jt * NB * rows_p, rows_p, rows_p, m, -1.0, 1.0, c->stream);
            continue;
        }
        OzSrc sx{}, sl{};
        sx.nseg = sl.nseg = nq;
        for (int q = 0; q < nq; q++) {
            sx.base[q] = X[q]; sx.ld[q] = rows_p; sx.rbs[q] = NB;
            sl.base[q] = f->L.blk(jt, k0 + q); sl.ld[q] = f->L.ld(k0 + q); sl.rbs[q] = NB;
        }
        launch_oz_slice(sx, 0, rows_p / NB, 0, ws.plane_rows, ws.scale.d(), reinterpret_cast<int*>(ws.expo.p),
                        reinterpret_cast<signed char*>(ws.planes.p), c->stream);
        launch_oz_slice(sl, 0, m / NB, jt * (int64_t)NB, Np, f->oz_scale[0], f->oz_expo[0], f->oz_planes[0], c->stream);
        if (launch_gemm_ozaki(W + jt * NB * rows_p, rows_p, rows_p, m, nq, &ws.maps, ws.scale.d(), 0, &f->oz_maps[0],
                              f->oz_scale[0], jt * (int64_t)NB, c->stream) != 0) {
            sb::set_error("int8 Ozaki sweep kernel could not be launched");
            return SB_ERR_CUDA;
        }
    }
    SB_CUDA(cudaGetLastError());
    return SB_OK;
}

// Joint factor of the observations [old; new] (sb_factor_append).  h = NB floor(N1 / NB) is the head (f's full
// block columns), r = N1 - h.  Block columns j < h / NB: f's rows [NB j, N1), then the N2 rows of V = K21 L^{-T}
// (V: rows_p x Np1, ld ldv, from the sweep).  The rest: S, the factor of the Schur complement of the head,
// order r + N2, whose packed storage is the tail of the joint one (both start on the block boundary h).
static int32_t factor_splice(sb_ctx* c, const sb_factor* f, const sb_factor* S, const double* V, int64_t ldv,
                             int64_t N2, std::unique_ptr<sb_factor>& out) {
    const int64_t nh = f->N / NB, h = nh * NB;
    std::unique_ptr<sb_factor> g;
    SB_TRY(factor_alloc(c, h + S->N, g));
    SB_CHECK(g->Np - h == S->Np, "append: Schur factor does not match the joint layout");
    launch_append_relayout(g->L, f->L, f->N, N2, V, ldv, h, c->stream);
    SB_CUDA(cudaMemcpyAsync(g->L.base + g->L.off(nh), S->L.base, (size_t)S->L.total() * sizeof(double),
                            cudaMemcpyDeviceToDevice, c->stream));
    SB_CUDA(cudaMemcpyAsync(g->invL, f->invL, (size_t)h * NB * sizeof(double), cudaMemcpyDeviceToDevice, c->stream));
    SB_CUDA(cudaMemcpyAsync(g->invL + h * NB, S->invL, S->invL.bytes, cudaMemcpyDeviceToDevice, c->stream));
    SB_CUDA(cudaMemcpyAsync(g->logdet_blk, f->logdet_blk, nh * sizeof(double), cudaMemcpyDeviceToDevice, c->stream));
    SB_CUDA(cudaMemcpyAsync(g->logdet_blk + nh, S->logdet_blk, S->logdet_blk.bytes, cudaMemcpyDeviceToDevice, c->stream));
    SB_CUDA(cudaGetLastError());
    SB_TRY(sum_logdet(c, g.get()));
    out = std::move(g);
    return SB_OK;
}

// Posterior step (a): rows [lo, hi) of a cross spec (K_{*f}, or K_{*u} for VFE) assembled into the zero-padded W
// (rows_p x cols, ld rows_p), then swept by triangular factors, W <- W L^{-T}, with keep and/or a row-sum-of-squares
// accumulator (trsm_sweep).  The caller sizes the sweep workspace (ws.init) for the factors it sweeps by.
struct CrossRows {
    sb_ctx* c;
    int64_t rows_p = 0;
    DevBuf W;
    SweepWs ws;
    explicit CrossRows(sb_ctx* ctx) : c(ctx), W(ctx), ws(ctx) {}
    int32_t assemble(const DevSpec& cross, int64_t lo, int64_t hi, int64_t cols) {
        rows_p = round_up(hi > lo ? hi - lo : 1, NB);
        SB_TRY(W.alloc((size_t)rows_p * cols * sizeof(double)));
        return assemble_dense(c, clip_rows(cross, lo, hi), W.d(), rows_p, cols);
    }
    int32_t sweep(sb_factor* f, bool keep, double* acc) { return trsm_sweep(c, f, W.d(), rows_p, ws, keep, acc); }
};

// Posterior step (c): Cm = prior - W W^T (rows_p x rows_p, ld rows_p) for the Ns test points, with W = K_{*f} L^{-T}
// kept in x.W (the append splices its columns into the joint factor)
struct PosteriorCov {
    DevSpec dc, dp;
    CrossRows x;
    DevBuf Cm;
    int64_t Ns = 0;
    explicit PosteriorCov(sb_ctx* c) : dc(c), dp(c), x(c), Cm(c) {}
    int32_t build(sb_ctx* c, sb_factor* f, const sb_covspec* cross, const sb_covspec* prior) {
        Ns = cross->nrows;
        SB_TRY(dc.build(cross, c->stream, false));
        SB_CHECK(prior->nrows == Ns, "prior spec size mismatch");
        SB_TRY(dp.build(prior, c->stream, false));
        SB_TRY(x.assemble(dc, 0, Ns, f->Np));
        SB_TRY(x.ws.init(x.rows_p, f->oz));
        SB_TRY(x.sweep(f, /*keep=*/true, nullptr));
        const int64_t Nsp = x.rows_p;
        SB_TRY(Cm.alloc((size_t)Nsp * Nsp * sizeof(double)));
        SB_TRY(assemble_dense(c, dp.blocks, Cm.d(), Nsp, Nsp));
        launch_gemm_nt(x.W.d(), Nsp, x.W.d(), Nsp, Cm.d(), Nsp, Nsp, Nsp, f->Np, -1.0, 1.0, c->stream);
        SB_CUDA(cudaGetLastError());
        return SB_OK;
    }
};

// Posterior step (d): the Cholesky factor of S = (Cm + noise, with the Schur complement of f's first h rows),
// of order r + Ns.  h = r = 0 (sb_predict_factor): S is the noisy posterior covariance.  h = NB floor(N / NB),
// r = N - h (sb_factor_append): S is the Schur complement of f's head in the joint matrix, whose first r rows
// are the old rows of f's partial last block, and its factor is spliced behind that head (factor_splice).  A
// failing pivot is reported in the order of the joint matrix.
static int32_t factor_posterior(sb_ctx* c, sb_factor* f, PosteriorCov& pc, const sb_noise* noise, int64_t h, int r,
                                sb_factor** out, int64_t* info) {
    const int64_t Ns = pc.Ns, Nsp = pc.x.rows_p;
    DevBuf nd(c);
    const bool pn_dense = noise && noise->dense, pn_diag = noise && noise->diag;
    if (pn_dense || pn_diag) {
        const size_t n = pn_dense ? (size_t)Ns * Ns : (size_t)Ns;
        SB_TRY(nd.alloc(n * sizeof(double)));
        SB_CUDA(cudaMemcpyAsync(nd.p, pn_dense ? noise->dense : noise->diag, n * sizeof(double), cudaMemcpyDefault,
                                c->stream));
    }
    launch_add_noise_dense(pc.Cm.d(), Nsp, Ns, noise ? noise->sigma2 : 0.0, pn_diag && !pn_dense ? nd.d() : nullptr,
                           pn_dense ? nd.d() : nullptr, c->stream);
    std::unique_ptr<sb_factor> fn;
    SB_TRY(factor_alloc(c, r + Ns, fn));
    launch_pack_schur(fn->L, r + Ns, r, pc.Cm.d(), Nsp, r ? f->L.blk(h / NB, h / NB) : nullptr, f->L.ld(h / NB),
                      r ? pc.x.W.d() + h * Nsp : nullptr, Nsp, c->stream);
    launch_fill_padding(fn->L, r + Ns, c->stream);
    int64_t info_s = 0;
    const int32_t st = factor_finish(c, fn.get(), &info_s, /*force_local=*/true);
    if (st == SB_ERR_NOT_POSDEF) {   // S's pivot index, in the order of the joint matrix
        if (info) *info = h + info_s;
        if (h > 0)
            sb::set_error("matrix is not positive definite; Cholesky factorization failed at pivot " +
                          std::to_string(h + info_s));
    }
    SB_TRY(st);
    if (h > 0) {
        std::unique_ptr<sb_factor> joint;
        SB_TRY(factor_splice(c, f, fn.get(), pc.x.W.d(), Nsp, Ns, joint));
        fn = std::move(joint);
    }
    *out = fn.release();
    return SB_OK;
}

// Posterior step (b): mean and/or var at the test points.  Multi-GPU: every rank holds the complete factor, so the
// test points are sharded by rows (contiguous chunks, as sb_row_chunk) with no communication until the final
// all-gather of mean / var.
int32_t sb_predict(sb_ctx* c, sb_factor* f, const sb_covspec* cross, const sb_covspec* prior_diag,
                   void* mean_out, void* var_out) {
    SB_CHECK(c && f && cross, "null argument");
    SB_CHECK(cross->ncols == f->N, "cross spec must be N* x N");
    Call call(c, Timed::predict);
    const int64_t Ns_all = cross->nrows;
    if (Ns_all == 0) return SB_OK;
    SB_CHECK(!mean_out || f->has_alpha, "posterior mean requested before sb_factor_set_data");
    const bool shard = c->world > 1;
    const RowChunk rc = row_chunk(Ns_all, c->rank, c->world);
    const int64_t Ns = rc.hi - rc.lo, chunk = rc.chunk, Np = f->Np;

    DevSpec dc(c), dp(c);
    SB_TRY(dc.build(cross, c->stream, false));
    if (var_out) {
        SB_CHECK(prior_diag != nullptr, "prior spec required for var/cov");
        SB_CHECK(prior_diag->nrows == Ns_all, "prior spec size mismatch");
        SB_TRY(dp.build(prior_diag, c->stream, true));
    }
    DevBuf gath(c);  // [2][world][chunk] gather buffer (mean, var) when sharded
    if (shard) SB_TRY(gath.alloc((size_t)2 * (c->world + 1) * chunk * sizeof(double)));
    double* g_send_m = shard ? gath.d() : nullptr;                       // chunk
    double* g_send_v = shard ? gath.d() + chunk : nullptr;               // chunk
    double* g_recv_m = shard ? gath.d() + 2 * chunk : nullptr;           // world*chunk
    double* g_recv_v = shard ? gath.d() + 2 * chunk + (size_t)c->world * chunk : nullptr;
    if (shard) SB_CUDA(cudaMemsetAsync(gath.p, 0, (size_t)2 * (c->world + 1) * chunk * sizeof(double), c->stream));
    CrossRows x(c);
    SB_TRY(x.assemble(dc, rc.lo, rc.hi, Np));
    const int64_t Nsp = x.rows_p;
    DevBuf mean(c), acc(c), pd(c);
    if (mean_out) {
        SB_TRY(mean.alloc(Nsp * sizeof(double)));
        launch_gemv_n(x.W.d(), Nsp, Nsp, Np, f->alpha, mean.d(), c->stream);
        if (shard) {
            if (Ns > 0) SB_CUDA(cudaMemcpyAsync(g_send_m, mean.p, Ns * sizeof(double), cudaMemcpyDeviceToDevice, c->stream));
        } else {
            SB_CUDA(cudaMemcpyAsync(mean_out, mean.p, Ns * sizeof(double), cudaMemcpyDefault, c->stream));
        }
    }
    if (var_out) {
        SB_TRY(acc.alloc(Nsp * sizeof(double)));
        SB_CUDA(cudaMemsetAsync(acc.p, 0, Nsp * sizeof(double), c->stream));
        // rows of V^T = W L^{-T}: block forward substitution from the right, tensor-core products only
        SB_TRY(x.ws.init(Nsp, f->oz));
        SB_TRY(x.sweep(f, /*keep=*/false, acc.d()));
        SB_TRY(pd.alloc(Nsp * sizeof(double)));
        SB_TRY(assemble_diag(c, clip_rows(dp, rc.lo, rc.hi), pd.d(), Nsp));
        launch_sub(pd.d(), pd.d(), acc.d(), Ns, c->stream);
        if (shard) {
            if (Ns > 0) SB_CUDA(cudaMemcpyAsync(g_send_v, pd.p, Ns * sizeof(double), cudaMemcpyDeviceToDevice, c->stream));
        } else {
            SB_CUDA(cudaMemcpyAsync(var_out, pd.p, Ns * sizeof(double), cudaMemcpyDefault, c->stream));
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
    return call.end();
}

int32_t sb_predict_cov(sb_ctx* c, sb_factor* f, const sb_covspec* cross,
                       const sb_covspec* prior_full, void* cov_out) {
    SB_CHECK(c && f && cross && prior_full && cov_out, "null argument");
    SB_CHECK(cross->ncols == f->N, "cross spec must be N* x N");
    Call call(c, Timed::predict);
    const int64_t Ns = cross->nrows;
    if (Ns == 0) return SB_OK;
    PosteriorCov pc(c);
    SB_TRY(pc.build(c, f, cross, prior_full));
    SB_CUDA(cudaMemcpy2DAsync(cov_out, Ns * sizeof(double), pc.Cm.p, pc.x.rows_p * sizeof(double),
                              Ns * sizeof(double), Ns, cudaMemcpyDefault, c->stream));
    SB_CUDA(cudaStreamSynchronize(c->stream));
    return call.end();
}

// cholesky(cov(f_post(x*)) + noise), formed and factorised on the device
int32_t sb_predict_factor(sb_ctx* c, sb_factor* f, const sb_covspec* cross, const sb_covspec* prior_full,
                          const sb_noise* noise, sb_factor** out, int64_t* info) {
    SB_CHECK(c && f && cross && prior_full && out, "null argument");
    *out = nullptr;
    if (info) *info = 0;
    SB_CHECK(cross->ncols == f->N, "cross spec must be N* x N");
    Call call(c, Timed::predict);
    if (cross->nrows == 0) return SB_OK;
    PosteriorCov pc(c);
    SB_TRY(pc.build(c, f, cross, prior_full));
    SB_TRY(factor_posterior(c, f, pc, noise, 0, 0, out, info));
    return call.end();
}

// Sequential conditioning without refactorising (AbstractGPs update_chol): the sweep V = K21 L^{-T} and
// P = K22 + Sigma2 - V V' are sb_predict_factor's; then only the Schur complement of f's full block columns is
// factorised and spliced behind them (factor_splice).  O(N2 N1^2 + N2^2 N1 + N2^3) against (N1 + N2)^3 / 3.
int32_t sb_factor_append(sb_ctx* c, sb_factor* f, const sb_covspec* cross, const sb_covspec* prior_full,
                         const sb_noise* noise, sb_factor** out, int64_t* info) {
    SB_CHECK(c && f && cross && prior_full && out, "null argument");
    *out = nullptr;
    if (info) *info = 0;
    SB_CHECK(cross->nrows > 0, "sb_factor_append: no new observations");
    SB_CHECK(cross->ncols == f->N, "cross spec must be N* x N");
    Call call(c, Timed::predict);
    PosteriorCov pc(c);
    SB_TRY(pc.build(c, f, cross, prior_full));
    const int64_t h = f->N / NB * NB;
    SB_TRY(factor_posterior(c, f, pc, noise, h, (int)(f->N - h), out, info));
    return call.end();
}

// ---- gradients of logpdf (SURVEY 8f.1) ------------------------------------------------------------
// dlogpdf/dtheta = 1/2 tr((alpha alpha' - K^{-1}) dK/dtheta)  -- what Zygote + the ChainRules glue of
// src/affine_transformations/cross.jl:8-22 deliver in the reference (examples/getting_started/
// script.jl:154-213).  K^{-1} = L^{-T} L^{-1} is formed once with the tensor-core sweep (I L^{-T}, then
// one NT product), after which every term costs one fused O(N^2) reduction.
static __global__ void qdiag_kernel(const double* alpha, const double* Kinv, int64_t ld, int64_t n, double* out) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = 0.5 * (alpha[i] * alpha[i] - Kinv[i * ld + i]);
}

int32_t sb_logpdf_grad(sb_ctx* c, sb_factor* f, const sb_covspec* spec, double* g_terms, void* g_noise_diag) {
    SB_CHECK(c && f && spec && g_terms && g_noise_diag, "null argument");
    SB_CHECK(f->has_alpha, "sb_logpdf_grad needs alpha: call sb_factor_set_data(delta) first");
    SB_CHECK(spec->symmetric == 1 && spec->nrows == f->N && spec->ncols == f->N, "spec must be the symmetric N x N spec of the factor");
    Call call(c);
    const int64_t N = f->N, Np = f->Np;
    DevSpec ds(c);
    SB_TRY(ds.build(spec, c->stream, false));
    DevBuf W(c), Kinv(c), g(c), qd(c);
    SweepWs ws(c);
    SB_TRY(W.alloc((size_t)Np * Np * sizeof(double)));
    SB_TRY(Kinv.alloc((size_t)Np * Np * sizeof(double)));
    SB_TRY(ws.init(Np, f->oz));
    SB_TRY(g.alloc((size_t)2 * (spec->nterms > 0 ? spec->nterms : 1) * sizeof(double)));
    SB_TRY(qd.alloc((size_t)N * sizeof(double)));
    SB_CUDA(cudaMemsetAsync(W.p, 0, (size_t)Np * Np * sizeof(double), c->stream));
    SB_CUDA(cudaMemsetAsync(g.p, 0, (size_t)2 * (spec->nterms > 0 ? spec->nterms : 1) * sizeof(double), c->stream));
    launch_set_scaled_identity(W.d(), Np, 1.0, c->stream);
    SB_TRY(trsm_sweep(c, f, W.d(), Np, ws, /*keep=*/true, nullptr));                       // W = L^{-T}
    launch_gemm_nt(W.d(), Np, W.d(), Np, Kinv.d(), Np, Np, Np, Np, 1.0, 0.0, c->stream);  // K^{-1} = W W'
    for (auto& b : ds.blocks) {
        const bool offdiag = b.row0 != b.col0;   // symmetric spec: blocks (i, j), j <= i; (i, i) is the full square
        launch_grad_reduce(b, f->alpha, Kinv.d(), Np, offdiag ? 2.0 : 1.0, g.d(), c->stream);
    }
    qdiag_kernel<<<(unsigned)((N + 255) / 256), 256, 0, c->stream>>>(f->alpha, Kinv.d(), Np, N, qd.d());
    g_launch_count++;
    SB_CUDA(cudaGetLastError());
    if (spec->nterms > 0)
        SB_CUDA(cudaMemcpyAsync(g_terms, g.p, (size_t)2 * spec->nterms * sizeof(double), cudaMemcpyDefault, c->stream));
    SB_CUDA(cudaMemcpyAsync(g_noise_diag, qd.p, (size_t)N * sizeof(double), cudaMemcpyDefault, c->stream));
    SB_CUDA(cudaStreamSynchronize(c->stream));
    return call.end();
}

int32_t sb_rand(sb_ctx* c, sb_factor* f, const void* z, int32_t S, void* out) {
    SB_CHECK(c && f && z && out && S >= 1, "bad argument");
    Call call(c);
    DevBuf zb(c), ob(c);
    SB_TRY(zb.alloc((size_t)f->Np * S * sizeof(double)));
    SB_TRY(ob.alloc((size_t)f->Np * S * sizeof(double)));
    SB_TRY(upload_padded(c, z, f->N, f->Np, S, zb.d()));
    launch_trmv_lower(f->L, f->N, zb.d(), ob.d(), S, c->stream);
    SB_CUDA(cudaGetLastError());
    SB_CUDA(cudaMemcpy2DAsync(out, f->N * sizeof(double), ob.p, f->Np * sizeof(double), f->N * sizeof(double),
                              S, cudaMemcpyDefault, c->stream));
    SB_CUDA(cudaStreamSynchronize(c->stream));
    return call.end();
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
    sb_ctx* ctx;
    std::unique_ptr<sb_factor> fu;  // chol(K_uu + jitter)
    std::unique_ptr<sb_factor> fl;  // chol(A A^T + I)
    DevArray<double> alpha{ctx};    // Mp, K_*u alpha = posterior mean
    int64_t N = 0, M = 0, Mp = 0;
    explicit sb_vfe(sb_ctx* c) : ctx(c) {}
    ~sb_vfe() {   // release order fu, fl, alpha (see ~sb_factor)
        fu.reset();
        fl.reset();
    }
};

constexpr int64_t VFE_CHUNK_ROWS = 16384;  // observation rows per chunk of the K_fu stream

// s2 = sigma_i^2 of the VFE observation noise (diagonal or scalar) read to the host and checked positive, and
// sinv = sigma_i^{-1}
static int32_t vfe_noise(const sb_noise* noise, int64_t N, double* s2, double* sinv) {
    if (noise->diag) SB_CUDA(cudaMemcpy(s2, noise->diag, N * sizeof(double), cudaMemcpyDefault));
    else for (int64_t i = 0; i < N; i++) s2[i] = noise->sigma2;
    for (int64_t i = 0; i < N; i++) {
        SB_CHECK(s2[i] > 0.0, "VFE needs positive observation noise");
        sinv[i] = 1.0 / sqrt(s2[i]);
    }
    return SB_OK;
}

int32_t sb_vfe_destroy(sb_vfe* v) {
    if (!v) return SB_OK;
    cudaSetDevice(v->ctx->device);
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
    Call call(c, Timed::total);
    *out = nullptr;
    if (info) *info = 0;
    const int64_t N = xu->nrows, M = xu->ncols;
    SB_CHECK(uu->nrows == M && uu->symmetric == 1, "uu must be the symmetric M x M spec of cov(fz)");
    SB_CHECK(ff_diag->nrows == N, "ff_diag must have N rows");
    SB_CHECK(N > 0 && M > 0, "empty problem");
    SB_CHECK(noise_f->dense == nullptr, "VFE needs diagonal observation noise");

    std::unique_ptr<sb_vfe> v(new sb_vfe(c));
    SB_TRY(factor_create_impl(c, uu, noise_u, v->fu, info, /*force_local=*/true));
    v->N = N;
    v->M = M;
    v->Mp = v->fu->Np;
    const int64_t Mp = v->Mp;

    // host O(N) prep: sigma^{-1}, delta~ = delta / sigma, log det Sigma_y, |delta~|^2
    std::vector<double> hd(N), sinv(N), hnoise(N);
    SB_CUDA(cudaMemcpy(hd.data(), delta, N * sizeof(double), cudaMemcpyDefault));
    SB_TRY(vfe_noise(noise_f, N, hnoise.data(), sinv.data()));
    double logdet_sy = 0.0, dd = 0.0;
    for (int64_t i = 0; i < N; i++) {
        logdet_sy += log(hnoise[i]);
        hd[i] *= sinv[i];
        dd += hd[i] * hd[i];
    }

    DevSpec dxu(c), dff(c);
    SB_TRY(dxu.build(xu, c->stream, false));
    SB_TRY(dff.build(ff_diag, c->stream, true));

    const int64_t NC = VFE_CHUNK_ROWS;
    DevBuf dsinv(c), ddt(c), W(c), T(c), D(c), vv(c), fro(c), varf(c);
    SweepWs ws(c);
    const int64_t nchunks_total = (N + NC - 1) / NC;
    SB_TRY(dsinv.alloc(N * sizeof(double)));
    SB_TRY(ddt.alloc(round_up(N, NC) * sizeof(double)));
    SB_TRY(W.alloc((size_t)NC * Mp * sizeof(double)));
    SB_TRY(T.alloc((size_t)NC * Mp * sizeof(double)));
    SB_TRY(ws.init(NC, v->fu->oz));
    SB_TRY(D.alloc((size_t)Mp * Mp * sizeof(double)));
    SB_TRY(vv.alloc((size_t)(Mp + 8) * sizeof(double)));
    SB_TRY(fro.alloc((size_t)(nchunks_total + 1) * sizeof(double)));
    SB_TRY(varf.alloc(N * sizeof(double)));
    SB_CUDA(cudaMemcpyAsync(dsinv.p, sinv.data(), N * sizeof(double), cudaMemcpyHostToDevice, c->stream));
    SB_CUDA(cudaMemsetAsync(ddt.p, 0, round_up(N, NC) * sizeof(double), c->stream));
    SB_CUDA(cudaMemcpyAsync(ddt.p, hd.data(), N * sizeof(double), cudaMemcpyHostToDevice, c->stream));
    SB_CUDA(cudaMemsetAsync(D.p, 0, (size_t)Mp * Mp * sizeof(double), c->stream));
    SB_CUDA(cudaMemsetAsync(vv.p, 0, (size_t)(Mp + 8) * sizeof(double), c->stream));
    SB_CUDA(cudaMemsetAsync(fro.p, 0, (size_t)(nchunks_total + 1) * sizeof(double), c->stream));

    for (int64_t ci = c->rank; ci < nchunks_total; ci += c->world) {  // chunks round-robin over ranks
        const int64_t r0 = ci * NC, r1 = r0 + NC < N ? r0 + NC : N;
        const int64_t rows = r1 - r0, rows_p = round_up(rows, NB);
        SB_TRY(assemble_dense(c, clip_rows(dxu, r0, r1), W.d(), rows_p, Mp));
        launch_rowscale(W.d(), rows_p, rows, Mp, dsinv.d() + r0, c->stream);
        SB_TRY(trsm_sweep(c, v->fu.get(), W.d(), rows_p, ws, /*keep=*/true, nullptr));
        launch_colsumsq(W.d(), rows_p * Mp, 0, 1, fro.d() + ci, c->stream);
        launch_gemv_t(W.d(), rows_p, rows, Mp, ddt.d() + r0, vv.d(), c->stream);
        launch_transpose(W.d(), rows_p, rows_p, Mp, T.d(), Mp, c->stream);
        launch_gemm_nt(T.d(), Mp, T.d(), Mp, D.d(), Mp, Mp, Mp, rows_p, 1.0, 1.0, c->stream);
    }
    SB_CUDA(cudaGetLastError());
    if (c->world > 1) {
        SB_NCCL(nccl_dl::AllReduce(D.p, D.p, (size_t)Mp * Mp, ncclDouble, ncclSum, c->comm, c->stream));
        SB_NCCL(nccl_dl::AllReduce(vv.p, vv.p, (size_t)Mp, ncclDouble, ncclSum, c->comm, c->stream));
        SB_NCCL(nccl_dl::AllReduce(fro.p, fro.p, (size_t)nchunks_total, ncclDouble, ncclSum, c->comm, c->stream));
    }
    // Lambda = chol(D + I)
    SB_TRY(factor_alloc(c, M, v->fl));
    launch_pack_lower(v->fl->L, D.d(), Mp, 1.0, c->stream);
    // (padding rows/cols of D are zero: +1 on the diagonal makes them identity)
    SB_CUDA(cudaGetLastError());
    SB_TRY(factor_finish(c, v->fl.get(), info, /*force_local=*/true));
    // w = L_Lambda^{-1} (A delta~)
    DevBuf q(c);
    SB_TRY(q.alloc(sizeof(double)));
    tri_solve(c, v->fl.get(), vv.d(), 1, false);
    launch_colsumsq(vv.d(), Mp, Mp, 1, q.d(), c->stream);
    // var(f, x) for the trace term
    SB_TRY(assemble_diag(c, dff.blocks, varf.d(), N));
    std::vector<double> hvar(N), hfro(nchunks_total);
    double hq = 0.0;
    SB_CUDA(cudaMemcpyAsync(hvar.data(), varf.p, N * sizeof(double), cudaMemcpyDeviceToHost, c->stream));
    SB_CUDA(cudaMemcpyAsync(hfro.data(), fro.p, nchunks_total * sizeof(double), cudaMemcpyDeviceToHost, c->stream));
    SB_CUDA(cudaMemcpyAsync(&hq, q.p, sizeof(double), cudaMemcpyDeviceToHost, c->stream));
    // posterior weights: m_eps = L_Lambda^{-T} w ; alpha = L_u^{-T} m_eps
    tri_solve(c, v->fl.get(), vv.d(), 1, true);
    tri_solve(c, v->fu.get(), vv.d(), 1, true);
    SB_TRY(v->alpha.alloc((size_t)Mp * sizeof(double)));
    SB_CUDA(cudaMemcpyAsync(v->alpha, vv.p, v->alpha.bytes, cudaMemcpyDeviceToDevice, c->stream));
    SB_CUDA(cudaGetLastError());
    SB_CUDA(cudaStreamSynchronize(c->stream));
    double tr = 0.0, fro_sum = 0.0;
    for (int64_t i = 0; i < N; i++) tr += hvar[i] / hnoise[i];
    for (double x : hfro) fro_sum += x;
    const double log2pi = 1.8378770664093454835606594728112;
    const double dtc = -((double)N * log2pi + logdet_sy + v->fl->logdet + dd - hq) / 2.0;
    out2[0] = dtc - (tr - fro_sum) / 2.0;  // elbo
    out2[1] = dtc;
    SB_TRY(call.end());
    *out = v.release();
    return SB_OK;
}

// Gradient of the elbo (reverse mode of sb_vfe_create; DESIGN.md §4).  With A = L_u^{-1} K_uf Sigma^{-1/2},
// B = A A' + I = L_B L_B', D = B - I, alpha the handle's posterior weights, beta = Sigma^{-1}(delta - K_fu alpha)
// and E = (I - B^{-1}) L_u^{-1}, the elbo's partial derivatives are
//   d/dK_fu = beta alpha' + Sigma^{-1/2} A' E              (N x M: streamed in the chunks of sb_vfe_create)
//   d/dK_uu = -(alpha alpha' + L_u^{-T} D E) / 2            (M x M: formed once)
//   d/dK_ff[i,i] = -1 / (2 sigma_i^2)
//   d/dsigma_i^2 = (beta_i^2 - (1 - |L_B^{-1} a_i|^2) / sigma_i^2) / 2 + (k_ii - sigma_i^2 |a_i|^2) / (2 sigma_i^4)
// and every term of the three specs is reduced against its weight as in sb_logpdf_grad.  Multi-GPU: the chunk
// parts (xu, ff_diag, observation noise) are partial sums over the chunks a rank owns, combined by one
// all-reduce; the M x M part is replicated.
int32_t sb_vfe_grad(sb_ctx* c, sb_vfe* v, const sb_covspec* uu, const sb_covspec* xu, const sb_covspec* ff_diag,
                    const sb_noise* noise_f, const void* delta, double* g_uu, double* g_xu, double* g_ff,
                    void* g_noise_u_diag, void* g_noise_f_diag) {
    SB_CHECK(c && v && uu && xu && ff_diag && noise_f && delta && g_uu && g_xu && g_ff && g_noise_u_diag &&
             g_noise_f_diag, "null argument");
    const int64_t N = v->N, M = v->M, Mp = v->Mp;
    SB_CHECK(xu->nrows == N && xu->ncols == M, "xu must be the N x M spec the handle was created from");
    SB_CHECK(uu->nrows == M && uu->ncols == M && uu->symmetric == 1, "uu must be the symmetric M x M spec of cov(fz)");
    SB_CHECK(ff_diag->nrows == N && ff_diag->ncols == N, "ff_diag must be the N x N diag spec of var(f, x)");
    SB_CHECK(noise_f->dense == nullptr, "VFE needs diagonal observation noise");
    Call call(c, Timed::total);

    // host O(N) prep: [delta | sigma^2 | sigma^-1 | d elbo / d K_ff[i,i]]
    std::vector<double> hobs(4 * N);
    double* hd = hobs.data();
    double* hs2 = hd + N;
    SB_CUDA(cudaMemcpy(hd, delta, N * sizeof(double), cudaMemcpyDefault));
    SB_TRY(vfe_noise(noise_f, N, hs2, hd + 2 * N));
    for (int64_t i = 0; i < N; i++) hd[3 * N + i] = -0.5 / hs2[i];

    DevSpec duu(c), dxu(c), dff(c);
    SB_TRY(duu.build(uu, c->stream, false));
    SB_TRY(dxu.build(xu, c->stream, false));
    SB_TRY(dff.build(ff_diag, c->stream, true));
    const int64_t NC = VFE_CHUNK_ROWS < round_up(N, NB) ? VFE_CHUNK_ROWS : round_up(N, NB);
    const int64_t nchunks_total = (N + VFE_CHUNK_ROWS - 1) / VFE_CHUNK_ROWS;
    const int64_t nuu = 2 * (int64_t)uu->nterms, nxu = 2 * (int64_t)xu->nterms, nff = 2 * (int64_t)ff_diag->nterms;
    const size_t mm = (size_t)Mp * Mp;
    DevBuf obs(c), part(c), guu(c), gnu(c), Wu(c), Et(c), A1(c), A2(c), W(c), S(c), cv(c);
    SweepWs ws(c);
    SB_TRY(obs.alloc(4 * N * sizeof(double)));
    SB_TRY(part.alloc((nxu + nff + N) * sizeof(double)));   // chunk partial sums: [g_xu | g_ff | g_noise_f]
    SB_TRY(guu.alloc((nuu > 0 ? nuu : 1) * sizeof(double)));
    SB_TRY(gnu.alloc(Mp * sizeof(double)));
    for (DevBuf* b : {&Wu, &Et, &A1, &A2}) SB_TRY(b->alloc(mm * sizeof(double)));
    SB_TRY(W.alloc((size_t)NC * Mp * sizeof(double)));
    SB_TRY(S.alloc((size_t)NC * Mp * sizeof(double)));
    SB_TRY(ws.init(NC > Mp ? NC : Mp, /*int8=*/false));   // one X buffer for the prologue and the chunks
    SB_TRY(cv.alloc((size_t)5 * NC * sizeof(double)));
    const double* d_delta = obs.d();
    const double* d_s2 = obs.d() + N;
    const double* d_sinv = obs.d() + 2 * N;
    const double* d_wff = obs.d() + 3 * N;
    double* g_part_xu = part.d();
    double* g_part_ff = part.d() + nxu;
    double* g_part_nf = part.d() + nxu + nff;
    double* t = cv.d();
    double* beta = cv.d() + NC;
    double* la = cv.d() + 2 * NC;
    double* lb = cv.d() + 3 * NC;
    double* kff = cv.d() + 4 * NC;
    SB_CUDA(cudaMemcpyAsync(obs.p, hobs.data(), 4 * N * sizeof(double), cudaMemcpyHostToDevice, c->stream));
    SB_CUDA(cudaMemsetAsync(part.p, 0, part.bytes, c->stream));
    SB_CUDA(cudaMemsetAsync(guu.p, 0, guu.bytes, c->stream));

    // M^3 prologue (DMMA sweeps, as ws has no digit planes yet, and products): E^T = L_u^{-T} (I - B^{-1}) and
    // P = L_u^{-T} D E
    for (DevBuf* b : {&Wu, &A1, &A2}) SB_CUDA(cudaMemsetAsync(b->p, 0, mm * sizeof(double), c->stream));
    launch_set_scaled_identity(Wu.d(), Mp, 1.0, c->stream);
    launch_set_scaled_identity(A1.d(), Mp, 1.0, c->stream);
    launch_set_scaled_identity(A2.d(), Mp, 1.0, c->stream);
    SB_TRY(trsm_sweep(c, v->fu.get(), Wu.d(), Mp, ws, /*keep=*/true, nullptr));            // Wu = L_u^{-T}
    SB_TRY(trsm_sweep(c, v->fl.get(), A1.d(), Mp, ws, /*keep=*/true, nullptr));            // A1 = L_B^{-T}
    launch_gemm_nt(A1.d(), Mp, A1.d(), Mp, A2.d(), Mp, Mp, Mp, Mp, -1.0, 1.0, c->stream);  // A2 = I - B^{-1}
    launch_gemm_nt(Wu.d(), Mp, A2.d(), Mp, Et.d(), Mp, Mp, Mp, Mp, 1.0, 0.0, c->stream);   // E^T
    launch_unpack_lower(v->fl->L, Mp, A1.d(), c->stream);                                  // A1 = L_B
    SB_CUDA(cudaMemsetAsync(A2.p, 0, mm * sizeof(double), c->stream));
    launch_set_scaled_identity(A2.d(), Mp, -1.0, c->stream);
    launch_gemm_nt(A1.d(), Mp, A1.d(), Mp, A2.d(), Mp, Mp, Mp, Mp, 1.0, 1.0, c->stream);   // A2 = D
    launch_gemm_nt(Wu.d(), Mp, A2.d(), Mp, A1.d(), Mp, Mp, Mp, Mp, 1.0, 0.0, c->stream);   // A1 = L_u^{-T} D
    launch_gemm_nt(A1.d(), Mp, Et.d(), Mp, A2.d(), Mp, Mp, Mp, Mp, 1.0, 0.0, c->stream);   // A2 = P
    for (auto& b : duu.blocks) {
        const bool offdiag = b.row0 != b.col0;   // symmetric spec: (i, j), j < i, stands for (j, i) too
        launch_grad_reduce_outer(b, -0.5, v->alpha, v->alpha, -0.5, A2.d(), Mp, offdiag ? 2.0 : 1.0, guu.d(), c->stream);
    }
    launch_vfe_uu_diag(v->alpha, A2.d(), Mp, M, gnu.d(), c->stream);
    SB_CUDA(cudaGetLastError());

    // the observation stream: the chunks of sb_vfe_create, round-robin over ranks
    if (v->fu->oz || v->fl->oz) SB_TRY(ws.add_planes(NC));
    for (int64_t ci = c->rank; ci < nchunks_total; ci += c->world) {
        const int64_t r0 = ci * VFE_CHUNK_ROWS, r1 = r0 + VFE_CHUNK_ROWS < N ? r0 + VFE_CHUNK_ROWS : N;
        const int64_t rows = r1 - r0, rows_p = round_up(rows, NB);
        const std::vector<BlockDev> xu_rows = clip_rows(dxu, r0, r1), ff_rows = clip_rows(dff, r0, r1);
        SB_CUDA(cudaMemsetAsync(la, 0, 2 * NC * sizeof(double), c->stream));   // la, lb
        SB_TRY(assemble_dense(c, xu_rows, W.d(), rows_p, Mp));                              // K_fu rows
        launch_gemv_n(W.d(), rows_p, rows_p, Mp, v->alpha, t, c->stream);                    // t = K_fu alpha
        launch_vfe_beta(d_delta + r0, t, d_s2 + r0, rows, rows_p, beta, c->stream);
        launch_rowscale(W.d(), rows_p, rows, Mp, d_sinv + r0, c->stream);
        SB_TRY(trsm_sweep(c, v->fu.get(), W.d(), rows_p, ws, /*keep=*/true, la));           // A' rows, |a_i|^2
        launch_gemm_nt(W.d(), rows_p, Et.d(), Mp, S.d(), rows_p, rows_p, Mp, Mp, 1.0, 0.0, c->stream);
        launch_rowscale(S.d(), rows_p, rows, Mp, d_sinv + r0, c->stream);                    // S = Sigma^{-1/2} A' E
        for (auto& b : xu_rows)
            launch_grad_reduce_outer(b, 1.0, beta, v->alpha, 1.0, S.d(), rows_p, 1.0, g_part_xu, c->stream);
        SB_TRY(assemble_diag(c, ff_rows, kff, NC));
        for (auto& b : ff_rows) launch_grad_diag(b, d_wff + r0, g_part_ff, c->stream);
        SB_TRY(trsm_sweep(c, v->fl.get(), W.d(), rows_p, ws, /*keep=*/false, lb));          // |L_B^{-1} a_i|^2
        launch_vfe_noise_grad(beta, la, lb, kff, d_s2 + r0, rows, g_part_nf + r0, c->stream);
    }
    SB_CUDA(cudaGetLastError());
    if (c->world > 1)
        SB_NCCL(nccl_dl::AllReduce(part.p, part.p, (size_t)(nxu + nff + N), ncclDouble, ncclSum, c->comm, c->stream));
    if (nuu > 0) SB_CUDA(cudaMemcpyAsync(g_uu, guu.p, nuu * sizeof(double), cudaMemcpyDefault, c->stream));
    if (nxu > 0) SB_CUDA(cudaMemcpyAsync(g_xu, g_part_xu, nxu * sizeof(double), cudaMemcpyDefault, c->stream));
    if (nff > 0) SB_CUDA(cudaMemcpyAsync(g_ff, g_part_ff, nff * sizeof(double), cudaMemcpyDefault, c->stream));
    SB_CUDA(cudaMemcpyAsync(g_noise_u_diag, gnu.p, M * sizeof(double), cudaMemcpyDefault, c->stream));
    SB_CUDA(cudaMemcpyAsync(g_noise_f_diag, g_part_nf, N * sizeof(double), cudaMemcpyDefault, c->stream));
    SB_CUDA(cudaStreamSynchronize(c->stream));
    return call.end();
}

// cov(f_approx_post(x*)) = K** - B'B + (L_Lambda^{-1} B)'(L_Lambda^{-1} B),  B = L_u^{-1} K_u*
// (AbstractGPs approx posterior, SURVEY App. A).  cross: N* x M dense spec, prior_full: N* x N*.
int32_t sb_vfe_predict_cov(sb_ctx* c, sb_vfe* v, const sb_covspec* cross, const sb_covspec* prior_full,
                           void* cov_out) {
    SB_CHECK(c && v && cross && prior_full && cov_out, "null argument");
    SB_CHECK(cross->ncols == v->M, "cross spec must be N* x M");
    SB_CHECK(prior_full->nrows == cross->nrows && prior_full->ncols == cross->nrows, "prior spec must be N* x N*");
    Call call(c);
    const int64_t Ns = cross->nrows, Mp = v->Mp;
    if (Ns == 0) return SB_OK;
    DevSpec dc(c), dp(c);
    SB_TRY(dc.build(cross, c->stream, false));
    SB_TRY(dp.build(prior_full, c->stream, false));
    CrossRows x(c);
    SB_TRY(x.assemble(dc, 0, Ns, Mp));
    const int64_t Nsp = x.rows_p;
    DevBuf Cm(c);
    SB_TRY(Cm.alloc((size_t)Nsp * Nsp * sizeof(double)));
    SB_TRY(assemble_dense(c, dp.blocks, Cm.d(), Nsp, Nsp));
    SB_TRY(x.ws.init(Nsp, v->fu->oz || v->fl->oz));
    SB_TRY(x.sweep(v->fu.get(), true, nullptr));      // W = B'
    launch_gemm_nt(x.W.d(), Nsp, x.W.d(), Nsp, Cm.d(), Nsp, Nsp, Nsp, Mp, -1.0, 1.0, c->stream);
    SB_TRY(x.sweep(v->fl.get(), true, nullptr));      // W = (L_Lambda^{-1} B)'
    launch_gemm_nt(x.W.d(), Nsp, x.W.d(), Nsp, Cm.d(), Nsp, Nsp, Nsp, Mp, 1.0, 1.0, c->stream);
    SB_CUDA(cudaGetLastError());
    SB_CUDA(cudaMemcpy2DAsync(cov_out, Ns * sizeof(double), Cm.p, Nsp * sizeof(double), Ns * sizeof(double), Ns,
                              cudaMemcpyDefault, c->stream));
    SB_CUDA(cudaStreamSynchronize(c->stream));
    return call.end();
}

int32_t sb_vfe_predict(sb_ctx* c, sb_vfe* v, const sb_covspec* cross, const sb_covspec* prior_diag,
                       void* mean_out, void* var_out) {
    SB_CHECK(c && v && cross, "null argument");
    SB_CHECK(cross->ncols == v->M, "cross spec must be N* x M");
    Call call(c);
    const int64_t Ns = cross->nrows, Mp = v->Mp;
    if (Ns == 0) return SB_OK;
    DevSpec dc(c), dp(c);
    SB_TRY(dc.build(cross, c->stream, false));
    CrossRows x(c);
    SB_TRY(x.assemble(dc, 0, Ns, Mp));
    const int64_t Nsp = x.rows_p;
    DevBuf mean(c), acc1(c), acc2(c), pd(c);
    if (mean_out) {
        SB_TRY(mean.alloc(Nsp * sizeof(double)));
        launch_gemv_n(x.W.d(), Nsp, Nsp, Mp, v->alpha, mean.d(), c->stream);
        SB_CUDA(cudaMemcpyAsync(mean_out, mean.p, Ns * sizeof(double), cudaMemcpyDefault, c->stream));
    }
    if (var_out) {
        SB_CHECK(prior_diag && prior_diag->nrows == Ns, "prior diag spec required for var");
        SB_TRY(dp.build(prior_diag, c->stream, true));
        SB_TRY(acc1.alloc(Nsp * sizeof(double)));
        SB_TRY(acc2.alloc(Nsp * sizeof(double)));
        SB_TRY(pd.alloc(Nsp * sizeof(double)));
        SB_CUDA(cudaMemsetAsync(acc1.p, 0, Nsp * sizeof(double), c->stream));
        SB_CUDA(cudaMemsetAsync(acc2.p, 0, Nsp * sizeof(double), c->stream));
        // B^T = K_*u L_u^{-T} (kept), then (L_Lambda^{-1} B)^T = B^T L_Lambda^{-T}
        SB_TRY(x.ws.init(Nsp, v->fu->oz || v->fl->oz));
        SB_TRY(x.sweep(v->fu.get(), true, acc1.d()));
        SB_TRY(x.sweep(v->fl.get(), false, acc2.d()));
        SB_TRY(assemble_diag(c, dp.blocks, pd.d(), Nsp));
        launch_sub(pd.d(), pd.d(), acc1.d(), Ns, c->stream);    // k** - |B|^2
        launch_axpy1(pd.d(), acc2.d(), Ns, c->stream);          //     + |L_Lambda^{-1} B|^2
        SB_CUDA(cudaMemcpyAsync(var_out, pd.p, Ns * sizeof(double), cudaMemcpyDefault, c->stream));
    }
    SB_CUDA(cudaGetLastError());
    SB_CUDA(cudaStreamSynchronize(c->stream));
    return call.end();
}

}  // extern "C"

