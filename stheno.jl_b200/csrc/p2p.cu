// Panel exchange of the multi-GPU Cholesky drivers (cholesky.cu): peer-to-peer over CUDA IPC, or the NCCL
// broadcast where the peers cannot be mapped.
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
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "sb_host.cuh"

using namespace sb;

namespace {

constexpr int P2P_SLOTS = 2 * OUTER_BLOCKS;
constexpr int64_t P2P_HEAD_ELEMS = 2 * (int64_t)NB * NB + 32;
constexpr size_t P2P_CTR_BYTES = 4096;
constexpr size_t P2P_HEAD_OFF = P2P_CTR_BYTES;
constexpr size_t P2P_PANEL_OFF = P2P_HEAD_OFF + (size_t)P2P_SLOTS * P2P_HEAD_ELEMS * sizeof(double);
constexpr int P2P_READY = 0, P2P_ACK = 64, P2P_ERR = 128;
static_assert(P2P_PANEL_OFF % 1024 == 0, "panel slots must stay 1 KB aligned");

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

}  // namespace

// Collective: make sure every rank has an arena with panel slots for order-Np factors, mapped by all.
// Falls back (state = -1, once, on every rank together) when CUDA IPC is not available.
int32_t p2p_ensure(sb_ctx* c, int64_t Np) {
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

uint32_t* P2PRun::ctr(sb_ctx* c) const { return reinterpret_cast<uint32_t*>(c->p2p.arena); }
double* P2PRun::head(char* base, int64_t k) const {
    return reinterpret_cast<double*>(base + P2P_HEAD_OFF) + (k % P2P_SLOTS) * P2P_HEAD_ELEMS;
}
double* P2PRun::slot(char* base, int s) const { return reinterpret_cast<double*>(base + P2P_PANEL_OFF) + (int64_t)s * slot_elems; }

// Before anything is written into slot k % 8 (TRSM output, pulled slab, packed head): the last panel this
// rank OWNED in that slot (k - 8m) must have been pulled by every peer.  Acks are monotone per owner, so
// one wait per new high-water mark is enough.
int32_t p2p_slot_guard(sb_ctx* c, P2PRun& R, int64_t k, cudaStream_t st) {
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

int32_t p2p_publish(sb_ctx* c, sb_factor* f, P2PRun& R, int64_t k, cudaStream_t st) {
    const int64_t bo = k * (int64_t)NB * NB;
    p2p_pack_head_kernel<<<NB * NB / 256, 256, 0, st>>>(f->invL + bo, f->ldiag + bo, f->logdet_blk + k, R.head(c->p2p.arena, k));
    p2p_signal_kernel<<<1, 32, 0, st>>>(R.peers, c->world, c->rank, P2P_READY + c->rank, R.ord[k], -1);
    SB_CUDA(cudaGetLastError());
    return SB_OK;
}

int32_t p2p_pull(sb_ctx* c, sb_factor* f, P2PRun& R, int64_t k, int owner, int64_t slab_off, size_t slab_elems,
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

// One grouped broadcast per panel: inverse of the diagonal block, the diagonal block itself, its
// logdet share and the tiled sub-diagonal panel.  Non-owners drop L_kk into their packed matrix, so
// after the sweep every rank holds the complete factor without any extra collective.
int32_t bcast_panel(sb_ctx* c, sb_factor* f, int64_t k, double* Pslab, size_t slab_elems, int owner,
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

int32_t p2p_exchange_col(sb_ctx* c, sb_factor* f, P2PRun& R, int64_t k, cudaStream_t st) {
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

// Start of a factorisation over the IPC-mapped arena: ordinal of every panel among its owner's panels, and (on
// stream st) a wait until every panel this rank published in earlier factorisations has been pulled by everyone.
int32_t p2p_run_begin(sb_ctx* c, sb_factor* f, P2PRun& R, int world, int rank, cudaStream_t st) {
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

// panel slot s of this rank's arena: the look-ahead driver's tiled panel buffers
double* p2p_panel_slot(sb_ctx* c, const P2PRun& R, int s) { return R.slot(c->p2p.arena, s); }

// After the streams have synchronised: a waiter that timed out fails the factorisation.
int32_t p2p_check(sb_ctx* c, const P2PRun& R) {
    if (R.on) {
        uint32_t err = 0;
        SB_CUDA(cudaMemcpy(&err, R.ctr(c) + P2P_ERR, sizeof(err), cudaMemcpyDeviceToHost));
        if (err) {
            sb::set_error("peer-to-peer panel exchange timed out (a peer rank stopped making progress)");
            return SB_ERR_NCCL;
        }
    }
    return SB_OK;
}

// Context teardown.  Collective, like the communicator: no peer may still be reading this arena.
void p2p_shutdown(sb_ctx* c) {
    if (c->p2p.arena) {
        cudaStreamSynchronize(c->stream);
        cudaStreamSynchronize(c->stream2);
        if (c->comm && c->p2p.xch) nccl_barrier(c, static_cast<char*>(c->p2p.xch) + 8 * sizeof(cudaIpcMemHandle_t));
        p2p_close(c);
    }
    if (c->p2p.xch) cudaFree(c->p2p.xch);
}
