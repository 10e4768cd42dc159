// Blocked right-looking Cholesky of the packed matrix (see DESIGN.md): the serial driver, the multi-GPU look-ahead
// driver and the wide panel phase of the int8 Ozaki path.
#include "sb_host.cuh"

using namespace sb;

namespace {

// flops and launches of the trailing updates, added to the context's counters once the factorisation has succeeded
struct TrailingTally {
    double flops = 0;
    int64_t launches = 0;
    void step(int64_t nblk, int64_t k0, int nq, int rank, int world) {   // the update after the step at k0
        const int64_t tiles = syrk_packed_tiles(nblk, k0, k0 + nq, nblk, rank, world);
        if (tiles > 0) { flops += (double)tiles * 2.0 * NB * NB * ((double)nq * NB); launches++; }
    }
    void commit(sb_timings& tm) const { tm.trailing_flops += flops; tm.trailing_launches += launches; }
};

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
// trailing-update rate bench.py measured at N = 65536 on one H100 80GB (700 W), 29.2 TFLOP/s over 132 SMs.
// It sizes the multi-GPU look-ahead reservation only.  The serial-chain latencies below have not been
// measured on H100.
constexpr double DMMA_HALF_TILE_US = 37.9;
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

// Panels q0 .. q1-1 of the outer step at block column k0: column catch-up, potrf, TRSM, exchange, untile.
// tm: one comm_ms interval per panel around its exchange (empty on one rank).
static int32_t panel_phase(sb_ctx* c, sb_factor* f, int64_t k0, int q0, int q1, double* const* Pw, const double* const* Pt,
                           int rank, int world, cudaStream_t st, Timer& tm, P2PRun* R = nullptr) {
    const bool p2p = R && R->on;
    const int64_t Np = f->Np;
    for (int q = q0; q < q1; q++) {
        const int64_t kq = k0 + q;
        const int64_t mq = Np - (kq + 1) * NB;
        const int owner = (int)(kq % world);
        double* Pq = Pw[q] + tiled_panel_elems((int64_t)q * NB);
        if (owner == rank) {
            if (q > 0) launch_syrk_packed(f->L, k0, Pt, q, kq, kq + 1, rank, world, st);
            launch_potrf_inv(f->L, kq, f->N, f->invL, f->logdet_blk, f->info_dev, st, world > 1 ? f->ldiag.d() : nullptr);
            if (p2p) SB_TRY(p2p_slot_guard(c, *R, kq, st));
            if (mq > 0)
                launch_trsm_tiled(f->L.blk(kq + 1, kq), f->L.ld(kq), f->invL + kq * (int64_t)NB * NB, Pq, mq, st);
        }
        cudaEvent_t x0 = tm.mark(st);
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
        tm.add(x0, tm.mark(st), &c->tm.comm_ms);
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

// Serial part of the wide panel phase (panel stream): column exchange, the 512 x 512 diagonal block, inv(L_512)
// and its digit planes.  Only small kernels: it runs on the few SMs the first part of T^B leaves free.
static int32_t wide_diag_phase(sb_ctx* c, sb_factor* f, int64_t k0, int nq, int rank, int world, cudaStream_t st,
                               Timer& tm, P2PRun* R) {
    const int64_t nblk = f->L.nblk();
    const bool bulk = nblk - (k0 + nq) > 0;            // rows under the step (then nq == OUTER_BLOCKS)
    if (world > 1) {
        if (!(R && R->on)) {
            sb::set_error("wide panel phase needs the peer-to-peer arena");
            return SB_ERR_UNSUPPORTED;
        }
        cudaEvent_t x0 = tm.mark(st);
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
        tm.add(x0, tm.mark(st), &c->tm.comm_ms);
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
    for (int q = 0; q < OUTER_BLOCKS; q++) {
        ws.base[q] = f->wide_W + (int64_t)q * NB * WIDE; ws.ld[q] = WIDE; ws.rbs[q] = NB;
        ws.diag[q] = f->L.blk(k0 + q, k0 + q); ws.dld[q] = f->L.ld(k0 + q);
    }
    ws.colsign = +1;   // column k of inv(L_512) times 2^ilogb(L_kk): see wide_bulk_phase
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
        as.diag[q] = f->L.blk(k0 + q, k0 + q); as.dld[q] = f->L.ld(k0 + q);
    }
    // Equilibrated panel solve: X = (A21 E^-1)(inv(L_512) E)^T with E = diag(2^ilogb(L_kk)).  A21[i, k] is of the
    // order of L21[i, k] L_kk, so without E the digit planes of a row would span the range of the step's diagonal
    // (for a diagonally scaled matrix D A D up to 2^60), and the small entries would lose their digits.
    as.colsign = -1;
    launch_oz_slice(as, 0, below, r0 * NB, Np, f->oz_scale[set], f->oz_expo[set], f->oz_planes[set], st);
    as.colsign = 0;    // the planes of X = L21 for the trailing update: rows only
    if (launch_panel_solve_ozaki(xcol, ldx, below * NB, &f->oz_maps[set], f->oz_scale[set], r0 * NB, &f->wide_wmaps,
                                 f->wide_wscale, st) != 0) {
        sb::set_error("int8 Ozaki panel solve failed to launch");
        return SB_ERR_CUDA;
    }
    launch_oz_slice(as, 0, below, r0 * NB, Np, f->oz_scale[set], f->oz_expo[set], f->oz_planes[set], st);
    SB_CUDA(cudaGetLastError());
    return SB_OK;
}

// End of a two-stream factorisation: the trailing stream waits for the panel stream and the host for both, a
// timed-out peer exchange fails the factorisation, and the driver's intervals (fine timing) are added up.
static int32_t finish_two_streams(sb_ctx* c, const P2PRun& R, Timer& tm) {
    cudaEvent_t e_pend = c->next_event();
    SB_CUDA(cudaEventRecord(e_pend, c->stream2));
    SB_CUDA(cudaStreamWaitEvent(c->stream, e_pend, 0));
    SB_CUDA(cudaGetLastError());
    SB_CUDA(cudaStreamSynchronize(c->stream));
    SB_TRY(p2p_check(c, R));
    tm.collect();   // exchange time includes waiting for the owner's panel work on the other ranks
    return SB_OK;
}

// Look-ahead factorisation (see above).  Panels move by the P2P exchange when the arena is mapped, else by the
// NCCL broadcast.
static int32_t cholesky_lookahead(sb_ctx* c, sb_factor* f, int world, int rank) {
    const int64_t nblk = f->L.nblk(), Np = f->Np;
    Timer tm(c, c->fine_timing);
    cudaStream_t s1 = c->stream, s2 = c->stream2;
    const int64_t nsteps = (nblk + OUTER_BLOCKS - 1) / OUTER_BLOCKS;
    double* Pw[2][OUTER_BLOCKS];
    const double* Pt[2][OUTER_BLOCKS];
    for (int set = 0; set < 2; set++)
        for (int q = 0; q < OUTER_BLOCKS; q++)
            Pt[set][q] = Pw[set][q] = f->panel + (int64_t)(set * OUTER_BLOCKS + q) * tiled_panel_elems(Np);
    std::vector<cudaEvent_t> ev_p(nsteps), ev_a(nsteps);
    for (int64_t s = 0; s < nsteps; s++) {
        ev_p[s] = c->next_event(); ev_a[s] = c->next_event();
    }
    cudaEvent_t e_start = c->next_event();
    // stream 2 starts after everything already queued on stream 1 (assembly)
    SB_CUDA(cudaEventRecord(e_start, s1));
    SB_CUDA(cudaStreamWaitEvent(s2, e_start, 0));
    P2PRun R;
    if (c->p2p.state == 1) {
        SB_TRY(p2p_run_begin(c, f, R, world, rank, s2));
        for (int set = 0; set < 2; set++)   // the arena slots ARE the tiled panel buffers
            for (int q = 0; q < OUTER_BLOCKS; q++) Pt[set][q] = Pw[set][q] = p2p_panel_slot(c, R, set * OUTER_BLOCKS + q);
    }
    {
        const int nq0 = outer_width(nblk, 0);
        SB_TRY(panel_phase(c, f, 0, 0, nq0, Pw[0], Pt[0], rank, world, s2, tm, &R));
        SB_CUDA(cudaEventRecord(ev_p[0], s2));
        tm.add(e_start, ev_p[0], &c->tm.panel_ms);  // only the first, un-hidden panel phase is on the critical path
    }
    TrailingTally tally;
    for (int64_t s = 0; s < nsteps; s++) {
        const int64_t k0 = s * OUTER_BLOCKS;
        const int nq = outer_width(nblk, k0);
        const int set = (int)(s & 1);
        const int64_t jt = k0 + nq;
        SB_CUDA(cudaStreamWaitEvent(s1, ev_p[s], 0));
        cudaEvent_t t0 = tm.mark(s1);
        if (jt < nblk) {
            const int64_t jA = jt + OUTER_BLOCKS < nblk ? jt + OUTER_BLOCKS : nblk;
            launch_syrk_packed(f->L, k0, Pt[set], nq, jt, jA, rank, world, s1);              // T^A: next panels' columns
            SB_CUDA(cudaEventRecord(ev_a[s], s1));
            if (s + 1 < nsteps) {
                const int nq1 = outer_width(nblk, jt);
                SB_CUDA(cudaStreamWaitEvent(s2, ev_a[s], 0));
                cudaEvent_t ch = tm.mark(s2);
                SB_TRY(panel_phase(c, f, jt, 0, nq1, Pw[set ^ 1], Pt[set ^ 1], rank, world, s2, tm, &R));
                SB_CUDA(cudaEventRecord(ev_p[s + 1], s2));
                tm.add(ch, tm.mark(s2), &c->tm.panel_chain_ms);
            }
            if (jA < nblk) {                                                                // T^B
                const double tilesB = 2.0 * (double)syrk_packed_tiles(nblk, k0, jA, nblk, rank, world);
                const int nq1 = outer_width(nblk, jt);
                const int reserve = (s + 1 < nsteps)
                    ? pick_lookahead_sms(c->num_sms, tilesB, nq1, Np - (jt + 1) * NB) : 0;
                launch_syrk_packed(f->L, k0, Pt[set], nq, jA, nblk, rank, world, s1, reserve);
            }
            tally.step(nblk, k0, nq, rank, world);
        }
        tm.add_trailing(t0, tm.mark(s1));
    }
    SB_TRY(finish_two_streams(c, R, tm));
    tally.commit(c->tm);
    return SB_OK;
}

// Factorisation with the wide panel phase (int8 Ozaki path).  Per outer step s, on the trailing stream:
//   T^A_s | T^B_s part 1 (leaves a few SMs free) | panel solve of step s+1 (whole GPU) | T^B_s part 2 (whole GPU)
// and on the panel stream, under T^B_s part 1: column exchange + diagonal block + inv(L_512) of step s+1.
// Part 1 is sized to the duration of that serial chain, so the SM reservation costs ~ 8 / 132 of the GPU for that long per step.
static int32_t cholesky_wide(sb_ctx* c, sb_factor* f, int world, int rank) {
    const int64_t nblk = f->L.nblk();
    Timer tm(c, c->fine_timing);
    cudaStream_t s1 = c->stream, s2 = c->stream2;
    const int64_t nsteps = (nblk + OUTER_BLOCKS - 1) / OUTER_BLOCKS;
    std::vector<cudaEvent_t> ev_d(nsteps), ev_a(nsteps);
    for (int64_t s = 0; s < nsteps; s++) {
        ev_d[s] = c->next_event(); ev_a[s] = c->next_event();
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
        const int nq = outer_width(nblk, k0);
        const int set = (int)(s & 1);
        SB_CUDA(cudaStreamWaitEvent(s1, ev_d[s], 0));
        cudaEvent_t b0 = tm.mark(s1);
        SB_TRY(wide_bulk_phase(c, f, k0, nq, set, s1));
        cudaEvent_t b1 = tm.mark(s1);
        tm.add(b0, b1, &c->tm.panel_ms);          // panel solves are on the critical path (whole GPU)
        if (s > 0) tm.add_trailing(b0, b1, -1.0);  // and lie in step s-1's trailing interval (the first precedes them all)
        return SB_OK;
    };
    auto diag = [&](int64_t s) -> int32_t {      // serial part of step s, panel stream
        const int64_t k0 = s * OUTER_BLOCKS;
        const int nq = outer_width(nblk, k0);
        cudaEvent_t ch = tm.mark(s2);
        SB_TRY(wide_diag_phase(c, f, k0, nq, rank, world, s2, tm, &R));
        SB_CUDA(cudaEventRecord(ev_d[s], s2));
        tm.add(ch, tm.mark(s2), &c->tm.panel_chain_ms);
        return SB_OK;
    };
    SB_TRY(diag(0));
    tm.add(e_start, ev_d[0], &c->tm.panel_ms);     // the first serial phase is not hidden
    SB_TRY(bulk(0));
    TrailingTally tally;
    for (int64_t s = 0; s < nsteps; s++) {
        const int64_t k0 = s * OUTER_BLOCKS;
        const int nq = outer_width(nblk, k0);
        const int set = (int)(s & 1);
        const int64_t jt = k0 + nq;
        cudaEvent_t t0 = tm.mark(s1);
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
            tally.step(nblk, k0, nq, rank, world);
        }
        tm.add_trailing(t0, tm.mark(s1));
    }
    SB_TRY(finish_two_streams(c, R, tm));
    tally.commit(c->tm);
    c->tm.trailing_int8_ops += 28.0 * tally.flops;
    return SB_OK;
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

}  // namespace

int32_t cholesky_packed(sb_ctx* c, sb_factor* f, bool force_local) {
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
    Timer tm(c, c->fine_timing);
    TrailingTally tally;
    // the OUTER_BLOCKS panels of an outer step, each in TILED layout (gemm_nt.cu); row block 0 <->
    // block row k0+1, panel q starts at row block q
    const double* Pt[OUTER_BLOCKS];
    double* Pw[OUTER_BLOCKS];
    for (int q = 0; q < OUTER_BLOCKS; q++) Pt[q] = Pw[q] = f->panel + (int64_t)q * tiled_panel_elems(Np);
    for (int64_t k0 = 0; k0 < nblk; k0 += OUTER_BLOCKS) {
        const int nq = outer_width(nblk, k0);
        // One panel at a time: the panel work up to the exchange is timed as panel_ms, the exchange as comm_ms.  Of
        // the untiles after the exchanges, only the last one before a trailing update is timed (as panel_ms).
        cudaEvent_t untiled = nullptr;
        for (int q = 0; q < nq; q++) {
            cudaEvent_t p0 = tm.mark(st);
            SB_TRY(panel_phase(c, f, k0, q, q + 1, Pw, Pt, rank, world, st, tm));
            if (tm.on) {
                const Timer::Span x = tm.spans.back();   // panel_phase's last interval: this panel's exchange
                tm.add(p0, x.a, &c->tm.panel_ms);
                untiled = x.b;
            }
        }
        const int64_t jt = k0 + nq;  // first trailing block column
        if (jt < nblk) {
            cudaEvent_t t0 = tm.mark(st);
            tm.add(untiled, t0, &c->tm.panel_ms);
            launch_syrk_packed(f->L, k0, Pt, nq, jt, nblk, rank, world, st);
            tm.add_trailing(t0, tm.mark(st));
            tally.step(nblk, k0, nq, rank, world);
        }
    }
    if (world > 1) SB_TRY(sync_info(c, f));
    SB_CUDA(cudaGetLastError());
    SB_CUDA(cudaStreamSynchronize(st));
    tm.collect();
    tally.commit(c->tm);
    return SB_OK;
}
