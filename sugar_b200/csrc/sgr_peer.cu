// sgr_peer.cu -- the view-parallel exchange over PEER MEMORY (NVLink 5 / NVSwitch): the ranks map each other's
// exchange buffers with CUDA IPC and the kernels of this file move the data themselves; there is no NCCL call and
// no host callback on the data path of a backward.  Driven by sugar_b200/parallel.py (ViewParallel, peer mode);
// the reference has no counterpart (1 view / 1 GPU, sugar_trainers/coarse_sdf.py:98,507).
//
// Every rank owns ONE peer-visible allocation (sgr_peer_alloc), laid out by the caller:
//     flags     u32[PEER_SLOTS][PEER_RANKS]  word [slot][j] is written by rank j only, monotonically (a step counter)
//     F0, F1    f32[3P+4]     this rank's SH factor block (dL/dRGB per Gaussian + its camera position), double-buffered by
//                             step parity (peers may still read step k-1's while step k's blend pass accumulates)
//     S         f32[11P+]     the 44-byte gradient records summed over the ranks (written by the owners of each slice)
//     STAGE[j]  f32[11P+]     records computed by rank j for the blocks THIS rank owns (j = 0 .. N-1, own included)
// Stream picture of one backward on rank r (main = the caller's stream, B = a high-priority side stream):
//     main  memset  blend ─sig(BLEND)─ wait(BLEND, all ranks) ─ pb chunk 0 ─sig(CHUNK 0)─ pb chunk 1 ─sig(CHUNK 1)─ ...  wait(B)
//              pb = the per-Gaussian pass (sgr_backward.cu, MULTI): bulk-loads (TMA) the other ranks' factor blocks of
//              its 64 Gaussians straight from their memory and writes dL_dsh summed over ALL views -- the all-gather is
//              fused into the consumer; bulk-stores (TMA) its 64 records into the staging array of the rank that owns
//              them -- the reduce-scatter is fused into the producer
//     B     wait(CHUNK 0, all) ─ reduce: sum the owned slice of chunk 0 over STAGE[0..N-1] (local loads), store the sums
//           into every rank's S (posted NVLink writes) ─sig(REDUCED 0)─ wait(CHUNK 1, all) ─ reduce ─ ... ; behind the
//           reduce of chunk c: wait(REDUCED c-1, all) ─ split S of chunk c-1 into the gradient arrays
// Chunks halve in size (SgrBackwardPlan.chunk_taper), so what is left after the last one is small.  A rank's main stream
// waits for its peers once per backward (BLEND); a wait that outlives its timeout traps (the context dies with an error
// instead of hanging the box).
#include <stdio.h>
#include <string.h>

#include <mutex>

#include "sgr_internal.cuh"

namespace sgr {

constexpr int PEER_RANKS = SGR_PEER_MAX_RANKS;  // flag row width (words)
constexpr int PEER_SLOTS = SGR_PEER_MAX_SLOTS;

__device__ __forceinline__ void st_release_sys(uint32_t *p, uint32_t v)
{
    asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t *p)
{
    uint32_t v;
    asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ uint32_t ld_relaxed_sys(const uint32_t *p)
{
    uint32_t v;
    asm volatile("ld.relaxed.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}

// Thread j tells rank j that this rank reached `slot` of step `seq`.  The signal is a kernel of its own: everything this
// rank enqueued on the stream before it has COMPLETED (stream order; a grid is complete only when its stores, local or
// into peer memory, have been performed) and sits in the owning GPU's L2, the point of coherence peers read through.
// The release store orders the flag behind them without a separate system-wide fence instruction.
__global__ void peer_signal_kernel(uint32_t *const *__restrict__ flag_tab, int nranks, int slot, int my_rank, uint32_t seq)
{
    const int j = threadIdx.x;
    if (j < nranks) st_release_sys(flag_tab[j] + (size_t)slot * PEER_RANKS + my_rank, seq);
}

// Block until every rank's word of the slots [slot0, slot0 + nslots) has reached `seq` (wrap-safe compare).
__global__ void peer_wait_kernel(const uint32_t *__restrict__ flags, int nranks, int slot0, int nslots, uint32_t seq,
                                 long long timeout_cycles)
{
    for (int idx = threadIdx.x; idx < nslots * nranks; idx += blockDim.x) {
        const uint32_t *w = flags + (size_t)(slot0 + idx / nranks) * PEER_RANKS + idx % nranks;
        // relaxed polls (each goes to L2, where the peers' flag stores land); one acquire once the word is there
        if ((int32_t)(ld_relaxed_sys(w) - seq) >= 0) {
            (void)ld_acquire_sys(w);
            continue;
        }
        const long long t0 = clock64();
        while ((int32_t)(ld_acquire_sys(w) - seq) < 0) {
            __nanosleep(32);
            if (clock64() - t0 > timeout_cycles) {
                printf("sugar_b200: peer wait timed out (slot %d, rank %d, seq %u, saw %u)\n", slot0 + idx / nranks,
                       idx % nranks, seq, ld_acquire_sys(w));
                __trap();
            }
        }
    }
}

// Flag handshake folded into a kernel (saves the microsecond-sized launches around it):
//  begin  threads 0 .. nranks-1 of every CTA poll the LOCAL flag words of `wait_slot` until all ranks reached `seq`;
//  end    every thread fences its stores system-wide, the CTAs count themselves on a local counter, and the last one
//         to finish writes `seq` into word [signal_slot][my_rank] of every rank's flags (and re-arms the counter).
struct PeerSync {
    const uint32_t *flags;      // local flag words; NULL: no wait
    uint32_t *const *flag_tab;  // every rank's flag words; NULL: no signal
    unsigned int *counter;      // local, zero between launches
    int wait_slot, signal_slot, nranks, my_rank;
    uint32_t seq;
    long long timeout_cycles;
};

__device__ __forceinline__ void peer_sync_begin(const PeerSync &s)
{
    if (!s.flags) return;
    if ((int)threadIdx.x < s.nranks) {
        const uint32_t *w = s.flags + (size_t)s.wait_slot * PEER_RANKS + threadIdx.x;
        if ((int32_t)(ld_relaxed_sys(w) - s.seq) < 0) {
            const long long t0 = clock64();
            while ((int32_t)(ld_relaxed_sys(w) - s.seq) < 0) {
                __nanosleep(32);
                if (clock64() - t0 > s.timeout_cycles) {
                    printf("sugar_b200: peer wait timed out in a fused kernel (slot %d, rank %d, seq %u)\n", s.wait_slot,
                           (int)threadIdx.x, s.seq);
                    __trap();
                }
            }
        }
        (void)ld_acquire_sys(w);
    }
    __syncthreads();
}

__device__ __forceinline__ void peer_sync_end(const PeerSync &s)
{
    if (!s.flag_tab) return;
    __shared__ int s_last;
    __threadfence_system();  // this thread's stores, local and into peer memory, are performed before what follows
    __syncthreads();
    if (threadIdx.x == 0) s_last = atomicAdd(s.counter, 1u) == gridDim.x - 1;
    __syncthreads();
    if (s_last) {
        if (threadIdx.x == 0) atomicExch(s.counter, 0u);
        __threadfence_system();  // the other CTAs' increments (each behind its own fence) have been observed
        if ((int)threadIdx.x < s.nranks)
            st_release_sys(s.flag_tab[threadIdx.x] + (size_t)s.signal_slot * PEER_RANKS + s.my_rank, s.seq);
    }
}

// Two-shot all-reduce of the record units [q0, q1) (16-byte units) this rank owns: loads from every rank's R in rank
// order (so the sum is the same bits whoever owns the slice), stores into every rank's S.  All of a thread's loads are
// issued before the first add: what hides the NVLink round trip is bytes in flight.
template <int NR>
__global__ void __launch_bounds__(256) peer_reduce_kernel(const float4 *const *__restrict__ rec_tab,
                                                          float4 *const *__restrict__ sum_tab, int nranks, size_t q0,
                                                          size_t q1, const PeerSync sync)
{
    peer_sync_begin(sync);
    const float4 *src[NR];
    float4 *dst[NR];
#pragma unroll
    for (int j = 0; j < NR; j++) {
        src[j] = rec_tab[j < nranks ? j : 0];
        dst[j] = sum_tab[j < nranks ? j : 0];
    }
    // U units per thread and trip, U * NR 16-byte loads in flight per thread: the kernel runs on a few CTAs per SM
    // (it shares the GPU with the per-Gaussian pass of the next chunk) and still covers the NVLink round trip
    constexpr int U = NR <= 2 ? 4 : (NR <= 4 ? 2 : 1);
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    for (size_t qb = q0 + (size_t)blockIdx.x * blockDim.x + threadIdx.x; qb < q1; qb += stride * U) {
        float4 v[U][NR];
#pragma unroll
        for (int u = 0; u < U; u++) {
            const size_t q = qb + (size_t)u * stride;
#pragma unroll
            for (int j = 0; j < NR; j++)
                if (j < nranks && q < q1) v[u][j] = __ldcg(src[j] + q);
        }
#pragma unroll
        for (int u = 0; u < U; u++) {
            const size_t q = qb + (size_t)u * stride;
            if (q >= q1) break;
            float4 a = v[u][0];
#pragma unroll
            for (int j = 1; j < NR; j++)
                if (j < nranks) {
                    a.x += v[u][j].x;
                    a.y += v[u][j].y;
                    a.z += v[u][j].z;
                    a.w += v[u][j].w;
                }
#pragma unroll
            for (int j = 0; j < NR; j++)
                if (j < nranks) __stcg(dst[j] + q, a);
        }
    }
    peer_sync_end(sync);
}

// any number of ranks (tables read per element)
__global__ void __launch_bounds__(256) peer_reduce_generic_kernel(const float4 *const *__restrict__ rec_tab,
                                                                  float4 *const *__restrict__ sum_tab, int nranks,
                                                                  size_t q0, size_t q1, const PeerSync sync)
{
    peer_sync_begin(sync);
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    for (size_t q = q0 + (size_t)blockIdx.x * blockDim.x + threadIdx.x; q < q1; q += stride) {
        float4 a = __ldcg(rec_tab[0] + q);
        for (int j = 1; j < nranks; j++) {
            const float4 v = __ldcg(rec_tab[j] + q);
            a.x += v.x;
            a.y += v.y;
            a.z += v.z;
            a.w += v.w;
        }
        for (int j = 0; j < nranks; j++) __stcg(sum_tab[j] + q, a);
    }
    peer_sync_end(sync);
}

}  // namespace sgr

extern "C" {
using namespace sgr;

int sgr_peer_alloc(size_t bytes, void **ptr)
{
    if (!ptr || bytes == 0) {
        set_error("bad arguments to sgr_peer_alloc");
        return SGR_EINVAL;
    }
    *ptr = nullptr;
    void *p = nullptr;
    SGR_CUDA(cudaMalloc(&p, bytes));  // a whole cudaMalloc allocation: its IPC handle maps it at offset 0
    cudaError_t e = cudaMemset(p, 0, bytes);
    if (e != cudaSuccess) {
        cudaFree(p);
        return cuda_fail(e, "cudaMemset");
    }
    SGR_CUDA(cudaDeviceSynchronize());
    *ptr = p;
    return SGR_OK;
}

int sgr_peer_free(void *ptr)
{
    if (ptr) SGR_CUDA(cudaFree(ptr));
    return SGR_OK;
}

int sgr_peer_export(const void *ptr, void *handle64)
{
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle size");
    if (!ptr || !handle64) {
        set_error("bad arguments to sgr_peer_export");
        return SGR_EINVAL;
    }
    cudaIpcMemHandle_t h;
    SGR_CUDA(cudaIpcGetMemHandle(&h, (void *)ptr));
    memcpy(handle64, &h, 64);
    return SGR_OK;
}

int sgr_peer_import(const void *handle64, void **ptr)
{
    if (!ptr || !handle64) {
        set_error("bad arguments to sgr_peer_import");
        return SGR_EINVAL;
    }
    cudaIpcMemHandle_t h;
    memcpy(&h, handle64, 64);
    *ptr = nullptr;
    SGR_CUDA(cudaIpcOpenMemHandle(ptr, h, cudaIpcMemLazyEnablePeerAccess));
    return SGR_OK;
}

int sgr_peer_close(void *ptr)
{
    if (ptr) SGR_CUDA(cudaIpcCloseMemHandle(ptr));
    return SGR_OK;
}

size_t sgr_peer_flag_bytes(void) { return (size_t)PEER_SLOTS * PEER_RANKS * sizeof(uint32_t); }

int sgr_peer_signal(void *const *flag_tab, int32_t nranks, int32_t slot, int32_t my_rank, uint32_t seq, void *stream)
{
    if (!flag_tab || nranks < 1 || nranks > PEER_RANKS || slot < 0 || slot >= PEER_SLOTS || my_rank < 0 ||
        my_rank >= nranks) {
        set_error("bad arguments to sgr_peer_signal");
        return SGR_EINVAL;
    }
    cudaStream_t st = (cudaStream_t)stream;
    SGR_LAUNCH(K_PEER_SYNC, st,
               peer_signal_kernel<<<1, 32 * ((nranks + 31) / 32), 0, st>>>((uint32_t *const *)flag_tab, nranks, slot, my_rank,
                                                                          seq));
    SGR_CUDA(cudaGetLastError());
    return SGR_OK;
}

int sgr_peer_wait(const void *flags, int32_t nranks, int32_t slot0, int32_t nslots, uint32_t seq, double timeout_s,
                  void *stream)
{
    if (!flags || nranks < 1 || nranks > PEER_RANKS || slot0 < 0 || nslots < 1 || slot0 + nslots > PEER_SLOTS) {
        set_error("bad arguments to sgr_peer_wait");
        return SGR_EINVAL;
    }
    cudaStream_t st = (cudaStream_t)stream;
    const long long cycles = (long long)((timeout_s > 0 ? timeout_s : 20.0) * 1.9e9);
    SGR_LAUNCH(K_PEER_SYNC, st,
               peer_wait_kernel<<<1, 32 * ((nslots * nranks + 31) / 32 > 4 ? 4 : (nslots * nranks + 31) / 32), 0, st>>>(
                   (const uint32_t *)flags, nranks, slot0, nslots, seq, cycles));
    SGR_CUDA(cudaGetLastError());
    return SGR_OK;
}

int sgr_peer_reduce_records_synced(const void *const *rec_tab, void *const *sum_tab, int32_t nranks, int32_t my_rank,
                                   int32_t p0, int32_t p1, const void *flags, int32_t wait_slot, void *const *flag_tab,
                                   int32_t signal_slot, uint32_t seq, void *counter, double timeout_s, void *stream)
{
    if (!rec_tab || !sum_tab || nranks < 1 || nranks > PEER_RANKS || my_rank < 0 || my_rank >= nranks || p0 < 0 ||
        p1 < p0 || (p0 & 63) || (flags && (wait_slot < 0 || wait_slot >= PEER_SLOTS)) ||
        (flag_tab && (signal_slot < 0 || signal_slot >= PEER_SLOTS || !counter))) {
        set_error("bad arguments to sgr_peer_reduce_records_synced (p0 must be a multiple of 64)");
        return SGR_EINVAL;
    }
    // ownership follows the per-Gaussian pass (PreBwdArgs::stage_tab): block b of the chunk's nb 64-record blocks belongs
    // to rank b * nranks / nb, i.e. this rank owns the blocks [ceil(r nb / n), ceil((r + 1) nb / n)).  One block = 176
    // 16-byte units; the chunk's last block may be partial (its last unit may run up to 12 bytes past record p1 - 1: the
    // arrays are padded).
    const int64_t nb = ((int64_t)(p1 - p0) + 63) / 64;
    const int64_t bs = (nb * my_rank + nranks - 1) / nranks, be = (nb * (my_rank + 1) + nranks - 1) / nranks;
    const size_t Q0 = (size_t)p0 * 11 / 4, Qend = ((size_t)p1 * 11 + 3) / 4;
    size_t q0 = Q0 + (size_t)bs * 176, q1 = Q0 + (size_t)be * 176;
    if (q1 > Qend) q1 = Qend;
    if (q0 > q1) q0 = q1;
    if (q1 == q0 && !flag_tab) return SGR_OK;  // nothing owned and nobody to tell
    cudaStream_t st = (cudaStream_t)stream;
    const int T = 256;
    // at most 2 CTAs of 256 threads per SM, grid-stride over the slice
    size_t blocks = (q1 - q0 + T - 1) / T;
    const size_t cap = (size_t)device_sm_count() * 2;
    if (blocks > cap) blocks = cap;
    if (blocks == 0) blocks = 1;  // the handshake still runs
    PeerSync sy;
    sy.flags = (const uint32_t *)flags;
    sy.flag_tab = (uint32_t *const *)flag_tab;
    sy.counter = (unsigned int *)counter;
    sy.wait_slot = wait_slot;
    sy.signal_slot = signal_slot;
    sy.nranks = nranks;
    sy.my_rank = my_rank;
    sy.seq = seq;
    sy.timeout_cycles = (long long)((timeout_s > 0 ? timeout_s : 20.0) * 1.9e9);
    const float4 *const *rt = (const float4 *const *)rec_tab;
    float4 *const *stb = (float4 *const *)sum_tab;
    SGR_LAUNCH(K_PEER_REDUCE, st,
               if (nranks <= 2) peer_reduce_kernel<2><<<(unsigned)blocks, T, 0, st>>>(rt, stb, nranks, q0, q1, sy);
               else if (nranks <= 4) peer_reduce_kernel<4><<<(unsigned)blocks, T, 0, st>>>(rt, stb, nranks, q0, q1, sy);
               else if (nranks <= 8) peer_reduce_kernel<8><<<(unsigned)blocks, T, 0, st>>>(rt, stb, nranks, q0, q1, sy);
               else peer_reduce_generic_kernel<<<(unsigned)blocks, T, 0, st>>>(rt, stb, nranks, q0, q1, sy));
    SGR_CUDA(cudaGetLastError());
    return SGR_OK;
}

}  // extern "C"

namespace sgr {

// The events that order the exchange's launches on the plan's signal stream (side = 0) and side stream (side = 1)
// behind earlier work, per device and launch index (< 20: rasterize_backward bounds the chunks), kept once created.
static int peer_event(int side, int index, cudaEvent_t *out)
{
    static std::mutex mu;
    static cudaEvent_t evs[SGR_MAX_DEVICES][2][20] = {};
    int dev = 0;
    const int rc = current_device(&dev);
    if (rc) return rc;
    std::lock_guard<std::mutex> lock(mu);
    cudaEvent_t *ev = &evs[dev][side][index];
    if (!*ev) SGR_CUDA(cudaEventCreateWithFlags(ev, cudaEventDisableTiming));
    *out = *ev;
    return SGR_OK;
}

// This backward's own signals: on `st`, or on the plan's signal stream behind an event recorded on `st` (so that the
// next kernel on `st` does not queue behind the signal's launch).
static int signal(const SgrPeerPlan *pp, cudaStream_t st, int slot, int ev_index, bool on_main = false)
{
    cudaStream_t sig = st;
    if (pp->peer_signal_stream && !on_main) {
        cudaEvent_t ev = nullptr;
        const int rc = peer_event(0, ev_index, &ev);
        if (rc) return rc;
        sig = (cudaStream_t)pp->peer_signal_stream;
        SGR_CUDA(cudaEventRecord(ev, st));
        SGR_CUDA(cudaStreamWaitEvent(sig, ev, 0));
    }
    return sgr_peer_signal(pp->peer_flag_tab, pp->peer_nranks, slot, pp->peer_rank, pp->peer_seq, sig);
}

// On the side stream: wait for every rank's REDUCED c, then split the sums of [p0, p1) into the gradient arrays.
static int split_chunk(const PeerBackward &b, int c, int p0, int p1)
{
    const SgrPeerPlan *pp = b.plan;
    cudaStream_t B = (cudaStream_t)pp->peer_side_stream;
    const int rc = sgr_peer_wait(pp->peer_flags, pp->peer_nranks, pp->peer_slot_reduced0 + c, 1, pp->peer_seq,
                                 pp->peer_timeout_s, B);
    if (rc) return rc;
    return finalize_impl(b.P, p0, p1, 0, 0, pp->peer_nranks, nullptr, nullptr, nullptr, 0, 0, nullptr, pp->peer_sums,
                         pp->peer_dsh_scale, b.dmeans3D, b.dopacity, b.dscales, b.drots, B,
                         "peer exchange: bad arguments to the record split");
}

int PeerBackward::blend_done(bool views)
{
    if (!plan) return SGR_OK;
    // BLEND goes out on `st` itself: the wait right behind it spins, and a spinning kernel must never be dispatched
    // ahead of a signal of its own rank that the peers need in order to answer
    int rc = signal(plan, st, plan->peer_slot_blend, 0, true);
    if (rc || !views) return rc;
    // the per-Gaussian pass sums every view's SH gradient into dL_dsh: the peers' factor blocks must be final
    return sgr_peer_wait(plan->peer_flags, plan->peer_nranks, plan->peer_slot_blend, 1, plan->peer_seq,
                         plan->peer_timeout_s, st);
}

int PeerBackward::chunk_done(int c, int p0, int p1)
{
    if (!plan) return SGR_OK;
    int rc = signal(plan, st, plan->peer_slot_chunk0 + c, 1 + c);
    if (rc || !plan->peer_side_stream) return rc;
    // The records' exchange of this chunk, on the side stream.  Its kernels spin on flags: they may start only once
    // THIS rank's own signal for the chunk is out (an event behind the signal kernel) -- a spinning kernel must never
    // sit in front of a signal some rank is waiting for.
    cudaStream_t B = (cudaStream_t)plan->peer_side_stream;
    cudaStream_t sig = plan->peer_signal_stream ? (cudaStream_t)plan->peer_signal_stream : st;
    cudaEvent_t e2 = nullptr;
    rc = peer_event(1, c, &e2);
    if (rc) return rc;
    SGR_CUDA(cudaEventRecord(e2, sig));
    SGR_CUDA(cudaStreamWaitEvent(B, e2, 0));
    unsigned int *counters = (unsigned int *)plan->peer_flags + (size_t)(PEER_SLOTS - 1) * PEER_RANKS;
    for (int r = 0; r < plan->peer_nranks; r++) {
        const bool me = r == plan->peer_rank;
        if (!me && !((plan->peer_emulate_ranks >> r) & 1)) continue;
        // one kernel: wait(CHUNK c, every rank) -> sum the owned slice -> its last CTA signals REDUCED c
        rc = sgr_peer_reduce_records_synced(plan->peer_rec_tab, plan->peer_sum_tab, plan->peer_nranks, r, p0, p1,
                                            plan->peer_flags, plan->peer_slot_chunk0 + c, me ? plan->peer_flag_tab : nullptr,
                                            plan->peer_slot_reduced0 + c, plan->peer_seq,
                                            me ? (void *)(counters + c) : nullptr, plan->peer_timeout_s, B);
        if (rc) return rc;
    }
    // the split of the chunk before runs behind this chunk's reduce: the other owners' slices of it have landed by
    // then, and only the last (smallest) chunk's reduce + split is exposed
    if (split_c >= 0) {
        rc = split_chunk(*this, split_c, split_p0, split_p1);
        if (rc) return rc;
    }
    split_c = c;
    split_p0 = p0;
    split_p1 = p1;
    return SGR_OK;
}

int PeerBackward::finish()
{
    if (!plan || !plan->peer_side_stream || split_c < 0) return SGR_OK;
    return split_chunk(*this, split_c, split_p0, split_p1);
}

}  // namespace sgr
