// step_kernel.cuh — the batched "event loop" kernel: one launch drains one batch for every group.
//
// Replaces, for all groups at once, the reference's per-context EventLoop path
// (M/support/EventLoop.java:87-101 + the RaftParticipant handlers and Async callbacks it runs).
//
//   K1 ack_quorum_commit : AE-Echo / IS-Echo + Leadership.State.{statSuccess,statFailure,updateIndex,
//                          majorIndices} + Leader.tryCommit + RocksLog.markCommitted
//                          (Leader.java:174-188,218-237,247-280; Leadership.java:53-130; RocksLog.java:100-109)
//   K6 replicate_plan    : Leader.prepareReplication / replicateLog / isReady (Leader.java:30-64,142-245)
//   K2..K5               : handlers.cuh
//
// Mapping (v4, after profiling two sub-warp-per-group versions, which were
// bound by divergence replays, redundant per-lane group work and register spills): ONE THREAD PER
// GROUP.  The thread keeps the group scalars and the Leadership.State of all F followers in registers
// for the whole batch and walks the rows in order, which is exactly the reference's serial order, so
// there is nothing to reconcile across lanes.  Consecutive threads own consecutive groups, so every
// column access is a coalesced 8/16-byte-per-thread load or store.
//   * inputs are staged by cp.async into a per-block shared-memory ring NST rows deep (each thread
//     copies only its own op and its F events, so no barrier is needed, only cp.async.wait_group):
//     NST-1 rows (~120 B per thread at R=3) are always in flight per thread without holding registers;
//   * FAST PATH, inline: SUBMIT / keepAlive on a prepared Leader and rows whose events are acks;
//   * SLOW PATH, out of line: everything else (elections, step-downs, inbound requests, flushes,
//     sweeps, term-run pushes, match-index rollbacks).  State is handed over through the tables so
//     the hot state never has its address taken.
#pragma once
#include "handlers.cuh"

namespace rafting {

struct KArgs { Tables T; InboxD in; OutboxD out; const CfgD* cfg; };   // block-shared copy of the kernel arguments

__device__ __forceinline__ Ctx make_ctx(const Tables& T, const CfgD* cfg, uint32_t gid, int64_t now, int64_t draw) {
    Ctx c; c.cfg = cfg; c.runs = T.g_runs + gid; c.gid = gid; c.F = T.F; c.G = T.G; c.now = now; c.draw = draw;
    return c;
}

// ---- state movement between HBM tables and registers (L2-coherent loads: the slow path hands state
//      over through the tables inside one launch) ----
__device__ __forceinline__ void load_hot(const Tables& T, uint32_t gid, GS& g) {
    const uint64_t m = __ldcg(T.g_meta + gid);
    g.word = (uint32_t)m; g.inc = (uint32_t)(m >> 32);
    g.term = __ldcg(T.g_term + gid); g.commit = __ldcg(T.g_commit + gid);
    g.lo = __ldcg(T.g_lo + gid); g.hi = __ldcg(T.g_hi + gid); g.timer = __ldcg(T.g_timer + gid);
    const longlong2 ep = __ldcg((const longlong2*)(T.g_epoch + gid)); g.epochIndex = ep.x; g.epochTerm = ep.y;
    const longlong2 r0 = __ldcg((const longlong2*)(T.g_runs + gid)); g.r0s = r0.x; g.r0t = r0.y;
    g.err = __ldcg(T.g_err + gid);
}
__device__ __forceinline__ void load_cold(const Tables& T, uint32_t gid, GS& g) {
    const longlong2 el = __ldcg((const longlong2*)(T.g_elect + gid));
    g.electTerm = el.x; g.electInc = (uint32_t)(uint64_t)el.y; g.votes = (int32_t)((uint64_t)el.y >> 32);
}
__device__ __forceinline__ void store_hot(const Tables& T, uint32_t gid, const GS& g) {
    T.g_meta[gid] = (uint64_t)g.word | ((uint64_t)g.inc << 32);
    T.g_commit[gid] = g.commit; T.g_hi[gid] = g.hi; T.g_timer[gid] = g.timer; T.g_err[gid] = g.err;
}
__device__ __forceinline__ void store_warm(const Tables& T, uint32_t gid, const GS& g) {
    T.g_term[gid] = g.term; T.g_lo[gid] = g.lo;
    i64x2 v; v.x = g.epochIndex; v.y = g.epochTerm; T.g_epoch[gid] = v;
    v.x = g.r0s; v.y = g.r0t; T.g_runs[gid] = v;
}
__device__ __forceinline__ void store_cold(const Tables& T, uint32_t gid, const GS& g) {
    i64x2 v; v.x = g.electTerm; v.y = (int64_t)((uint64_t)g.electInc | ((uint64_t)(uint32_t)g.votes << 32));
    T.g_elect[gid] = v;
}
__device__ __forceinline__ void load_lane(const Tables& T, size_t li, LS& s) {
    const longlong2 nm = __ldcg((const longlong2*)(T.l_nm + li)), es = __ldcg((const longlong2*)(T.l_es + li)),
                    fr = __ldcg((const longlong2*)(T.l_fr + li));
    const int4 cn = __ldcg(T.l_cnt + li);
    s.next = nm.x; s.match = nm.y; s.lastEpoch = es.x; s.reqSucc = es.y; s.reqFail = fr.x; s.lastReq = fr.y;
    s.inflight = cn.x; s.rej = cn.y; s.fail = cn.z; s.pending = cn.w;
}
__device__ __forceinline__ void store_lane(const Tables& T, size_t li, const LS& s) {
    i64x2 v; int4 cn;
    v.x = s.next; v.y = s.match; T.l_nm[li] = v;
    v.x = s.lastEpoch; v.y = s.reqSucc; T.l_es[li] = v;
    v.x = s.reqFail; v.y = s.lastReq; T.l_fr[li] = v;
    cn.x = s.inflight; cn.y = s.rej; cn.z = s.fail; cn.w = s.pending; T.l_cnt[li] = cn;
}

// ---------------------------------------------------------------------------------------------
// the kernel
// ---------------------------------------------------------------------------------------------
#ifndef RAFTING_MINBLOCKS
#define RAFTING_MINBLOCKS 8
#endif
#ifndef RAFTING_MINBLOCKS4
#define RAFTING_MINBLOCKS4 1        // FT = 4 (R <= 5)
#endif
#ifndef RAFTING_TPB
#define RAFTING_TPB 64
#endif
constexpr int TPB = RAFTING_TPB;         // threads (= groups) per block: 64K groups / 64 = 1024 blocks = 7.8 per SM on 132 SMs (one wave)

__device__ __forceinline__ void cp_async16(void* smem, const void* gmem) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"((uint32_t)__cvta_generic_to_shared(smem)), "l"(gmem) : "memory");
}
__device__ __forceinline__ void cp_async8(void* smem, const void* gmem) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"((uint32_t)__cvta_generic_to_shared(smem)), "l"(gmem) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

template <int FT>
struct __align__(16) Stage {             // one staged input row of this block
    i64x2    op_nr[TPB];
    i64x2    op_ab[TPB];
    i64x2    ev_tn[TPB * FT];
    i64x2    ev_el[TPB * FT];
    uint64_t op_meta[TPB];
    uint64_t ev_meta[TPB * FT];
};


// Pre-pass of a step that may carry inbound requests: sorts the positions of the batch into NCLS classes so that a
// warp of the step kernel runs ONE kind of work instead of waiting for its slowest lane:
//   0 follower, 1 candidate, 2 leader that will need the generic handlers (not prepared / closed, or an op other than
//   SUBMIT / TIMEOUT in some row)   -> slow_group, the whole step with the generic handlers
//   3 leader steady state            -> the register-resident fast path
// perm holds NCLS regions of n positions; cnt the class sizes.  One thread per position; block-level compaction, one
// atomicAdd per block and class (the order of the blocks' chunks inside a class is irrelevant: groups are independent,
// and a chunk stays contiguous for coalescing).
constexpr int NCLS = 4;
constexpr uint32_t INBOX_INTERNAL_SLOW_ELSEWHERE = 1u << 30;   // InboxD.flags: the slow classes run in slow_kernel
__global__ void __launch_bounds__(256) classify_kernel(Tables T, InboxD in, uint32_t* __restrict__ perm, uint32_t* __restrict__ cnt) {
    __shared__ uint32_t wcnt[NCLS][8], base[NCLS];
    const uint32_t i = blockIdx.x * 256u + threadIdx.x;
    const bool valid = i < in.n;
    int cls = -1;
    if (valid) {
        const uint32_t gid = in.gids ? in.gids[i] : i;
        if (gid >= T.G) cls = 2;
        else {
            const uint32_t w = (uint32_t)T.g_meta[gid];
            const uint32_t role = w & W_ROLE_MASK;
            if (role == RAFTING_ROLE_FOLLOWER) cls = 0;
            else if (role == RAFTING_ROLE_CANDIDATE) cls = 1;
            else {
                bool slow = !((w & W_ALIVE) && (w & W_PREPARED));
                if (!slow && in.op_meta)
                    for (uint32_t r = 0; r < in.rows; r++)
                        if (!(in.row_now && in.row_now[r] != 0) && RAFTING_OP_KIND((uint32_t)in.op_meta[(size_t)r * in.n + i]) > RAFTING_OP_TIMEOUT) { slow = true; break; }
                cls = slow ? 2 : 3;
            }
        }
    }
    const uint32_t lane = threadIdx.x & 31u, wq = threadIdx.x >> 5;
    uint32_t mine = 0;
#pragma unroll
    for (int k = 0; k < NCLS; k++) {
        const uint32_t m = __ballot_sync(0xffffffffu, cls == k);
        if (lane == 0) wcnt[k][wq] = __popc(m);
        if (cls == k) mine = m;
    }
    __syncthreads();
    if (threadIdx.x < NCLS) {
        uint32_t tot = 0;
        for (int k = 0; k < 8; k++) { const uint32_t c = wcnt[threadIdx.x][k]; wcnt[threadIdx.x][k] = tot; tot += c; }
        base[threadIdx.x] = tot ? atomicAdd(cnt + threadIdx.x, tot) : 0u;
    }
    __syncthreads();
    if (valid) perm[(size_t)cls * in.n + base[cls] + wcnt[cls][wq] + __popc(mine & ((1u << lane) - 1u))] = i;
}

#define RAFTING_BODY_NS unrolled
#define RAFTING_UNROLL _Pragma("unroll")
#include "step_body.inc"
#undef RAFTING_BODY_NS
#undef RAFTING_UNROLL
#define RAFTING_BODY_NS looped
#define RAFTING_UNROLL _Pragma("unroll 1")
#include "step_body.inc"
#undef RAFTING_BODY_NS
#undef RAFTING_UNROLL

}  // namespace rafting

#ifndef RAFTING_PAIR_MINBLOCKS
#define RAFTING_PAIR_MINBLOCKS 8     // 8 x 128 threads per SM (<= 64 registers): 64 K groups x 2 lanes fit in one wave on
                                     // 132 SMs; on an H100 faster than 7 blocks (72 registers, 118 K lanes per wave) despite more spills
#endif
#include "pair_kernel.cuh"
