// pair_kernel.cuh — the steady-state leader path for R = 3 with ONE THREAD PER (GROUP, FOLLOWER): v7 of the hot kernel.
//
// Why: the thread-per-group kernel (step_body.inc, v6) is issue/latency bound, not HBM bound — 64 K groups give only
// 16 warps per SM on an H100's 132 SMs, each walking one long dependent chain of ~820 instructions per row.  Almost all of a row's
// work is per follower — Leader.replicateLog's loop body (Leader.java:156-238) and the AE-Echo / IS-Echo callbacks
// (Leader.java:174-188,218-237 -> Leadership.State.statSuccess/statFailure/updateIndex, Leadership.java:53-114) — so it is
// split over the two follower lanes of a group: twice the warps, about half the instructions per thread.  The group
// scalars are replicated in both lanes and kept identical by construction: whatever changes them (isReady, the newEntry
// count, tryCommit + markCommitted) is computed by both lanes from values exchanged with one warp shuffle.
//
// Serial order (DESIGN.md §3) is preserved exactly:
//   * replicateLog: follower f's plan depends on the group scalars and on State f only (the one cross-follower effect —
//     an Error raised for follower f aborts the loop for the followers after it — only exists on the general path, and a
//     row that needs the general path for ANY follower is handed to the generic handler as a whole, decided before
//     anything is mutated);
//   * acks in lane order: ack f touches State f only, then calls tryCommit, which reads every matchIndex.  Lane 0's ack
//     therefore sees (match0', match1) and lane 1's (match0', match1'): both lanes evaluate both calls, in that order,
//     from the exchanged before/after values;
//   * anything else (vote replies, a higher term in a reply, a matchIndex rollback, sweep rows that fire, groups that are
//     not prepared Leaders) leaves through slow_row — the same out-of-line generic handler the v6 kernel uses — with the
//     state handed over through the tables.  The decision "generic from lane f on" depends only on pre-row state, so the
//     lanes below f are applied first, exactly as the serial loop would have.
#pragma once

namespace rafting {
namespace pair {

using namespace unrolled;

constexpr int PTPB = 2 * TPB;            // threads per block: TPB groups x 2 follower lanes

struct __align__(16) PStage {            // one staged input row of a block (TPB groups)
    i64x2    op_nr[TPB];
    i64x2    op_ab[TPB];
    i64x2    ev_tn[PTPB];
    i64x2    ev_el[PTPB];
    uint64_t op_meta[TPB];
    uint64_t ev_meta[PTPB];
};

// The group scalars the fast path only reads — only the generic handler (slow_row) changes them: one copy per group slot
// in shared memory rather than a register copy in each lane of the pair, which at the 64-register cap one wave needs
// pushed the row loop's state into local memory.  Lane 0 fills its slot from the tables after every (re)load, and a pair
// __syncwarp publishes it to lane 1.  GS's copies of these fields are not read inside the row loop.
struct PSlab {
    int64_t  term[TPB], lo[TPB], epochIndex[TPB], epochTerm[TPB], r0s[TPB], r0t[TPB];
    uint32_t inc[TPB];
};
__device__ __forceinline__ void load_slab(const Tables& T, uint32_t gid, PSlab& s, uint32_t tl) {
    s.inc[tl] = (uint32_t)(__ldcg(T.g_meta + gid) >> 32);
    s.term[tl] = __ldcg(T.g_term + gid); s.lo[tl] = __ldcg(T.g_lo + gid);
    const longlong2 ep = __ldcg((const longlong2*)(T.g_epoch + gid)); s.epochIndex[tl] = ep.x; s.epochTerm[tl] = ep.y;
    const longlong2 r0 = __ldcg((const longlong2*)(T.g_runs + gid)); s.r0s[tl] = r0.x; s.r0t[tl] = r0.y;
}
__device__ __forceinline__ void slab_to_gs(const PSlab& s, uint32_t tl, GS& g) {
    g.inc = s.inc[tl]; g.term = s.term[tl]; g.lo = s.lo[tl];
    g.epochIndex = s.epochIndex[tl]; g.epochTerm = s.epochTerm[tl]; g.r0s = s.r0s[tl]; g.r0t = s.r0t[tl];
}

// v, through an empty asm the compiler cannot move out of the row loop: the table addresses the rare hand-off to slow_row
// derives from it are computed where they are used, not hoisted and carried (in local memory) around the loop
__device__ __forceinline__ uint32_t in_place(uint32_t v) { asm volatile("" : "+r"(v)); return v; }

// term_at for an index outside the newest term run: the walk over the older runs.  Rare on the leader stream (a commit
// index below the newest run), and out of line so that the run table's address is not carried across the ack path.
// .x: found, .y: the term
__device__ __noinline__ i64x2 term_at_older(const i64x2* runs, uint32_t G, uint32_t word, int64_t lo, int64_t hi,
                                            int64_t r0s, int64_t r0t, int64_t idx) {
    GS g; g.word = word; g.lo = lo; g.hi = hi; g.r0s = r0s; g.r0t = r0t;
    Ctx c; c.runs = const_cast<i64x2*>(runs); c.G = G;
    int64_t t = 0;
    const bool found = term_at(g, c, idx, t);
    i64x2 v; v.x = found; v.y = t;
    return v;
}

// tryCommit for R = 3 on explicit matchIndex values (Leader.java:247-280, Leadership.java:116-130: sorted[F/2] of two
// values is the larger one, sorted[0] the smaller)
__device__ __forceinline__ void try_commit2(GS& g, const PSlab& s, uint32_t tl, const Tables& T, uint32_t gid, int64_t ma, int64_t mb) {
    const int64_t full = ma < mb ? ma : mb, major = ma < mb ? mb : ma;
    if (major == 0) return;
    int64_t t;
    if (nruns_of(g) > 0 && major >= s.r0s[tl] && major <= g.hi) t = s.r0t[tl];
    else {
        const i64x2 v = term_at_older(T.g_runs + gid, T.G, g.word, s.lo[tl], g.hi, s.r0s[tl], s.r0t[tl], major);
        if (!v.x) { flag_err(g, RAFTING_ERR_TRY_COMMIT_FAILED); return; }
        t = v.y;
    }
    const int64_t ci = (t == s.term[tl]) ? major : full;
    if (ci != 0 && ci != g.commit) { const int e = commit_log(g, ci); if (e) flag_err(g, e); }
}

// The inbox and the outbox rows stream through L2 once per launch (about 222 MB at config #2, against about 14 MB of
// group tables): their traffic carries evict-first hints, so that L2 keeps the tables, which every launch reads and
// writes back, rather than the stream.  Hints only: no device setting changes, and the values are the same.
__device__ __forceinline__ uint64_t l2_evict_first() {
    uint64_t p; asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p)); return p;
}
__device__ __forceinline__ void cp_async16_ef(void* smem, const void* gmem, uint64_t pol) {
    asm volatile("cp.async.cg.shared.global.L2::cache_hint [%0], [%1], 16, %2;"
                 ::"r"((uint32_t)__cvta_generic_to_shared(smem)), "l"(gmem), "l"(pol) : "memory");
}
__device__ __forceinline__ void cp_async8_ef(void* smem, const void* gmem, uint64_t pol) {
    asm volatile("cp.async.ca.shared.global.L2::cache_hint [%0], [%1], 8, %2;"
                 ::"r"((uint32_t)__cvta_generic_to_shared(smem)), "l"(gmem), "l"(pol) : "memory");
}
__device__ __forceinline__ void st_stream(uint64_t* p, uint64_t v) { __stcs((unsigned long long*)p, (unsigned long long)v); }
__device__ __forceinline__ void st_stream(int64_t* p, int64_t v) { __stcs((long long*)p, (long long)v); }
__device__ __forceinline__ void st_stream(uint32_t* p, uint32_t v) { __stcs((unsigned int*)p, v); }
__device__ __forceinline__ void st_stream(i64x2* p, int64_t x, int64_t y) { __stcs((longlong2*)p, make_longlong2(x, y)); }

template <int NST>
__global__ void __launch_bounds__(PTPB, RAFTING_PAIR_MINBLOCKS)
pair_kernel(Tables T, InboxD in, OutboxD out, const CfgD* __restrict__ cfgp, CfgD cfg) {
    static_assert(NST >= 2, "the ring needs at least two stages");
    __shared__ KArgs ka;
    __shared__ PSlab slab;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    PStage* stage = reinterpret_cast<PStage*>(smem_raw);
    // a programmatic launch behind this one (launch_pair) may start its blocks as soon as these exit
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    if (threadIdx.x == 0) { ka.T = T; ka.in = in; ka.out = out; ka.cfg = cfgp; }
    __syncthreads();
    const uint32_t tid = threadIdx.x, f = tid & 1u, tl = tid >> 1;       // follower lane, group slot in the block
    // position in the batch (launched without a class sort: in.perm is null, launch_pair checks it).  A pair past the end of
    // the batch stages, computes and indexes with position 0, so none of its copies reads past the caller's columns
    const uint32_t i0 = blockIdx.x * TPB + tl;
    bool valid = i0 < in.n;
    const uint32_t i = valid ? i0 : 0u;
    uint32_t gid = valid ? (in.gids ? in.gids[i] : i) : 0u;
    if (gid >= T.G) { valid = false; gid = 0; }
    // every thread of a warp stays in the row loop (full-mask shuffles); an invalid pair computes on group 0 and stores nothing
    const size_t li = (size_t)gid * 2u + f;
    const bool hasOps = in.op_meta != nullptr, hasEv = in.ev_meta != nullptr, hasAb = in.op_ab != nullptr, hasEl = in.ev_el != nullptr;

#define PAIR_ISSUE(R_)                                                                                          \
    {                                                                                                           \
        const uint32_t r_ = (R_);                                                                               \
        if (r_ < in.rows) {                                                                                     \
            PStage& st_ = stage[r_ % NST];                                                                      \
            const uint32_t gi_ = r_ * in.n + i;                                                                 \
            const uint64_t pol_ = l2_evict_first();                                                             \
            if (hasOps) {                                                                                       \
                if (f == 0) cp_async8_ef(&st_.op_meta[tl], in.op_meta + gi_, pol_);                             \
                else { cp_async16_ef(&st_.op_nr[tl], in.op_nr + gi_, pol_); if (hasAb) cp_async16_ef(&st_.op_ab[tl], in.op_ab + gi_, pol_); } \
            }                                                                                                   \
            if (hasEv) {                                                                                        \
                const uint32_t li_ = gi_ * 2u + f;                                                              \
                cp_async8_ef(&st_.ev_meta[tid], in.ev_meta + li_, pol_);                                        \
                cp_async16_ef(&st_.ev_tn[tid], in.ev_tn + li_, pol_);                                           \
                if (hasEl) cp_async16_ef(&st_.ev_el[tid], in.ev_el + li_, pol_);                                \
            }                                                                                                   \
        }                                                                                                       \
        cp_async_commit();                                                                                      \
    }
#pragma unroll
    for (int p = 0; p < NST - 1; p++) PAIR_ISSUE((uint32_t)p);
    // the inbox is read-only here and written by no step kernel; the tables and the outbox are the previous launch's: wait
    // for it (a no-op unless this is a programmatic launch)
    asm volatile("griddepcontrol.wait;" ::: "memory");
    if (f == 0) load_slab(T, gid, slab, tl);   // published by the row loop's first __syncwarp
    GS g; LS x;                                 // of GS only word, commit, hi, timer, err and dirty are live in the row loop
    load_hot(T, gid, g); g.dirty = 0;
    if (!valid) g.word = 0;
    load_lane(T, li, x);

    const uint32_t lane = threadIdx.x & 31u;
    for (uint32_t r = 0; r < in.rows; r++) {
        const uint32_t gi = r * in.n + i;
        cp_async_wait<NST - 2>();                              // my copies of row r have landed
        __syncwarp();                                          // ... and my peer's; both of us are done with row r-1
        PAIR_ISSUE(r + (uint32_t)(NST - 1));                   // refills the stage row r-1 used
        const PStage& st = stage[r % NST];
        const bool alive = (g.word & W_ALIVE) != 0;
        const bool leaderLive = alive && role_of(g) == RAFTING_ROLE_LEADER && (g.word & W_PREPARED);

        // ================= group op =================
        // Every ballot below sits in warp-uniform control flow (hasOps, hasEv and "sweep row" are properties of the batch,
        // not of a group); what differs per group only guards the use of the exchanged bits.
        const int64_t sweep = in.row_now ? in.row_now[r] : 0;
        uint32_t meta = 0, kind = RAFTING_OP_NONE; int64_t now = 0;
        bool slowOp = false, handled = false;
        uint32_t repMeta = 0;
        uint64_t pm = 0; int64_t p0 = 0, p1 = 0, l0 = 0, l1 = 0;       // this lane's plan
        if (sweep != 0) {
            if (timer_fires(g.word, g.timer, sweep)) { kind = RAFTING_OP_TIMEOUT; slowOp = true; }
        } else if (hasOps) {
            meta = (uint32_t)st.op_meta[tl]; now = st.op_nr[tl].x;
            const bool unav = hasAb && (((uint64_t)st.op_ab[tl].x >> f) & 1ull) != 0;
            kind = RAFTING_OP_KIND(meta);
            const bool submit = kind == RAFTING_OP_SUBMIT, hb = kind == RAFTING_OP_TIMEOUT;
            const bool fastOk = leaderLive && (hb || (submit && nruns_of(g) > 0 && slab.r0t[tl] == slab.term[tl]));
            // Leader.isReady (Leader.java:52-64) needs every follower's State: one ballot
            const bool myReady = state_ready(x, cfg.avail_critical_point, cfg.recovery_cool_down_ms, now);
            const uint32_t rb = (__ballot_sync(0xffffffffu, myReady) >> (lane & ~1u)) & 3u;
            bool ready = true;
            uint32_t count = 0;
            if (submit) {
                ready = rb != 0;                                        // ready followers >= 1 and 1 + ready > F / 2 == 1
                count = RAFTING_OP_COUNT(meta); if (count == 0) count = 1;
            }
            // replicateLog for my follower: which branch (Leader.java:156-217), decided before anything changes
            const int64_t hiNew = (submit && ready) ? g.hi + (int64_t)count : g.hi;
            // two constants, not a division by a runtime value: the division is a subroutine CALL on the row's chain
            const int limit = hb ? RAFTING_IN_FLIGHT_LIMIT / 10 : RAFTING_IN_FLIGHT_LIMIT, fetch = RAFTING_REPLICATE_LIMIT >> (hb ? 1 : 0);
            const int64_t p = (int64_t)((uint64_t)x.next - 1u);
            int cls;                                                    // 4 unavailable, 3 in-flight limit, 2 snapshot, 1 entries, 0 general
            if (unav) cls = 4;
            else if (x.inflight > limit) cls = 3;
            else if (x.pending) cls = 2;
            else cls = (nruns_of(g) > 0 && p > slab.epochIndex[tl] && p >= slab.r0s[tl] && p >= slab.lo[tl] && p <= hiNew) ? 1 : 0;
            const uint32_t gb = (__ballot_sync(0xffffffffu, cls != 0) >> (lane & ~1u)) & 3u;
            if (kind != RAFTING_OP_NONE) {
                if (!fastOk || (ready && gb != 3u)) slowOp = true;      // the generic handler takes the whole row
                else if (!ready) {                                      // NotReadyException (RaftStub.java:83-87): no newEntry, no replicateLog
                    g.word &= ~W_READY;
                    flag_err(g, RAFTING_ERR_NOT_READY); repMeta = (uint32_t)RAFTING_ERR_NOT_READY << 8;
                } else {
                    if (submit) { g.word |= W_READY; g.hi = hiNew; }
                    else g.timer = (I64MAX - cfg.heartbeat_ms < now) ? I64MAX : now + cfg.heartbeat_ms;   // resetTimer, Leader branch
                    const uint64_t hbit = hb ? (1ull << 4) : 0ull, incBits = (uint64_t)slab.inc[tl] << 32;
                    if (now > x.lastReq) x.lastReq = now;               // :158
                    if (cls == 4) { stat_failure(x, now, true, false); pm = RAFTING_PLAN_UNAVAILABLE | hbit | incBits; }
                    else if (cls == 3) pm = RAFTING_PLAN_SKIP_INFLIGHT | hbit | incBits;
                    else if (cls == 2) {
                        pm = RAFTING_PLAN_IS | hbit | incBits; p0 = slab.epochIndex[tl]; p1 = slab.epochTerm[tl]; l0 = p0; l1 = g.commit;
                        x.inflight++;
                    } else {
                        const int64_t lastIdx = (g.hi - p > (int64_t)fetch) ? p + fetch : g.hi;
                        pm = RAFTING_PLAN_AE | hbit | ((uint64_t)(lastIdx - p) << 16) | incBits; p0 = p; p1 = slab.r0t[tl]; l0 = lastIdx; l1 = g.commit;
                        x.inflight++;
                    }
                }
            }
        }
        if (slowOp) {
            // ---- the generic handler takes the whole row (op + events): state goes through the tables (pair-uniform) ----
            const uint32_t pmask = 3u << (lane & ~1u);
            const uint32_t hg = in_place(gid);
            const size_t hl = (size_t)hg * 2u + f;
            if (valid) {
                store_lane(T, hl, x);
                if (f == 0) { g.inc = slab.inc[tl]; store_hot(T, hg, g); if (out.ballot_meta) out.ballot_meta[gi] = 0; }
            }
            __syncwarp(pmask);
            uint32_t dirty = g.dirty;
            if (valid && f == 0) dirty = slow_row<2, false>(&ka, i, hg, r, kind, sweep, 1u | (hasEv ? 2u : 0u), 0u, g.dirty);
            if (f == 0) load_slab(T, hg, slab, tl);
            __syncwarp(pmask);
            dirty = __shfl_sync(pmask, dirty, lane & ~1u);
            load_hot(T, hg, g); g.dirty = dirty; if (!valid) g.word = 0;
            load_lane(T, hl, x);
            handled = true;
        } else if (valid) {
            if (out.plan_meta) {
                const size_t pl = (size_t)gi * 2u + f;
                st_stream(out.plan_meta + pl, pm);
                if (pm != 0) { st_stream(out.plan_pp + pl, p0, p1); st_stream(out.plan_lc + pl, l0, l1); st_stream(out.plan_epoch + pl, slab.epochIndex[tl]); }
            }
            if (f == 0) { if (out.rep_meta) st_stream(out.rep_meta + gi, repMeta); if (out.ballot_meta) st_stream(out.ballot_meta + gi, (uint64_t)0); }
        }

        // ================= lane events: AE-Echo / IS-Echo (Leader.java:174-188,218-237) =================
        if (hasEv) {                                            // warp-uniform
            const uint64_t em = handled ? 0ull : st.ev_meta[tid];     // the generic handler already ran this row's events
            const uint32_t ek = RAFTING_EVM_KIND(em);
            i64x2 etn = {0, 0}, eel = {0, 0};
            if (ek != RAFTING_EV_NONE) { etn = st.ev_tn[tid]; if (hasEl) eel = st.ev_el[tid]; }
            const bool ok = RAFTING_EVM_OUTCOME(em) == RAFTING_OUT_OK, snap = ek == RAFTING_EV_IS_ACK;
            const bool isAck = ek == RAFTING_EV_AE_ACK || ek == RAFTING_EV_IS_ACK;
            const bool mine = isAck && leaderLive && RAFTING_EVM_INC(em) == slab.inc[tl];   // addressed to the live Leadership.State
            // what the serial loop hands to the generic handler "from this lane on": other kinds, a higher term
            // (Leader.java:178-180,224-226), a matchIndex rollback (Leadership.java:76-81)
            const bool bail = alive && (ek > RAFTING_EV_IS_ACK || (mine && ok && (etn.x > slab.term[tl] || (snap ? eel.x : eel.y) < x.match)));
            const uint32_t bb = (__ballot_sync(0xffffffffu, bail) >> (lane & ~1u)) & 3u;
            const uint32_t bailAt = bb == 0 ? 2u : (uint32_t)(__ffs((int)bb) - 1);
            const int64_t mo = x.match;
            bool tc = false;
            if (mine && f < bailAt) {
                x.inflight--;
                if (ok) {
                    const bool success = RAFTING_EVM_SUCCESS(em) != 0;
                    if (success && !snap && eel.x == x.lastEpoch && !x.pending) {
                        // statSuccess + updateIndex for a successful AppendEntries ack at the known epoch (Leadership.java:53-63,98-102,111-113)
                        if (etn.y > x.reqSucc) x.reqSucc = etn.y;
                        x.fail = 0; x.rej = 0;
                        if (eel.y > x.match) { x.next = (int64_t)((uint64_t)eel.y + 1u); x.match = eel.y; }
                        if (x.next <= eel.x) x.pending = 1;
                    } else {
                        stat_success(x, etn.y, !success);
                        update_index(x, eel.x, snap ? eel.x : eel.y, success, snap);
                    }
                    tc = !snap && success;
                } else stat_failure(x, etn.y, RAFTING_EVM_OUTCOME(em) == RAFTING_OUT_ERROR, false);
            }
            // tryCommit after ack 0 sees (match0', match1); after ack 1 (match0', match1'): both lanes evaluate both, in order
            const uint32_t tb = (__ballot_sync(0xffffffffu, tc) >> (lane & ~1u)) & 3u;
            const int64_t mn = x.match;
            const int64_t peerOld = __shfl_xor_sync(0xffffffffu, mo, 1), peerNew = __shfl_xor_sync(0xffffffffu, mn, 1);
            if (tb) {
                const int64_t m0n = f == 0 ? mn : peerNew, m1o = f == 0 ? peerOld : mo, m1n = f == 0 ? peerNew : mn;
                if (tb & 1u) try_commit2(g, slab, tl, T, gid, m0n, m1o);
                if (tb & 2u) try_commit2(g, slab, tl, T, gid, m0n, m1n);
            }
            if (bailAt < 2u) {
                // pair-uniform: the generic handler finishes this row from lane bailAt on
                const uint32_t pmask = 3u << (lane & ~1u);
                const uint32_t hg = in_place(gid);
                const size_t hl = (size_t)hg * 2u + f;
                if (valid) { store_lane(T, hl, x); if (f == 0) { g.inc = slab.inc[tl]; store_hot(T, hg, g); } }
                __syncwarp(pmask);
                uint32_t dirty = g.dirty;
                if (valid && f == 0) dirty = slow_row<2, false>(&ka, i, hg, r, 0u, 0, 2u, bailAt, g.dirty);
                if (f == 0) load_slab(T, hg, slab, tl);
                __syncwarp(pmask);
                dirty = __shfl_sync(pmask, dirty, lane & ~1u);
                load_hot(T, hg, g); g.dirty = dirty; if (!valid) g.word = 0;
                load_lane(T, hl, x);
            }
        }
    }
    cp_async_wait<0>();
    if (!valid) return;
    // ---- write back: lane f its Leadership.State, lane 0 the group columns the fast path can change ----
    store_lane(T, li, x);
    if (f == 0) { slab_to_gs(slab, tl, g); store_hot(T, gid, g); write_group_columns(in, out, i, gid, g); }
#undef PAIR_ISSUE
}

}  // namespace pair
}  // namespace rafting
