// handlers.cuh — device-side restatement of the reference's per-event handlers (used by step_kernel.cuh).
//
// One THREAD owns one group (RaftContext) for the whole batch: the group scalars (GS) and the
// Leadership.State of every follower (LS[F]) live in that thread's registers.  Everything here is
// plain sequential code per group — the reference's own execution model (one event loop turn at a
// time per context, M/support/EventLoop.java:87-101) — and parallelism comes from the number of groups.
//   K2 vote_tally        : RV-Echo / PV-Echo + Membership.isBetter (Candidate.java:112-134,
//                          Follower.java:249-270, Membership.java:74-108)
//   K3 ae_request_check  : *.appendEntries, logContains, purgeEntries, RocksLog.conflict/truncate/append
//                          (Follower.java:35-88,177-221; Candidate.java:28-41; Leader.java:66-86; RocksLog.java:169-225)
//   K4 vote_request_check: *.preVote / requestVote / installSnapshot, logUpToDate
//                          (Follower.java:91-153,193-207; Candidate.java:43-72; Leader.java:88-111; RaftMember.java:61-66)
//   K5 timer_sweep       : RaftRoutine.resetTimer / electionTimeout / keepAlive (RaftRoutine.java:53-130)
// K1 (ack_quorum_commit) and K6 (replicate_plan) touch the follower slots and live in step_kernel.cuh.
// Pure integer work: the roofline is HBM bandwidth, no tensor cores.
#pragma once
#include "tables.cuh"

namespace rafting {

constexpr int64_t I64MAX = INT64_MAX;
constexpr int     KRUNS  = RAFTING_TERM_RUNS;

struct GS {                       // group scalars, replicated in every lane of the sub-warp
    uint32_t word, inc, err, dirty;          // dirty: bit0 persist, bit1 commit
    int64_t  term, commit, lo, hi, timer, epochIndex, epochTerm, electTerm;
    uint32_t electInc; int32_t votes;
    int64_t  r0s, r0t;                       // newest term run (start, term)
};
struct LS {                       // Leadership.State of this lane's follower
    int64_t next, match, lastEpoch, reqSucc, reqFail, lastReq;
    int32_t inflight, rej, fail, pending;
};
struct RowOut {                   // ballot emitted by the current row (written once at row end)
    uint64_t bm; int64_t bt; i64x2 bl;
};
struct Ctx {
    const CfgD* cfg;
    i64x2*   runs;                // &g_runs[gid], stride G
    uint32_t gid, F, G;
    int64_t  now, draw;
};
struct Reply { int valid, success; int64_t term; };

// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ int role_of(const GS& g) { return (int)(g.word & W_ROLE_MASK); }
// The sweep's firing rule on a group's meta word and timer: a sweep row at time t fires the implied TIMEOUT of a live group whose
// timer is at or before t, where a follower's or candidate's timer of 0 or INT64_MAX never fires.  The step kernels and the due
// selection (timers.cuh) must agree on it exactly, so this is its only statement.  The timer is taken by reference so that a
// caller whose GS lives in local memory (slow_group) reads it only once the tests before it have passed.
__device__ __forceinline__ bool timer_fires(uint32_t word, const int64_t& timer, int64_t t) {
    if (!(word & W_ALIVE)) return false;
    if ((word & W_ROLE_MASK) == RAFTING_ROLE_LEADER) return timer <= t;
    return timer > 0 && timer != I64MAX && timer <= t;
}
// armed: some sweep, however late, fires it
__device__ __forceinline__ bool timer_armed(uint32_t word, int64_t timer) { return timer_fires(word, timer, I64MAX); }
__device__ __forceinline__ int ballot_of(const GS& g) { return (int)((g.word >> W_BALLOT_SH) & 0xff) - 1; }
__device__ __forceinline__ int leader_of(const GS& g) { return (int)((g.word >> W_LEADER_SH) & 0xff) - 1; }
__device__ __forceinline__ int nruns_of(const GS& g) { return (int)((g.word >> W_NRUNS_SH) & 0xf); }
__device__ __forceinline__ void set_nruns(GS& g, int n) {
    g.word = (g.word & ~(0xfu << W_NRUNS_SH)) | ((uint32_t)n << W_NRUNS_SH);
}
__device__ __forceinline__ void set_leader(GS& g, int slot) {
    g.word = (g.word & ~(0xffu << W_LEADER_SH)) | ((uint32_t)(slot + 1) << W_LEADER_SH);
}
__device__ __forceinline__ int lane_to_slot(const Ctx& c, int f) { return f < (int)c.cfg->local_slot ? f : f + 1; }
__device__ __forceinline__ int majority(const Ctx& c) { return (int)c.cfg->replicas / 2 + 1; }   // RaftContext.java:170
__device__ __forceinline__ void flag_err(GS& g, int code) {
    uint32_t cnt = (g.err >> 16) + 1; if (cnt > 0xffffu) cnt = 0xffffu;
    g.err = (cnt << 16) | (uint32_t)code;
}

// ---------------------------------------------------------------------------------------------
// run-length term table (replaces RocksLog.get(i).term(), RocksLog.java:122-128)
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ bool term_at(const GS& g, const Ctx& c, int64_t idx, int64_t& t) {
    const int n = nruns_of(g);
    if (n == 0 || idx < g.lo || idx > g.hi) return false;
    if (idx >= g.r0s) { t = g.r0t; return true; }
    bool found = false;
#pragma unroll 1
    for (int k = 1; k < n; k++) {                    // n is group-uniform; idx may differ per lane
        i64x2 r = c.runs[(size_t)k * c.G];
        if (!found && idx >= r.x) { t = r.y; found = true; }
    }
    return found;
}
__device__ __noinline__ void push_run(GS& g, const Ctx& c, int64_t start, int64_t term) {
    const int n = nruns_of(g);
    if (n >= 1) {
        for (int k = n - 1; k >= 1; k--) c.runs[(size_t)(k + 1) * c.G] = c.runs[(size_t)k * c.G];
        i64x2 r; r.x = g.r0s; r.y = g.r0t;
        c.runs[(size_t)1 * c.G] = r;
    }
    g.r0s = start; g.r0t = term;
    if (n == 0) g.lo = start;
    set_nruns(g, n + 1);
}
__device__ __noinline__ void pop_run(GS& g, const Ctx& c) {
    const int n = nruns_of(g);
    if (n <= 1) { set_nruns(g, 0); return; }
    i64x2 r = c.runs[(size_t)1 * c.G];
    for (int k = 1; k <= n - 2; k++) c.runs[(size_t)k * c.G] = c.runs[(size_t)(k + 1) * c.G];
    g.r0s = r.x; g.r0t = r.y;
    set_nruns(g, n - 1);
}
// RocksLog.truncate — RocksLog.java:219-225
__device__ __forceinline__ void log_truncate(GS& g, const Ctx& c, int64_t index) {
    if (nruns_of(g) > 0 && g.hi >= index) {
        g.hi = index - 1;
        while (nruns_of(g) > 0 && g.r0s > g.hi) pop_run(g, c);
    }
}
// RocksLog.flush — RocksLog.java:228-242 (deleteRange end-exclusive: the entry at `index` survives)
__device__ __noinline__ int log_flush(GS& g, const Ctx& c, int64_t index, int64_t term) {
    if (index < g.epochIndex) return RAFTING_ERR_FLUSH_RANGE;
    const int n = nruns_of(g);
    if (n > 0) {
        if (index > g.hi) set_nruns(g, 0);
        else if (index > g.lo) {
            if (g.r0s <= index) { g.r0s = index; set_nruns(g, 1); }
            else {
                int keep = n;
                for (int k = 1; k < n; k++) {
                    i64x2 r = c.runs[(size_t)k * c.G];
                    if (keep == n && r.x <= index) {
                        keep = k + 1;
                        r.x = index; c.runs[(size_t)k * c.G] = r;
                    }
                }
                set_nruns(g, keep);
            }
            g.lo = index;
        }
    }
    g.epochIndex = index; g.epochTerm = term;
    return 0;
}
__device__ __forceinline__ void log_append_one(GS& g, const Ctx& c, int64_t idx, int64_t term) {
    if (nruns_of(g) > 0 && term == g.r0t) g.hi = idx;
    else { push_run(g, c, idx, term); g.hi = idx; }
}
__device__ __forceinline__ void last_or_epoch(const GS& g, int64_t& idx, int64_t& term) {
    if (nruns_of(g) > 0) { idx = g.hi; term = g.r0t; } else { idx = g.epochIndex; term = g.epochTerm; }
}

// ---------------------------------------------------------------------------------------------
// Leadership.State methods — Leadership.java:40-114
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void stat_success(LS& s, int64_t now, bool reject) {           // :53-63
    if (now > s.reqSucc) s.reqSucc = now;
    s.fail = 0;
    s.rej = reject ? (int32_t)((uint32_t)s.rej + 1u) : 0;
}
__device__ __forceinline__ void stat_failure(LS& s, int64_t now, bool unreachable, bool reject) {   // :65-73
    if (now > s.reqFail) s.reqFail = now;
    if (unreachable) s.fail = (int32_t)((uint32_t)s.fail + 1u);
    if (reject) s.rej = (int32_t)((uint32_t)s.rej + 1u);
}
__device__ __forceinline__ bool state_ready(const LS& s, int32_t crit, int64_t cool, int64_t now) {   // :44-51
    bool unhealthy = (crit > 0 && (uint32_t)s.fail > (uint32_t)crit) ||
                     (cool > 0 && (int64_t)((uint64_t)now - (uint64_t)s.reqFail) < cool);
    return s.reqSucc != 0 && !(s.pending || unhealthy);
}
// round(ln(e + r)) as an integer threshold table (Leadership.java:105); verified against libm by
// tests/test_backoff_table.py for every boundary and every r < 2^16
__host__ __device__ __forceinline__ int64_t backoff_step(int32_t r) {
    if (r < 0) return 0;   // unreachable: ln of a negative argument is NaN, Math.round(NaN) == 0
    if (r <= 1) return 1;        if (r <= 9) return 2;         if (r <= 30) return 3;
    if (r <= 87) return 4;       if (r <= 241) return 5;       if (r <= 662) return 6;
    if (r <= 1805) return 7;     if (r <= 4912) return 8;      if (r <= 13357) return 9;
    if (r <= 36312) return 10;   if (r <= 98713) return 11;    if (r <= 268334) return 12;
    if (r <= 729413) return 13;  if (r <= 1982756) return 14;  if (r <= 5389695) return 15;
    if (r <= 14650716) return 16; if (r <= 39824781) return 17; if (r <= 108254985) return 18;
    if (r <= 294267563) return 19; if (r <= 799902174) return 20; if (r <= 2147483647) return 21;
    return 21;
}
__device__ __forceinline__ int update_index(LS& s, int64_t epoch, int64_t index, bool success, bool snapshot) {  // :75-114
    if (index < s.match) return RAFTING_ERR_MATCH_ROLLBACK;
    if (epoch < s.lastEpoch) return 0;
    if (epoch > s.lastEpoch) { s.lastEpoch = epoch; s.next = s.next > epoch ? s.next : epoch; }
    if ((s.pending != 0) != snapshot) return 0;
    const int64_t e1 = (int64_t)((uint64_t)epoch + 1u);
    if (s.pending) {
        if (success) { s.next = s.next > e1 ? s.next : e1; s.pending = 0; }
    } else {
        if (success) {
            if (index > s.match) { s.next = (int64_t)((uint64_t)index + 1u); s.match = index; }
        } else if (s.match == 0) {
            int64_t step = backoff_step(s.rej);
            int64_t a = (int64_t)((uint64_t)s.next - (uint64_t)step);
            int64_t nx = a > e1 ? a : e1;
            int64_t b = (int64_t)((uint64_t)s.next - 1u);
            s.next = b < nx ? b : nx;
        }
    }
    if (s.next <= epoch && !s.pending) s.pending = 1;
    return 0;
}

// ---------------------------------------------------------------------------------------------
// Membership.isBetter — Membership.java:74-108 (the filter is never null once a group is open)
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ int is_better(int nr, int64_t nt, int nb, int cr, int64_t ct, int cb) {
    if (nt != ct) return nt > ct;
    if (nr != cr) {
        if (nr == RAFTING_ROLE_LEADER) return cr == RAFTING_ROLE_CANDIDATE ? 1 : -RAFTING_ERR_LEADER_UNCHANGED;
        return nr == RAFTING_ROLE_FOLLOWER;
    }
    if (nr == RAFTING_ROLE_LEADER) return 0;
    if (nr == RAFTING_ROLE_FOLLOWER) return 1;
    if (nb != cb) return -RAFTING_ERR_BALLOT_MISMATCH;
    return 0;
}

// RaftRoutine.resetTimer — RaftRoutine.java:86-130.  g.timer: deadline (non-leader) / next keepAlive (leader)
__device__ __forceinline__ bool reset_timer(GS& g, const Ctx& c, bool muted, bool ticketNull) {
    const bool leader = role_of(g) == RAFTING_ROLE_LEADER;
    const int64_t moment = ticketNull ? 0 : (leader ? I64MAX : g.timer);
    if (!ticketNull && moment < 0) return false;
    int64_t draw = c.draw != 0 ? c.draw : rafting_draw(c.cfg->timer_seed, c.gid, g.inc, c.cfg->election_ms);
    const int64_t timeout = leader ? c.cfg->heartbeat_ms : (muted ? I64MAX : draw);
    const int64_t a = (moment == I64MAX) ? 0 : ((moment < I64MAX - 1 ? moment : I64MAX - 1) + 1);
    const int64_t b = (I64MAX - timeout < c.now) ? I64MAX : c.now + timeout;
    if (leader) {
        const int64_t delay = ticketNull ? 0 : timeout;
        g.timer = (I64MAX - delay < c.now) ? I64MAX : c.now + delay;
    } else {
        g.timer = a > b ? a : b;
    }
    return true;
}

__device__ __forceinline__ void emit_ballot(const GS& g, const Ctx& c, RowOut& ro, int kind, int64_t term) {
    int64_t li, lt; last_or_epoch(g, li, lt);
    ro.bm = (uint64_t)kind | ((uint64_t)g.inc << 32);
    ro.bt = term; ro.bl.x = li; ro.bl.y = lt;
}

// RaftRoutine.trySwitch + switchTo + convertTo — RaftRoutine.java:140-216
__device__ __forceinline__ int switch_to(GS& g, const Ctx& c, RowOut& ro, int role, int64_t term, int ballot) {
    int better = is_better(role, term, ballot, role_of(g), g.term, ballot_of(g));
    if (better < 0) return -better;
    if (!better) return 0;
    // convertTo: the old ticket is fenced and dropped; the old role's AsyncHead dies with its incarnation
    g.word = (g.word & ~(W_ROLE_MASK | W_TIMEOUT_DET | W_PREPARED | (0xffu << W_BALLOT_SH) | (0xffu << W_LEADER_SH)))
             | (uint32_t)role | ((uint32_t)(ballot + 1) << W_BALLOT_SH);
    g.term = term;
    g.inc++;
    g.dirty |= 1u;                                           // RaftMember ctor persists (term, lastCandidate)
    g.votes = 0;
    if (role == RAFTING_ROLE_CANDIDATE) {                    // Candidate ctor -> startElection (Candidate.java:22-25,90-143)
        g.votes = 1;
        emit_ballot(g, c, ro, RAFTING_BALLOT_VOTE, term);
    }
    reset_timer(g, c, false, true);
    return 0;
}

// RaftContext.commitLog + RocksLog.markCommitted — RaftContext.java:244-255, RocksLog.java:100-109
__device__ __forceinline__ int commit_log(GS& g, int64_t ci) {
    if (ci < g.commit) return RAFTING_ERR_COMMIT_ROLLBACK;
    if (ci > g.commit) { g.commit = ci; g.dirty |= 2u; }
    return 0;
}

// ---------------------------------------------------------------------------------------------
// inbound requests
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ int log_contains(const GS& g, const Ctx& c, int64_t index, int64_t term) {   // Follower.java:177-191
    if (index == 0 && term == 0) return 1;
    if (index == 0 || term == 0) return -RAFTING_ERR_INDEX_TERM_ZERO;
    if (index <= g.epochIndex) {
        if (index == g.epochIndex && term != g.epochTerm) return -RAFTING_ERR_EPOCH_TERM_MISMATCH;
        return 1;
    }
    int64_t t;
    return term_at(g, c, index, t) && t == term;
}
__device__ __forceinline__ int log_up_to_date(const GS& g, int64_t index, int64_t term) {              // Follower.java:193-207
    if (nruns_of(g) > 0) return term > g.r0t || (term == g.r0t && index >= g.hi);
    if ((index > g.epochIndex && term < g.epochTerm) || (index == g.epochIndex && term != g.epochTerm))
        return -RAFTING_ERR_IMPOSSIBLE_LOG;
    return index >= g.epochIndex;
}

// Follower.appendEntries body — Follower.java:52-87 + RocksLog.conflict/truncate/append (RocksLog.java:169-225).
// FIX: the instantiation of the kernels that honour cfg.flags (engine.cu launch_step); with FIX = false the opt-in branches
// are not compiled, and the code is the reference's.
template <bool FIX>
__device__ __noinline__ int follower_append(GS& g, const Ctx& c, RowOut& ro, int peer, int64_t term, int64_t prevIndex,
                                            int64_t prevTerm, int64_t first, uint32_t n, const int64_t* terms,
                                            int64_t leaderCommit, Reply& rep) {
    set_leader(g, peer);
    int err = 0;
    int lc = log_contains(g, c, prevIndex, prevTerm);
    if (lc < 0) err = -lc;
    else if (!lc) { rep.valid = 1; rep.success = 0; rep.term = g.term; }
    else {
        if (n > 0 && first <= g.epochIndex) {                                // purgeEntries :209-221
            int64_t skip = g.epochIndex - first + 1;
            if ((uint64_t)skip >= n) n = 0; else { first += skip; terms += skip; n -= (uint32_t)skip; }
        }
        if (n > 0) {
            int64_t conflictIndex = 0;                                       // RocksLog.conflict :199-216
            for (uint32_t i = 0; i < n; i++) {
                int64_t t;
                if (!term_at(g, c, first + i, t)) break;
                if (t != terms[i]) { conflictIndex = first + i; break; }
            }
            const bool nonEmpty = nruns_of(g) > 0;
            const int64_t hiAfter = (conflictIndex != 0 && nonEmpty && g.hi >= conflictIndex) ? conflictIndex - 1 : g.hi;
            const bool emptyAfter = !nonEmpty || hiAfter < g.lo;
            int64_t prevLogIndex = g.epochIndex;
            if (!emptyAfter && g.lo <= first) prevLogIndex = first < hiAfter ? first : hiAfter;   // seekForPrev
            else if (!emptyAfter) err = RAFTING_ERR_LOG_SHAPE;
            if (!err) {
                // capacity pre-check of the run table: reject before mutating anything
                const bool firstPutOk = emptyAfter ? (first == g.epochIndex + 1) : true;
                const bool contOk = !(first > prevLogIndex + 1);
                if (firstPutOk && contOk) {
                    uint32_t runs = 0; int64_t lastT = 0; bool have = false;
                    if (!emptyAfter) {
                        const int nr = nruns_of(g);
                        if (g.r0s <= hiAfter) { runs = (uint32_t)nr; lastT = g.r0t; have = true; }
                        else {
                            for (int k = 1; k < nr; k++) {
                                i64x2 r = c.runs[(size_t)k * c.G];
                                if (!have && r.x <= hiAfter) { runs = (uint32_t)(nr - k); lastT = r.y; have = true; }
                            }
                        }
                    }
                    for (uint32_t i = 0; i < n; i++)
                        if (first + i > prevLogIndex && (!have || terms[i] != lastT)) { runs++; lastT = terms[i]; have = true; }
                    if (runs > (uint32_t)KRUNS) err = RAFTING_ERR_TERM_RUNS_OVERFLOW;
                }
            }
            if (!err) {
                if (conflictIndex != 0) log_truncate(g, c, conflictIndex);   // Follower.java:70-72
                if (emptyAfter && first != g.epochIndex + 1) err = RAFTING_ERR_LOG_NOT_FOLLOW_EPOCH;
                else if (first > prevLogIndex + 1) err = RAFTING_ERR_LOG_NOT_CONTINUOUS;
                else
                    for (uint32_t i = 0; i < n; i++) {
                        // RocksLog.java:183-191: put everything above prevLogIndex; keys that already
                        // exist there hold the same term (no conflict was found), so only the tail grows
                        const int64_t idx = first + i;
                        if (idx > prevLogIndex && (nruns_of(g) == 0 || idx > g.hi)) log_append_one(g, c, idx, terms[i]);
                    }
            }
        }
        if (!err && leaderCommit > g.epochIndex && nruns_of(g) > 0) {       // Follower.java:76-82
            int64_t ci = leaderCommit < g.hi ? leaderCommit : g.hi;
            if constexpr (FIX)
                if ((c.cfg->flags & RAFTING_CFG_LENIENT_FOLLOWER_COMMIT) && ci < g.commit) ci = g.commit;   // ignored, not asserted
            err = commit_log(g, ci);
        }
    }
    reset_timer(g, c, false, false);                                         // finally :83-85
    if (!err && !rep.valid) { rep.valid = 1; rep.success = 1; rep.term = term; }
    return err;
}
// Follower.appendEntries — Follower.java:35-88
template <bool FIX>
__device__ __forceinline__ int follower_append_entries(GS& g, const Ctx& c, RowOut& ro, int peer, int64_t term, int64_t prevIndex,
                                                       int64_t prevTerm, int64_t first, uint32_t n, const int64_t* terms,
                                                       int64_t leaderCommit, Reply& rep) {
    if (term < g.term) { rep.valid = 1; rep.success = 0; rep.term = g.term; return 0; }
    reset_timer(g, c, true, false);
    if (term > g.term || (g.word & W_TIMEOUT_DET)) {
        int err = switch_to(g, c, ro, RAFTING_ROLE_FOLLOWER, term, ballot_of(g));
        if (err) return err;
        reset_timer(g, c, true, false);
    } else if (leader_of(g) != -1 && peer != leader_of(g)) {
        return RAFTING_ERR_FOLLOWER_TWO_LEADERS;
    }
    return follower_append<FIX>(g, c, ro, peer, term, prevIndex, prevTerm, first, n, terms, leaderCommit, rep);
}
template <bool FIX>
__device__ __forceinline__ int op_append_entries(GS& g, const Ctx& c, RowOut& ro, int peer, int64_t term, int64_t prevIndex,
                                                 int64_t prevTerm, int64_t first, uint32_t n, const int64_t* terms,
                                                 int64_t leaderCommit, Reply& rep) {
    const int role = role_of(g);
    if (role == RAFTING_ROLE_LEADER) {                                       // Leader.java:66-86
        if (peer == (int)c.cfg->local_slot) return RAFTING_ERR_LEADER_SELF_AE;
        if (term < g.term) { rep.valid = 1; rep.success = 0; rep.term = g.term; return 0; }
        if (term == g.term) return RAFTING_ERR_TWO_LEADERS;
        int err = switch_to(g, c, ro, RAFTING_ROLE_FOLLOWER, g.term, ballot_of(g));
        if (err) return err;
    } else if (role == RAFTING_ROLE_CANDIDATE) {                             // Candidate.java:28-41
        if (term < g.term) { rep.valid = 1; rep.success = 0; rep.term = g.term; return 0; }
        int err = switch_to(g, c, ro, RAFTING_ROLE_FOLLOWER, term, ballot_of(g));
        if (err) return err;
    }
    return follower_append_entries<FIX>(g, c, ro, peer, term, prevIndex, prevTerm, first, n, terms, leaderCommit, rep);
}
// Follower.requestVote — Follower.java:108-127
__device__ __forceinline__ int follower_request_vote(GS& g, const Ctx& c, RowOut& ro, int peer, int64_t term, int64_t lastIndex,
                                                     int64_t lastTerm, Reply& rep) {
    if (term < g.term) { rep.valid = 1; rep.success = 0; rep.term = g.term; return 0; }
    if (term == g.term) { rep.valid = 1; rep.success = peer == ballot_of(g); rep.term = g.term; return 0; }
    reset_timer(g, c, true, false);
    int up = log_up_to_date(g, lastIndex, lastTerm);
    if (up < 0) return -up;
    int err = switch_to(g, c, ro, RAFTING_ROLE_FOLLOWER, term, up ? peer : -1);
    if (err) return err;
    rep.valid = 1; rep.success = peer == ballot_of(g); rep.term = g.term;
    return 0;
}
template <bool FIX>
__device__ __forceinline__ int op_request_vote(GS& g, const Ctx& c, RowOut& ro, int peer, int64_t term, int64_t lastIndex,
                                               int64_t lastTerm, Reply& rep) {
    const int role = role_of(g), self = (int)c.cfg->local_slot;
    if (role == RAFTING_ROLE_LEADER) {                                       // Leader.java:93-111
        if (term < g.term) { rep.valid = 1; rep.success = 0; rep.term = g.term; return 0; }
        if (term == g.term) {
            if (ballot_of(g) == self) { rep.valid = 1; rep.success = 0; rep.term = g.term; return 0; }
            return RAFTING_ERR_LEADER_VOTE_SELF;
        }
        int err = switch_to(g, c, ro, RAFTING_ROLE_FOLLOWER, g.term, peer);
        if (err) return err;
    } else if (role == RAFTING_ROLE_CANDIDATE) {                             // Candidate.java:49-72
        if (peer == self) return RAFTING_ERR_CANDIDATE_SELF_RV;
        if (term < g.term) { rep.valid = 1; rep.success = 0; rep.term = g.term; return 0; }
        if (term == g.term) {
            if (peer != ballot_of(g)) { rep.valid = 1; rep.success = 0; rep.term = g.term; return 0; }
            else if (ballot_of(g) != self) return RAFTING_ERR_CANDIDATE_VOTE_SELF;
        }
        int err;
        if constexpr (FIX) {
            // RAFTING_CFG_STRICT_CANDIDATE_VOTE: step down at the own term first (as Leader.java:106-108 does), so that
            // Follower.requestVote applies logUpToDate to the higher-term request
            const bool strict = (c.cfg->flags & RAFTING_CFG_STRICT_CANDIDATE_VOTE) && term > g.term;
            err = strict ? switch_to(g, c, ro, RAFTING_ROLE_FOLLOWER, g.term, ballot_of(g))
                         : switch_to(g, c, ro, RAFTING_ROLE_FOLLOWER, term, peer);
        } else {
            err = switch_to(g, c, ro, RAFTING_ROLE_FOLLOWER, term, peer);
        }
        if (err) return err;
    }
    return follower_request_vote(g, c, ro, peer, term, lastIndex, lastTerm, rep);
}
template <bool FIX>
__device__ __forceinline__ int op_pre_vote(GS& g, const Ctx& c, RowOut& ro, int peer, int64_t term, int64_t lastIndex,
                                           int64_t lastTerm, Reply& rep) {
    const int role = role_of(g);
    if (role == RAFTING_ROLE_LEADER) { rep.valid = 1; rep.success = 0; rep.term = g.term; return 0; }   // Leader.java:88-91
    if (role == RAFTING_ROLE_CANDIDATE) return op_request_vote<FIX>(g, c, ro, peer, term, lastIndex, lastTerm, rep);  // Candidate.java:43-46
    if (term <= g.term || !(g.word & W_TIMEOUT_DET)) { rep.valid = 1; rep.success = 0; rep.term = g.term; return 0; }
    reset_timer(g, c, true, false);
    int up = log_up_to_date(g, lastIndex, lastTerm);
    reset_timer(g, c, false, false);
    if (up < 0) return -up;
    rep.valid = 1; rep.success = up; rep.term = g.term;
    return 0;
}
// installSnapshot — RaftMember.java:61-66, Follower.java:130-153
__device__ __forceinline__ int op_install_snapshot(GS& g, const Ctx& c, RowOut& ro, int64_t term, int hostResult, Reply& rep) {
    if (role_of(g) != RAFTING_ROLE_FOLLOWER) {
        if (term >= g.term) return RAFTING_ERR_IS_BEFORE_AE;
        rep.valid = 1; rep.success = 0; rep.term = g.term; return 0;
    }
    reset_timer(g, c, true, false);
    if (term < g.term) { rep.valid = 1; rep.success = 0; rep.term = g.term; return 0; }
    if (term > g.term) return RAFTING_ERR_IS_BEFORE_AE;
    if (g.word & W_TIMEOUT_DET) {
        int err = switch_to(g, c, ro, RAFTING_ROLE_FOLLOWER, g.term, ballot_of(g));
        if (err) return err;
        reset_timer(g, c, true, false);
    }
    rep.valid = 1; rep.success = hostResult; rep.term = g.term;
    reset_timer(g, c, false, false);
    return 0;
}


}  // namespace rafting
