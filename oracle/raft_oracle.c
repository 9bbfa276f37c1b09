/*
 * raft_oracle.c — CPU restatement of curioloop/rafting's per-context EventLoop path.
 * TEST INFRASTRUCTURE ONLY (see raft_oracle.h).  PARITY UNPINNED BY UPSTREAM TESTS.
 *
 * One `ogroup_t` == one RaftContext with its live RaftParticipant object, its TimerTicket, its
 * in-memory RaftLog (RocksLog semantics, index -> term only) and, for a Leader, one
 * Leadership.State per remote node.  Each function names the reference lines it restates;
 * M/ = the reference's src/main/java/io/lubricant/consensus/raft/.
 *
 * "throw" is modelled by returning a positive RAFTING_ERR_* code up the call chain; effects
 * performed before the throw point stay, exactly as in the JVM (the event loop catches Throwable
 * and logs it: M/support/EventLoopGroup.java:40-44).
 *
 * Canonical serial order (the parity spec, DESIGN.md §3): per group, events run in stream order;
 * ContextEventLoop.execute(.., urgent=true) hand-offs from callback threads (trySwitchTo,
 * RaftContext.java:205-215; tryCommit, Leader.java:263-274) take effect immediately after the
 * callback that issued them.
 */
#include "raft_oracle.h"

#include <math.h>
#include <pthread.h>
#include <sched.h>
#include <stdlib.h>
#include <string.h>

#define I64_MAX INT64_MAX
#define MAXF (RAFTING_MAX_REPLICAS - 1)

/* ------------------------------------------------------------------------------------------ */
/* Leadership.State — M/context/member/Leadership.java:26-38                                   */
/* ------------------------------------------------------------------------------------------ */
typedef struct {
    int64_t lastRequest, requestSuccess, requestFailure;
    int32_t requestInFlight, recentRejection, recentFailure;
    int64_t lastEpoch, nextIndex, matchIndex;
    int     pendingInstallation;
} ostate_t;

/* in-memory RaftLog with RocksLog semantics — M/command/storage/RocksLog.java:82-242.
   Stored keys are the contiguous range [lo, hi] (empty iff hi < lo); terms[i - base] = term(i). */
typedef struct {
    int64_t epochIndex, epochTerm;   /* RocksLog.epochEntry */
    int64_t commitIndex;             /* RocksLog.commitIndex (volatile, never persisted) */
    int64_t lo, hi, base;
    int64_t* terms;
    size_t   cap;
} olog_t;

typedef struct {
    int      alive;                  /* RaftContext.stillRunning */
    int      role;                   /* class of the live RaftParticipant */
    int64_t  term;                   /* RaftMember.currentTerm */
    int      ballot;                 /* RaftMember.lastCandidate as node slot, -1 == null */
    uint32_t incarnation;            /* counts RaftMember constructions (RaftMember.java:20-26) */
    int      memberNull;             /* membershipFilter.get() == null (before initialize) */
    /* Follower — Follower.java:21-24 */
    int      currentLeader;
    int      timeoutDetected;
    /* election round of the live object: Follower.prepareElection / Candidate.startElection */
    int      votes;
    /* Candidate.elected + its AsyncHead surviving onFencing (Candidate.java:75-80) */
    uint32_t electedInc;
    int      electedAborted;
    int64_t  electedTerm;
    /* Leader — Leader.java:23-24 */
    int      prepared;               /* followerStatus != null */
    ostate_t st[MAXF];
    /* TimerTicket — TimerTicket.java, RaftRoutine.java:86-130 */
    int      ticketNull;
    int64_t  deadline;
    int64_t  hbDue;                  /* heartbeatKeeper schedule time of the Leader's ticket */
    olog_t   log;
    uint32_t errWord;
    int      persistDirty, commitDirty, readyBit;
} ogroup_t;

struct orc_pool;
struct orc_engine {
    rafting_cfg_t cfg;
    uint32_t F;
    ogroup_t* groups;
    uint64_t events;
    struct orc_pool* pool;   /* the loop threads (ContextLoop-k, ContextManager.java:46), created on first use */
};

/* per-event context: where outputs of the running event go */
typedef struct {
    orc_engine_t* e;
    ogroup_t* g;
    uint32_t gid;
    int64_t now;
    int64_t draw;          /* 0 => counter-based draw */
    /* outbox slots of the current (row, group) */
    uint64_t* plan_meta; rafting_i64x2_t* plan_pp; rafting_i64x2_t* plan_lc; int64_t* plan_epoch; /* [F] */
    uint64_t* ballot_meta; int64_t* ballot_term; rafting_i64x2_t* ballot_last;
} octx_t;

/* ------------------------------------------------------------------------------------------ */
/* helpers                                                                                    */
/* ------------------------------------------------------------------------------------------ */
static inline int lane_to_slot(const orc_engine_t* e, uint32_t f) {
    return (int)(f < e->cfg.local_slot ? f : f + 1);
}
static inline int majority(const orc_engine_t* e) { return (int)e->cfg.replicas / 2 + 1; } /* RaftContext.java:170 */

static void flag_err(ogroup_t* g, int code) {
    uint32_t cnt = (g->errWord >> 16) + 1; if (cnt > 0xffff) cnt = 0xffff;
    g->errWord = (cnt << 16) | (uint32_t)code;
}

int64_t orc_draw(uint64_t seed, uint32_t gid, uint32_t incarnation, int64_t election_ms) {
    return rafting_draw(seed, gid, incarnation, election_ms);
}

/* ------------------------------------------------------------------------------------------ */
/* RaftLog model                                                                              */
/* ------------------------------------------------------------------------------------------ */
static int log_empty(const olog_t* l) { return l->hi < l->lo; }
static int log_get(const olog_t* l, int64_t index, int64_t* term) {          /* RocksLog.java:122-128 */
    if (log_empty(l) || index < l->lo || index > l->hi) return 0;
    *term = l->terms[index - l->base];
    return 1;
}
static int log_last(const olog_t* l, int64_t* index, int64_t* term) {       /* RocksLog.java:117-119,244-253 */
    if (log_empty(l)) return 0;
    *index = l->hi; *term = l->terms[l->hi - l->base];
    return 1;
}
static uint32_t log_runs(const olog_t* l) {
    if (log_empty(l)) return 0;
    uint32_t n = 1;
    for (int64_t i = l->lo + 1; i <= l->hi; i++)
        if (l->terms[i - l->base] != l->terms[i - 1 - l->base]) n++;
    return n;
}
static void log_reserve(olog_t* l, int64_t upto) {
    if (log_empty(l)) { /* re-base an empty store lazily */ }
    size_t need = (size_t)(upto - l->base + 1);
    if (need <= l->cap) return;
    /* compact first: drop the dead prefix below lo */
    if (!log_empty(l) && l->lo > l->base) {
        size_t live = (size_t)(l->hi - l->lo + 1);
        memmove(l->terms, l->terms + (l->lo - l->base), live * sizeof(int64_t));
        l->base = l->lo;
        need = (size_t)(upto - l->base + 1);
        if (need <= l->cap) return;
    }
    size_t cap = l->cap ? l->cap : 16;
    while (cap < need) cap *= 2;
    l->terms = (int64_t*)realloc(l->terms, cap * sizeof(int64_t));
    l->cap = cap;
}
static void log_put(olog_t* l, int64_t index, int64_t term) {
    if (log_empty(l)) { l->base = index; l->lo = index; l->hi = index - 1; }
    log_reserve(l, index);
    l->terms[index - l->base] = term;
    if (index > l->hi) l->hi = index;
}
/* RocksLog.truncate — RocksLog.java:219-225 */
static void log_truncate(olog_t* l, int64_t index) {
    if (!log_empty(l) && l->hi >= index) l->hi = index - 1;   /* deleteRange(index, last+1) */
    if (l->hi < l->lo) { l->hi = l->lo - 1; }
}
/* RocksLog.flush — RocksLog.java:228-242.  deleteRange(epochIndex, index) is END-EXCLUSIVE: the
   entry at `index` itself survives and stays visible to get()/last(). */
static int log_flush(olog_t* l, int64_t index, int64_t term) {
    if (index < l->epochIndex) return RAFTING_ERR_FLUSH_RANGE;
    if (!log_empty(l)) {
        if (index > l->hi) { l->lo = l->hi + 1; }
        else if (index > l->lo) l->lo = index;
    }
    l->epochIndex = index; l->epochTerm = term;
    return 0;
}

/* ------------------------------------------------------------------------------------------ */
/* Leadership.State methods                                                                    */
/* ------------------------------------------------------------------------------------------ */
/* increaseMono — Leadership.java:40-42 */
static void increase_mono(int64_t* field, int64_t next) { if (next > *field) *field = next; }

/* statSuccess — Leadership.java:53-63 */
static void stat_success(ostate_t* s, int64_t now, int reject) {
    increase_mono(&s->requestSuccess, now);
    if (s->recentFailure != 0) s->recentFailure = 0;
    if (reject) s->recentRejection = (int32_t)((uint32_t)s->recentRejection + 1u);
    else if (s->recentRejection != 0) s->recentRejection = 0;
}
/* statFailure — Leadership.java:65-73 */
static void stat_failure(ostate_t* s, int64_t now, int unreachable, int reject) {
    increase_mono(&s->requestFailure, now);
    if (unreachable) s->recentFailure = (int32_t)((uint32_t)s->recentFailure + 1u);
    if (reject) s->recentRejection = (int32_t)((uint32_t)s->recentRejection + 1u);
}
/* isUnhealthy / isReady — Leadership.java:44-51 */
static int state_unhealthy(const ostate_t* s, int32_t crit, int64_t cool, int64_t now) {
    return (crit > 0 && (uint32_t)s->recentFailure > (uint32_t)crit) ||
           (cool > 0 && (int64_t)((uint64_t)now - (uint64_t)s->requestFailure) < cool);
}
static int state_ready(const ostate_t* s, int32_t crit, int64_t cool, int64_t now) {
    return s->requestSuccess != 0 && !(s->pendingInstallation || state_unhealthy(s, crit, cool, now));
}
/* round(ln(e + r)) — Leadership.java:105, double arithmetic exactly as the JVM does it */
int64_t orc_backoff_step(int32_t r) {
    double v = log(M_E + (double)r);
    return (int64_t)floor(v + 0.5);      /* Math.round(double) == floor(x + 0.5) */
}
/* updateIndex — Leadership.java:75-114 */
static int update_index(ostate_t* s, int64_t epoch, int64_t index, int success, int snapshot) {
    if (index < s->matchIndex) return RAFTING_ERR_MATCH_ROLLBACK;          /* :76-81 */
    if (epoch < s->lastEpoch) return 0;                                     /* :83 */
    if (epoch > s->lastEpoch) {                                             /* :84-88 */
        s->lastEpoch = epoch;
        s->nextIndex = s->nextIndex > epoch ? s->nextIndex : epoch;
    }
    if (s->pendingInstallation != snapshot) return 0;                       /* :90 */
    if (s->pendingInstallation) {                                           /* :92-96 */
        if (success) {
            int64_t e1 = (int64_t)((uint64_t)epoch + 1u);
            s->nextIndex = s->nextIndex > e1 ? s->nextIndex : e1;
            s->pendingInstallation = 0;
        }
    } else {
        if (success) {                                                      /* :98-102 */
            if (index > s->matchIndex) {
                s->nextIndex = (int64_t)((uint64_t)index + 1u);
                s->matchIndex = index;
            }
        } else if (s->matchIndex == 0) {                                    /* :103-108 */
            int64_t step = orc_backoff_step(s->recentRejection);
            int64_t e1 = (int64_t)((uint64_t)epoch + 1u);
            int64_t a = (int64_t)((uint64_t)s->nextIndex - (uint64_t)step);
            int64_t next = a > e1 ? a : e1;
            int64_t b = (int64_t)((uint64_t)s->nextIndex - 1u);
            s->nextIndex = b < next ? b : next;
        }
    }
    if (s->nextIndex <= epoch && !s->pendingInstallation) s->pendingInstallation = 1;  /* :111-113 */
    return 0;
}
/* Test hook for the upstream golden vectors (oracle/java/GoldenGen.java): one Leadership.State method applied to a flat
   state vector [lastRequest, requestSuccess, requestFailure, requestInFlight, recentRejection, recentFailure, lastEpoch,
   nextIndex, matchIndex, pendingInstallation].  op: 0 statSuccess(now, reject)  1 statFailure(now, unreachable, reject)
   2 isReady(criticalPoint, coolDown, now) -> ret = {isReady, isUnhealthy}  3 updateIndex(epoch, index, success, snapshot).
   Returns the per-event error code (RAFTING_ERR_MATCH_ROLLBACK for the AbstractMethodError). */
int orc_state_apply(int64_t st[10], int op, const int64_t* a, int64_t ret[2]) {
    ostate_t s; memset(&s, 0, sizeof(s));
    s.lastRequest = st[0]; s.requestSuccess = st[1]; s.requestFailure = st[2]; s.requestInFlight = (int32_t)st[3];
    s.recentRejection = (int32_t)st[4]; s.recentFailure = (int32_t)st[5]; s.lastEpoch = st[6]; s.nextIndex = st[7];
    s.matchIndex = st[8]; s.pendingInstallation = (int)st[9];
    int err = 0;
    if (op == 0) stat_success(&s, a[0], (int)a[1]);
    else if (op == 1) stat_failure(&s, a[0], (int)a[1], (int)a[2]);
    else if (op == 2) { ret[0] = state_ready(&s, (int32_t)a[0], a[1], a[2]); ret[1] = state_unhealthy(&s, (int32_t)a[0], a[1], a[2]); }
    else if (op == 3) err = update_index(&s, a[0], a[1], (int)a[2], (int)a[3]);
    else return -1;
    st[0] = s.lastRequest; st[1] = s.requestSuccess; st[2] = s.requestFailure; st[3] = s.requestInFlight;
    st[4] = s.recentRejection; st[5] = s.recentFailure; st[6] = s.lastEpoch; st[7] = s.nextIndex; st[8] = s.matchIndex;
    st[9] = s.pendingInstallation;
    return err;
}
/* majorIndices — Leadership.java:116-130 */
static int cmp_i64(const void* a, const void* b) {
    int64_t x = *(const int64_t*)a, y = *(const int64_t*)b;
    return x < y ? -1 : x > y;
}
void orc_major_indices(const int64_t* match, int n, int64_t out[2]) {
    int64_t tmp[MAXF];
    memcpy(tmp, match, (size_t)n * sizeof(int64_t));
    qsort(tmp, (size_t)n, sizeof(int64_t), cmp_i64);      /* Arrays.sort */
    out[0] = tmp[0];
    out[1] = tmp[n / 2];
}

/* ------------------------------------------------------------------------------------------ */
/* Membership.isBetter — Membership.java:74-108.  returns 1/0, or -code on AssertionError      */
/* ------------------------------------------------------------------------------------------ */
int orc_is_better(int nr, int64_t nt, int nb, int cr, int64_t ct, int cb, int cur_null) {
    if (cur_null) return 1;                                   /* :75-77 */
    if (nt != ct) return nt > ct;                             /* :80-82 */
    if (nr != cr) {                                           /* :84-93 */
        if (nr == RAFTING_ROLE_LEADER) {
            if (cr == RAFTING_ROLE_CANDIDATE) return 1;
            return -RAFTING_ERR_LEADER_UNCHANGED;
        }
        return nr == RAFTING_ROLE_FOLLOWER;
    } else {                                                  /* :94-101 */
        if (nr == RAFTING_ROLE_LEADER) return 0;
        if (nr == RAFTING_ROLE_FOLLOWER) return 1;
    }
    if (nb != cb) return -RAFTING_ERR_BALLOT_MISMATCH;        /* :103-105 */
    return 0;
}

/* ------------------------------------------------------------------------------------------ */
/* RaftRoutine.resetTimer — RaftRoutine.java:86-130 (participant == the live one)              */
/* ------------------------------------------------------------------------------------------ */
static int64_t ctx_draw(octx_t* c) {
    if (c->draw != 0) return c->draw;
    return rafting_draw(c->e->cfg.timer_seed, c->gid, c->g->incarnation, c->e->cfg.election_ms);
}
static int reset_timer(octx_t* c, int muted) {
    ogroup_t* g = c->g;
    int64_t moment = g->ticketNull ? 0 : g->deadline;                       /* :95-96 */
    if (!g->ticketNull && moment < 0) return 0;                             /* :97-98 */
    int64_t now = c->now;
    int leader = g->role == RAFTING_ROLE_LEADER;
    int64_t timeout = leader ? c->e->cfg.heartbeat_ms : (muted ? I64_MAX : ctx_draw(c));   /* :101-103 */
    int64_t a = (moment == I64_MAX) ? 0 : ((moment < I64_MAX - 1 ? moment : I64_MAX - 1) + 1);  /* :105-106 */
    int64_t b = (I64_MAX - timeout < now) ? I64_MAX : now + timeout;        /* :107 */
    int64_t deadline = a > b ? a : b;
    /* reset == true: serial order never sees an already-fired schedule (:109-111) */
    if (leader) {                                                           /* :116-118 */
        g->deadline = I64_MAX;
        int64_t delay = g->ticketNull ? 0 : timeout;
        g->hbDue = (I64_MAX - delay < now) ? I64_MAX : now + delay;
    } else {                                                                /* :119-122 */
        g->deadline = deadline;
    }
    g->ticketNull = 0;
    return 1;
}

/* ------------------------------------------------------------------------------------------ */
/* election broadcasts                                                                        */
/* ------------------------------------------------------------------------------------------ */
static void last_or_epoch(const olog_t* l, int64_t* idx, int64_t* term) {   /* Follower.java:230-235, Candidate.java:94-99 */
    if (!log_last(l, idx, term)) { *idx = l->epochIndex; *term = l->epochTerm; }
}
static void emit_ballot(octx_t* c, int kind, int64_t term) {
    int64_t li, lt; last_or_epoch(&c->g->log, &li, &lt);
    if (c->ballot_meta) {
        *c->ballot_meta = (uint64_t)kind | ((uint64_t)c->g->incarnation << 32);
        *c->ballot_term = term;
        c->ballot_last->x = li; c->ballot_last->y = lt;
    }
}
/* Follower.prepareElection — Follower.java:223-279 */
static void prepare_election(octx_t* c) {
    ogroup_t* g = c->g;
    g->timeoutDetected = 1;                                                  /* :225 */
    g->votes = 1;                                                            /* :249 */
    emit_ballot(c, RAFTING_BALLOT_PREVOTE, (int64_t)((uint64_t)g->term + 1u)); /* :246,257 */
}
/* Candidate.startElection — Candidate.java:90-143 */
static void start_election(octx_t* c) {
    ogroup_t* g = c->g;
    g->votes = 1;                                                            /* :112 */
    emit_ballot(c, RAFTING_BALLOT_VOTE, g->term);                            /* :120 */
}

/* ------------------------------------------------------------------------------------------ */
/* RaftRoutine.trySwitch / switchTo / convertTo — RaftRoutine.java:140-216                      */
/* returns 0 (done or not-better no-op) or a positive error code                               */
/* ------------------------------------------------------------------------------------------ */
static int switch_to(octx_t* c, int role, int64_t term, int ballot) {
    ogroup_t* g = c->g;
    int better = orc_is_better(role, term, ballot, g->role, g->term, g->ballot, g->memberNull);  /* :142-151 */
    if (better < 0) return -better;
    if (!better) return 0;                      /* switchTo(ctx, null): latest membership already applied (:166-168) */
    /* convertTo — :183-216 */
    if (!g->ticketNull) {
        /* exist.term() > member.term(): unreachable, membership terms are monotone (:188-191) */
        if (g->deadline > 0) {                                               /* :192-197 */
            g->deadline = RAFTING_TIMER_FENCING;
            /* onFencing(): Follower aborts its qualifier (Follower.java:171-175), Leader its
               replication head (Leader.java:113-117), Candidate its election head unless elected
               (Candidate.java:75-80).  The aborted heads die with the object: later replies carry
               a stale incarnation.  An elected Candidate's head was recorded when it was elected. */
        }
        g->ticketNull = 1;                                                   /* :198 */
    }
    /* constructor: RaftMember.java:20-26 persists (term, lastCandidate) */
    g->memberNull = 0;
    g->role = role; g->term = term; g->ballot = ballot;
    g->incarnation++;
    g->persistDirty = 1;
    g->currentLeader = -1; g->timeoutDetected = 0;                           /* Follower.java:21-24 */
    g->votes = 0;
    g->prepared = 0;                                                         /* Leader.java:24 */
    if (role == RAFTING_ROLE_CANDIDATE) start_election(c);                   /* Candidate.java:22-25 */
    if (!reset_timer(c, 0)) { /* AssertionError :213-215, unreachable: ticket is null */ }
    return 0;
}

/* ------------------------------------------------------------------------------------------ */
/* RaftContext.commitLog + RocksLog.markCommitted — RaftContext.java:244-255, RocksLog.java:100-109 */
/* ------------------------------------------------------------------------------------------ */
static int commit_log(ogroup_t* g, int64_t commitIndex) {
    if (commitIndex < g->log.commitIndex) return RAFTING_ERR_COMMIT_ROLLBACK;
    if (commitIndex > g->log.commitIndex) { g->log.commitIndex = commitIndex; g->commitDirty = 1; }
    return 0;   /* commitState / compactLog are host-side (apply + compaction) */
}

/* Leader.tryCommit — Leader.java:247-280 */
static int try_commit(octx_t* c) {
    ogroup_t* g = c->g; uint32_t F = c->e->F;
    int64_t m[MAXF], mi[2];
    for (uint32_t f = 0; f < F; f++) m[f] = g->st[f].matchIndex;
    orc_major_indices(m, (int)F, mi);
    int64_t full = mi[0], major = mi[1];
    if (full > major) return RAFTING_ERR_IMPOSSIBLE_REPL;                    /* :251-253 */
    if (major != 0) {
        int64_t t;
        if (!log_get(&g->log, major, &t)) { flag_err(g, RAFTING_ERR_TRY_COMMIT_FAILED); return 0; } /* NPE, :277 */
        int64_t ci = (t == g->term) ? major : full;                          /* :257-261 */
        if (ci != 0 && ci != g->log.commitIndex) return commit_log(g, ci);   /* :262-275 */
    }
    return 0;
}

/* ------------------------------------------------------------------------------------------ */
/* Leader.prepareReplication / replicateLog — Leader.java:30-50,142-245                         */
/* ------------------------------------------------------------------------------------------ */
static void prepare_replication(octx_t* c) {
    ogroup_t* g = c->g;
    if (g->prepared) return;                                                 /* :31 */
    int64_t li, lt; last_or_epoch(&g->log, &li, &lt);                        /* :32-34 */
    for (uint32_t f = 0; f < c->e->F; f++) {
        memset(&g->st[f], 0, sizeof(ostate_t));
        g->st[f].lastEpoch = g->log.epochIndex;                              /* :39 */
        g->st[f].nextIndex = (int64_t)((uint64_t)li + 1u);                   /* :40 */
    }
    g->prepared = 1;
}
static void put_plan(octx_t* c, uint32_t f, int kind, int hb, uint32_t count,
                     int64_t p0, int64_t p1, int64_t lastIndex, int64_t leaderCommit, int64_t epochIndex) {
    if (!c->plan_meta) return;
    c->plan_meta[f] = (uint64_t)kind | ((uint64_t)(hb ? 1 : 0) << 4) | ((uint64_t)count << 16) |
                      ((uint64_t)c->g->incarnation << 32);
    c->plan_pp[f].x = p0; c->plan_pp[f].y = p1;
    c->plan_lc[f].x = lastIndex; c->plan_lc[f].y = leaderCommit;
    c->plan_epoch[f] = epochIndex;
}
static int replicate_log(octx_t* c, int heartbeat, uint64_t unavail) {
    ogroup_t* g = c->g; olog_t* l = &g->log;
    prepare_replication(c);                                                  /* :145 */
    const int64_t epochIndex = l->epochIndex, epochTerm = l->epochTerm;      /* :152 */
    const int64_t leaderCommit = l->commitIndex;                             /* :153 */
    const int64_t now = c->now;                                              /* :155 */
    for (uint32_t f = 0; f < c->e->F; f++) {                                 /* :156 */
        ostate_t* s = &g->st[f];
        increase_mono(&s->lastRequest, now);                                 /* :158 */
        if ((unavail >> f) & 1u) {                                           /* :241-243 */
            stat_failure(s, now, 1, 0);
            put_plan(c, f, RAFTING_PLAN_UNAVAILABLE, heartbeat, 0, 0, 0, 0, 0, epochIndex);
            continue;
        }
        int limit = RAFTING_IN_FLIGHT_LIMIT / (heartbeat ? 10 : 1);          /* :162 */
        if (s->requestInFlight > limit) {                                    /* :163-166 */
            put_plan(c, f, RAFTING_PLAN_SKIP_INFLIGHT, heartbeat, 0, 0, 0, 0, 0, epochIndex);
            continue;
        }
        if (s->pendingInstallation) {                                        /* :168-190 */
            put_plan(c, f, RAFTING_PLAN_IS, heartbeat, 0, epochIndex, epochTerm, epochIndex, leaderCommit, epochIndex);
            s->requestInFlight++;                                            /* :173 */
            continue;
        }
        int64_t prevTerm = epochTerm, prevIndex = epochIndex, lastIndex;     /* :192 */
        int64_t nm1 = (int64_t)((uint64_t)s->nextIndex - 1u);
        int64_t nextIndex = nm1 > epochIndex ? nm1 : epochIndex;             /* :193 */
        int fetch = RAFTING_REPLICATE_LIMIT >> (heartbeat ? 1 : 0);          /* :194 */
        /* RaftLog.batch(nextIndex, fetch + 1) — RocksLog.java:131-166 */
        int64_t idx = nextIndex; int64_t len = fetch + 1;
        if (idx == epochIndex) { idx++; len--; }                             /* RocksLog :134-137 */
        int64_t e_first = 0, e_count = 0;                                    /* returned entries [e_first, e_first+e_count) */
        if (len > 0 && !log_empty(l)) {
            int64_t hiKey = idx + len - 1;
            if (idx < l->lo && l->lo <= hiKey) return RAFTING_ERR_LOG_VACANCY; /* RocksLog :161-163 (Error: aborts the loop) */
            int64_t a = idx > l->lo ? idx : l->lo;
            int64_t b = hiKey < l->hi ? hiKey : l->hi;
            if (a <= b) { e_first = a; e_count = b - a + 1; }
        }
        uint32_t count;
        if (e_count > 0) {                                                   /* :196 */
            if (e_first == nextIndex) {                                      /* :198-201 */
                int64_t t = 0; log_get(l, e_first, &t);
                prevTerm = t; prevIndex = e_first;
                e_first++; e_count--;
            } else if (e_first != epochIndex + 1) {                          /* :202-204 */
                return RAFTING_ERR_LOG_START;
            }
            lastIndex = (e_count == 0) ? prevIndex : e_first + e_count - 1;  /* :205-209 */
            count = (uint32_t)e_count;
        } else {
            lastIndex = epochIndex;                                          /* :210-212 */
            count = 0;
        }
        put_plan(c, f, RAFTING_PLAN_AE, heartbeat, count, prevIndex, prevTerm, lastIndex, leaderCommit, epochIndex); /* :216 */
        s->requestInFlight++;                                                /* :217 */
    }
    return 0;
}

/* Leader.isReady — Leader.java:52-64 */
static int leader_ready(octx_t* c) {
    ogroup_t* g = c->g;
    if (!g->prepared) return 0;
    int ready = 1, half = (int)c->e->F / 2;
    for (uint32_t f = 0; f < c->e->F; f++)
        if (state_ready(&g->st[f], c->e->cfg.avail_critical_point, c->e->cfg.recovery_cool_down_ms, c->now) &&
            ++ready > half) return 1;
    return 0;
}

/* ------------------------------------------------------------------------------------------ */
/* group ops                                                                                  */
/* ------------------------------------------------------------------------------------------ */
typedef struct { int valid; int success; int64_t term; } oreply_t;
static oreply_t reply(int64_t term, int success) { oreply_t r = {1, success, term}; return r; }

/* RaftStub.process -> Leader.acceptCommand -> RaftContext.acceptCommand -> RocksLog.newEntry
   (RaftStub.java:79-91, Leader.java:128-140, RaftContext.java:223-237, RocksLog.java:82-89) */
static int op_submit(octx_t* c, uint32_t count, uint64_t unavail) {
    ogroup_t* g = c->g; olog_t* l = &g->log;
    if (g->role != RAFTING_ROLE_LEADER) return RAFTING_ERR_NOT_LEADER;
    int ready = leader_ready(c);
    g->readyBit = ready;
    if (!ready) return RAFTING_ERR_NOT_READY;
    if (count == 0) count = 1;
    int64_t li, lt; int has = log_last(l, &li, &lt);
    if (!has && l->epochIndex != 0) return RAFTING_ERR_LOG_SHAPE;   /* reference would restart at index 1 */
    if ((!has || lt != g->term) && log_runs(l) >= RAFTING_TERM_RUNS) return RAFTING_ERR_TERM_RUNS_OVERFLOW;
    int64_t index = has ? li + 1 : 1;                               /* RocksLog :83-84 */
    for (uint32_t k = 0; k < count; k++) log_put(l, index + k, g->term);
    return replicate_log(c, 0, unavail);                            /* Leader.java:135 */
}

/* RaftRoutine.keepAlive / electionTimeout + *.onTimeout — RaftRoutine.java:53-77,
   Leader.java:119-126, Follower.java:156-168, Candidate.java:82-88 */
static int op_timeout(octx_t* c, uint64_t unavail) {
    ogroup_t* g = c->g;
    if (g->role == RAFTING_ROLE_LEADER) {
        if (g->deadline > 0 && reset_timer(c, 0)) return replicate_log(c, 1, unavail);
        return 0;
    }
    if (!(g->deadline > 0)) return 0;                               /* :66-67 */
    g->deadline = RAFTING_TIMER_TIMEOUT;                            /* :68 */
    if (g->role == RAFTING_ROLE_FOLLOWER) {
        if (c->e->cfg.pre_vote) {                                   /* Follower.java:158-164 */
            int64_t t = g->term;
            int err = switch_to(c, RAFTING_ROLE_FOLLOWER, g->term, g->ballot);
            if (err) return err;
            if (g->role == RAFTING_ROLE_FOLLOWER && g->term == t) prepare_election(c);
            return 0;
        }
        return switch_to(c, RAFTING_ROLE_CANDIDATE, (int64_t)((uint64_t)g->term + 1u), (int)c->e->cfg.local_slot); /* :166 */
    }
    /* Candidate.onTimeout — Candidate.java:82-88 */
    return switch_to(c, RAFTING_ROLE_CANDIDATE, (int64_t)((uint64_t)g->term + 1u), (int)c->e->cfg.local_slot);
}

/* Follower.logContains — Follower.java:177-191.  returns 1/0 or -err */
static int log_contains(const olog_t* l, int64_t index, int64_t term) {
    if (index == 0 && term == 0) return 1;
    if (index == 0 || term == 0) return -RAFTING_ERR_INDEX_TERM_ZERO;
    if (index <= l->epochIndex) {
        if (index == l->epochIndex && term != l->epochTerm) return -RAFTING_ERR_EPOCH_TERM_MISMATCH;
        return 1;
    }
    int64_t t;
    return log_get(l, index, &t) && t == term;
}
/* Follower.logUpToDate — Follower.java:193-207.  returns 1/0 or -err */
static int log_up_to_date(const olog_t* l, int64_t index, int64_t term) {
    int64_t li, lt;
    if (log_last(l, &li, &lt)) return term > lt || (term == lt && index >= li);
    if ((index > l->epochIndex && term < l->epochTerm) || (index == l->epochIndex && term != l->epochTerm))
        return -RAFTING_ERR_IMPOSSIBLE_LOG;
    return index >= l->epochIndex;
}

/* Follower.appendEntries body after the role pre-filters — Follower.java:52-87 */
static int follower_append(octx_t* c, int peer, int64_t term, int64_t prevIndex, int64_t prevTerm,
                           int64_t first, uint32_t n, const int64_t* terms, int64_t leaderCommit, oreply_t* rep) {
    ogroup_t* g = c->g; olog_t* l = &g->log;
    g->currentLeader = peer;                                                 /* :54 */
    int err = 0;
    int lc = log_contains(l, prevIndex, prevTerm);                           /* :57 */
    if (lc < 0) { err = -lc; goto finally; }
    if (!lc) { *rep = reply(g->term, 0); goto finally; }                     /* :58 */
    /* purgeEntries — :209-221 */
    if (n > 0 && first <= l->epochIndex) {
        int64_t skip = l->epochIndex - first + 1;
        if ((uint64_t)skip >= n) { n = 0; } else { first += skip; terms += skip; n -= (uint32_t)skip; }
    }
    if (n > 0) {                                                             /* :68 */
        /* RocksLog.conflict — RocksLog.java:199-216 */
        int64_t conflictIndex = 0;
        for (uint32_t i = 0; i < n; i++) {
            int64_t t;
            if (!log_get(l, first + i, &t)) break;                           /* NOT_FOUND: the rest is new */
            if (t != terms[i]) { conflictIndex = first + i; break; }
        }
        /* RocksLog.append pre-checks — RocksLog.java:170-188 (entries are contiguous by construction) */
        int64_t hiAfter = (conflictIndex != 0 && !log_empty(l) && l->hi >= conflictIndex) ? conflictIndex - 1 : l->hi;
        int emptyAfter = log_empty(l) || hiAfter < l->lo;
        int64_t prevLogIndex;
        if (!emptyAfter && l->lo <= first) prevLogIndex = first < hiAfter ? first : hiAfter;   /* seekForPrev */
        else if (!emptyAfter) { err = RAFTING_ERR_LOG_SHAPE; goto finally; }  /* stored keys all above entries[0] */
        else prevLogIndex = l->epochIndex;
        /* capacity pre-check of the engine's run-length term table: reject before mutating */
        {
            /* runs after truncate */
            uint32_t runs = 0; int64_t lastT = 0; int have = 0;
            if (!emptyAfter) {
                for (int64_t i = l->lo; i <= hiAfter; i++) {
                    int64_t t = l->terms[i - l->base];
                    if (!have || t != lastT) { runs++; lastT = t; have = 1; }
                }
            }
            for (uint32_t i = 0; i < n; i++) {
                if (first + i > prevLogIndex) {
                    if (!have || terms[i] != lastT) { runs++; lastT = terms[i]; have = 1; }
                }
            }
            int firstPutOk = emptyAfter ? (first == l->epochIndex + 1) : 1;
            int contOk = !(first > prevLogIndex + 1);
            if (firstPutOk && contOk && runs > RAFTING_TERM_RUNS) { err = RAFTING_ERR_TERM_RUNS_OVERFLOW; goto finally; }
        }
        if (conflictIndex != 0) log_truncate(l, conflictIndex);              /* Follower.java:70-72 */
        if (emptyAfter && first != l->epochIndex + 1) { err = RAFTING_ERR_LOG_NOT_FOLLOW_EPOCH; goto finally; } /* RocksLog :175-177 */
        if (first > prevLogIndex + 1) { err = RAFTING_ERR_LOG_NOT_CONTINUOUS; goto finally; }                   /* RocksLog :185-187 */
        for (uint32_t i = 0; i < n; i++)
            if (first + i > prevLogIndex) log_put(l, first + i, terms[i]);   /* RocksLog :183-191 */
    }
    if (leaderCommit > l->epochIndex) {                                      /* Follower.java:76-82 */
        int64_t li, lt;
        if (log_last(l, &li, &lt)) {
            int64_t ci = leaderCommit < li ? leaderCommit : li;
            /* RAFTING_CFG_LENIENT_FOLLOWER_COMMIT (opt-in, NOT the reference): a leader that knows less than this
               follower about what is committed is simply ignored, as in the Raft paper (commitIndex = max(...)) */
            if ((c->e->cfg.flags & RAFTING_CFG_LENIENT_FOLLOWER_COMMIT) && ci < g->log.commitIndex) ci = g->log.commitIndex;
            err = commit_log(g, ci);
            if (err) goto finally;
        }
    }
finally:
    reset_timer(c, 0);                                                       /* :83-85 */
    if (!err && !rep->valid) *rep = reply(term, 1);                          /* :87 */
    return err;
}

static int follower_append_entries(octx_t* c, int peer, int64_t term, int64_t prevIndex, int64_t prevTerm,
                                   int64_t first, uint32_t n, const int64_t* terms, int64_t leaderCommit,
                                   oreply_t* rep);

/* dispatch of RaftParticipant.appendEntries by the live role */
static int op_append_entries(octx_t* c, int peer, int64_t term, int64_t prevIndex, int64_t prevTerm,
                             int64_t first, uint32_t n, const int64_t* terms, int64_t leaderCommit, oreply_t* rep) {
    ogroup_t* g = c->g;
    int err;
    switch (g->role) {
    case RAFTING_ROLE_LEADER:                                                /* Leader.java:66-86 */
        if (peer == (int)c->e->cfg.local_slot) return RAFTING_ERR_LEADER_SELF_AE;
        if (term < g->term) { *rep = reply(g->term, 0); return 0; }
        if (term == g->term) return RAFTING_ERR_TWO_LEADERS;
        err = switch_to(c, RAFTING_ROLE_FOLLOWER, g->term, g->ballot);
        if (err) return err;
        return follower_append_entries(c, peer, term, prevIndex, prevTerm, first, n, terms, leaderCommit, rep);
    case RAFTING_ROLE_CANDIDATE:                                             /* Candidate.java:28-41 */
        if (term < g->term) { *rep = reply(g->term, 0); return 0; }
        err = switch_to(c, RAFTING_ROLE_FOLLOWER, term, g->ballot);
        if (err) return err;
        return follower_append_entries(c, peer, term, prevIndex, prevTerm, first, n, terms, leaderCommit, rep);
    default:
        return follower_append_entries(c, peer, term, prevIndex, prevTerm, first, n, terms, leaderCommit, rep);
    }
}
/* Follower.appendEntries — Follower.java:35-88 */
static int follower_append_entries(octx_t* c, int peer, int64_t term, int64_t prevIndex, int64_t prevTerm,
                                   int64_t first, uint32_t n, const int64_t* terms, int64_t leaderCommit,
                                   oreply_t* rep) {
    ogroup_t* g = c->g;
    if (term < g->term) { *rep = reply(g->term, 0); return 0; }              /* :39-41 */
    reset_timer(c, 1);                                                       /* :43 */
    if (term > g->term || g->timeoutDetected) {                              /* :45-47 */
        int err = switch_to(c, RAFTING_ROLE_FOLLOWER, term, g->ballot);
        if (err) return err;
        /* re-dispatch on the fresh Follower: term == currentTerm, !timeoutDetected */
        reset_timer(c, 1);
    } else if (g->currentLeader != -1 && peer != g->currentLeader) {         /* :48-50 */
        return RAFTING_ERR_FOLLOWER_TWO_LEADERS;                             /* timer stays muted */
    }
    return follower_append(c, peer, term, prevIndex, prevTerm, first, n, terms, leaderCommit, rep);
}

/* Follower.requestVote — Follower.java:108-127 */
static int follower_request_vote(octx_t* c, int peer, int64_t term, int64_t lastIndex, int64_t lastTerm, oreply_t* rep) {
    ogroup_t* g = c->g;
    if (term < g->term) { *rep = reply(g->term, 0); return 0; }              /* :112-113 */
    if (term == g->term) { *rep = reply(g->term, peer == g->ballot); return 0; }  /* :114-116 */
    reset_timer(c, 1);                                                       /* :118 */
    int up = log_up_to_date(&g->log, lastIndex, lastTerm);                   /* :122 */
    if (up < 0) return -up;                                                  /* timer stays muted */
    int voteFor = up ? peer : -1;                                            /* :123 */
    int err = switch_to(c, RAFTING_ROLE_FOLLOWER, term, voteFor);            /* :125 */
    if (err) return err;
    *rep = reply(g->term, peer == g->ballot);                                /* :126 -> :114-116 */
    return 0;
}
static int op_request_vote(octx_t* c, int peer, int64_t term, int64_t lastIndex, int64_t lastTerm, oreply_t* rep) {
    ogroup_t* g = c->g; int err;
    switch (g->role) {
    case RAFTING_ROLE_LEADER:                                                /* Leader.java:93-111 */
        if (term < g->term) { *rep = reply(g->term, 0); return 0; }
        if (term == g->term) {
            if (g->ballot == (int)c->e->cfg.local_slot) { *rep = reply(g->term, 0); return 0; }
            return RAFTING_ERR_LEADER_VOTE_SELF;
        }
        err = switch_to(c, RAFTING_ROLE_FOLLOWER, g->term, peer);
        if (err) return err;
        return follower_request_vote(c, peer, term, lastIndex, lastTerm, rep);
    case RAFTING_ROLE_CANDIDATE:                                             /* Candidate.java:49-72 */
        if (peer == (int)c->e->cfg.local_slot) return RAFTING_ERR_CANDIDATE_SELF_RV;
        if (term < g->term) { *rep = reply(g->term, 0); return 0; }
        if (term == g->term) {
            if (peer != g->ballot) { *rep = reply(g->term, 0); return 0; }
            else if (g->ballot != (int)c->e->cfg.local_slot) return RAFTING_ERR_CANDIDATE_VOTE_SELF;
        }
        /* RAFTING_CFG_STRICT_CANDIDATE_VOTE (opt-in, NOT the reference): step down at the own term first, like the Leader
           does (Leader.java:106-108), so that Follower.requestVote applies logUpToDate to the higher-term request */
        if ((c->e->cfg.flags & RAFTING_CFG_STRICT_CANDIDATE_VOTE) && term > g->term)
            err = switch_to(c, RAFTING_ROLE_FOLLOWER, g->term, g->ballot);
        else
            err = switch_to(c, RAFTING_ROLE_FOLLOWER, term, peer);
        if (err) return err;
        return follower_request_vote(c, peer, term, lastIndex, lastTerm, rep);
    default:
        return follower_request_vote(c, peer, term, lastIndex, lastTerm, rep);
    }
}
static int op_pre_vote(octx_t* c, int peer, int64_t term, int64_t lastIndex, int64_t lastTerm, oreply_t* rep) {
    ogroup_t* g = c->g;
    switch (g->role) {
    case RAFTING_ROLE_LEADER: *rep = reply(g->term, 0); return 0;            /* Leader.java:88-91 */
    case RAFTING_ROLE_CANDIDATE: return op_request_vote(c, peer, term, lastIndex, lastTerm, rep);  /* Candidate.java:43-46 */
    default: {                                                               /* Follower.java:91-105 */
        if (term <= g->term || !g->timeoutDetected) { *rep = reply(g->term, 0); return 0; }
        reset_timer(c, 1);
        int up = log_up_to_date(&g->log, lastIndex, lastTerm);
        reset_timer(c, 0);                                                   /* finally */
        if (up < 0) return -up;
        *rep = reply(g->term, up);
        return 0;
    }
    }
}
/* installSnapshot — RaftMember.java:61-66, Follower.java:130-153 */
static int op_install_snapshot(octx_t* c, int peer, int64_t term, int hostResult, oreply_t* rep) {
    ogroup_t* g = c->g; (void)peer;
    if (g->role != RAFTING_ROLE_FOLLOWER) {
        if (term >= g->term) return RAFTING_ERR_IS_BEFORE_AE;
        *rep = reply(g->term, 0); return 0;
    }
    reset_timer(c, 1);                                                       /* :134 (before the term checks) */
    if (term < g->term) { *rep = reply(g->term, 0); return 0; }              /* :136-137, timer stays muted */
    if (term > g->term) return RAFTING_ERR_IS_BEFORE_AE;                     /* :138-139 */
    if (g->timeoutDetected) {                                                /* :140-143 */
        int err = switch_to(c, RAFTING_ROLE_FOLLOWER, g->term, g->ballot);
        if (err) return err;
        reset_timer(c, 1);
    }
    *rep = reply(g->term, hostResult);                                       /* :148-149 (download/apply is host IO) */
    reset_timer(c, 0);                                                       /* :150-152 */
    return 0;
}

/* ------------------------------------------------------------------------------------------ */
/* lane events (Async callbacks)                                                              */
/* ------------------------------------------------------------------------------------------ */
/* AE-Echo / IS-Echo — Leader.java:174-188,218-237 */
static int ev_ack(octx_t* c, uint32_t f, int kind, int outcome, int success, int64_t respTerm,
                  int64_t epochAtSend, int64_t lastAtSend, uint32_t inc) {
    ogroup_t* g = c->g;
    if (!(g->role == RAFTING_ROLE_LEADER && inc == g->incarnation && g->prepared)) return 0;  /* dead State object */
    ostate_t* s = &g->st[f];
    s->requestInFlight--;                                                    /* :176 / :221 */
    if (outcome == RAFTING_OUT_OK) {
        if (respTerm > g->term) {                                            /* :178-180 / :224-226 */
            return switch_to(c, RAFTING_ROLE_FOLLOWER, respTerm, lane_to_slot(c->e, f));
        }
        stat_success(s, c->now, !success);                                   /* :182 / :228 */
        int snapshot = kind == RAFTING_EV_IS_ACK;
        int err = update_index(s, epochAtSend, snapshot ? epochAtSend : lastAtSend, success, snapshot); /* :183 / :229 */
        if (err) return err;
        if (!snapshot && success) return try_commit(c);                      /* :230-232 */
    } else {
        stat_failure(s, c->now, outcome == RAFTING_OUT_ERROR, 0);            /* :186 / :235 */
    }
    return 0;
}
/* PV-Echo — Follower.java:258-270 */
static int ev_prevote_reply(octx_t* c, uint32_t f, int outcome, int success, int64_t respTerm, uint32_t inc) {
    ogroup_t* g = c->g;
    if (!(g->role == RAFTING_ROLE_FOLLOWER && inc == g->incarnation && g->timeoutDetected)) return 0;
    if (outcome != RAFTING_OUT_OK) return 0;
    int64_t nextTerm = (int64_t)((uint64_t)g->term + 1u);
    if (respTerm > nextTerm) return switch_to(c, RAFTING_ROLE_FOLLOWER, respTerm, lane_to_slot(c->e, f));
    if (success) {
        if (++g->votes >= majority(c->e))
            return switch_to(c, RAFTING_ROLE_CANDIDATE, nextTerm, (int)c->e->cfg.local_slot);
    }
    return 0;
}
/* RV-Echo — Candidate.java:112-134 */
static int ev_vote_reply(octx_t* c, uint32_t f, int outcome, int success, int64_t respTerm, uint32_t inc) {
    ogroup_t* g = c->g;
    if (g->role == RAFTING_ROLE_CANDIDATE && inc == g->incarnation) {
        if (outcome != RAFTING_OUT_OK) return 0;
        if (respTerm > g->term) return switch_to(c, RAFTING_ROLE_FOLLOWER, respTerm, lane_to_slot(c->e, f));
        if (success) {
            if (++g->votes >= majority(c->e)) {
                g->electedInc = g->incarnation; g->electedTerm = g->term; g->electedAborted = 0;  /* elected = true */
                return switch_to(c, RAFTING_ROLE_LEADER, g->term, (int)c->e->cfg.local_slot);
            }
        }
        return 0;
    }
    /* replies to an elected Candidate keep running its callback after it was fenced
       (Candidate.onFencing skips the abort when elected — Candidate.java:75-80) */
    if (g->electedInc != 0 && inc == g->electedInc && !g->electedAborted) {
        if (outcome != RAFTING_OUT_OK) return 0;
        if (respTerm > g->electedTerm) {
            g->electedAborted = 1;                                           /* head.abortRequests() */
            return switch_to(c, RAFTING_ROLE_FOLLOWER, respTerm, lane_to_slot(c->e, f));
        }
        if (success) return switch_to(c, RAFTING_ROLE_LEADER, g->electedTerm, (int)c->e->cfg.local_slot);
    }
    return 0;
}

/* ------------------------------------------------------------------------------------------ */
/* engine                                                                                     */
/* ------------------------------------------------------------------------------------------ */
orc_engine_t* orc_create(const rafting_cfg_t* cfg) {
    if (!cfg || cfg->replicas < 2 || cfg->replicas > RAFTING_MAX_REPLICAS || cfg->local_slot >= cfg->replicas)
        return NULL;
    orc_engine_t* e = (orc_engine_t*)calloc(1, sizeof(*e));
    e->cfg = *cfg;
    e->F = cfg->replicas - 1;
    e->groups = (ogroup_t*)calloc(cfg->max_groups, sizeof(ogroup_t));
    return e;
}
static void pool_destroy(struct orc_pool* p);
void orc_destroy(orc_engine_t* e) {
    if (!e) return;
    pool_destroy(e->pool);
    for (uint32_t i = 0; i < e->cfg.max_groups; i++) free(e->groups[i].log.terms);
    free(e->groups); free(e);
}

/* ContextManager.buildContext + RaftContext.initialize — RaftContext.java:91-113 */
int orc_group_open(orc_engine_t* e, uint32_t gid, const rafting_group_init_t* in) {
    if (!e || gid >= e->cfg.max_groups || !in) return RAFTING_E_INVAL;
    ogroup_t* g = &e->groups[gid];
    if (g->alive) return RAFTING_E_INVAL;
    free(g->log.terms);
    memset(g, 0, sizeof(*g));
    olog_t* l = &g->log;
    l->epochIndex = in->epoch_index; l->epochTerm = in->epoch_term;
    l->commitIndex = in->commit_index;
    l->lo = 1; l->hi = 0;
    if (in->last_index >= in->first_index) {
        if (in->first_index != in->epoch_index && in->first_index != in->epoch_index + 1) return RAFTING_E_INVAL;
        for (int64_t i = in->first_index; i <= in->last_index; i++) log_put(l, i, in->last_term);
    }
    g->alive = 1; g->memberNull = 1; g->ticketNull = 1;
    g->currentLeader = -1; g->ballot = -1;
    octx_t c; memset(&c, 0, sizeof(c));
    c.e = e; c.g = g; c.gid = gid; c.now = in->now_ms; c.draw = in->rand_ms;
    switch_to(&c, RAFTING_ROLE_FOLLOWER, in->term, in->ballot);             /* :104 */
    g->persistDirty = 0;
    return 0;
}
int orc_group_open_bulk(orc_engine_t* e, uint32_t first, uint32_t count, const rafting_group_init_t* inits) {
    for (uint32_t i = 0; i < count; i++) { int r = orc_group_open(e, first + i, &inits[i]); if (r) return r; }
    return 0;
}
/* restart over a stored log spanning several terms: runs[k] = (first index, term), oldest first */
int orc_group_load_runs(orc_engine_t* e, uint32_t gid, const rafting_i64x2_t* runs, uint32_t n) {
    if (!e || !runs || gid >= e->cfg.max_groups || n == 0) return RAFTING_E_INVAL;
    if (n > RAFTING_TERM_RUNS) return RAFTING_E_CAPACITY;
    olog_t* l = &e->groups[gid].log;
    if (!e->groups[gid].alive || log_empty(l) || runs[0].x != l->lo) return RAFTING_E_INVAL;
    int64_t lastT; log_get(l, l->hi, &lastT);
    if (runs[n - 1].y != lastT) return RAFTING_E_INVAL;
    for (uint32_t k = 1; k < n; k++)
        if (runs[k].x <= runs[k - 1].x || runs[k].x > l->hi || runs[k].y == runs[k - 1].y) return RAFTING_E_INVAL;
    for (uint32_t k = 0; k < n; k++) {
        int64_t end = (k + 1 < n) ? runs[k + 1].x - 1 : l->hi;
        for (int64_t i = runs[k].x; i <= end; i++) l->terms[i - l->base] = runs[k].y;
    }
    return 0;
}
int orc_group_close(orc_engine_t* e, uint32_t gid) {
    if (!e || gid >= e->cfg.max_groups) return RAFTING_E_INVAL;
    e->groups[gid].alive = 0;
    return 0;
}

static uint32_t role_word(const ogroup_t* g) {
    return (uint32_t)g->role | ((uint32_t)(g->ballot + 1) << 8) | ((uint32_t)(g->currentLeader + 1) << 16) |
           ((uint32_t)(g->timeoutDetected ? 1 : 0) << 24) | ((uint32_t)(g->readyBit ? 1 : 0) << 25) |
           ((uint32_t)(g->persistDirty ? 1 : 0) << 30) | ((uint32_t)(g->commitDirty ? 1 : 0) << 31);
}

/* one row of one group: [sweep?] op(r); ev(r,0); ...; ev(r,F-1) — the canonical serial order (DESIGN.md §3) */
static void step_row(orc_engine_t* e, const rafting_inbox_t* in, const rafting_outbox_t* out,
                     uint32_t i, uint32_t n, uint32_t gid, ogroup_t* g, uint32_t r, uint64_t* events) {
    const uint32_t F = e->F;
    size_t gi = (size_t)r * n + i;
    octx_t c; memset(&c, 0, sizeof(c));
    c.e = e; c.g = g; c.gid = gid;
    if (out->plan_meta) {
        c.plan_meta = out->plan_meta + gi * F; c.plan_pp = out->plan_pp + gi * F;
        c.plan_lc = out->plan_lc + gi * F; c.plan_epoch = out->plan_epoch + gi * F;
        for (uint32_t f = 0; f < F; f++) c.plan_meta[f] = 0;
    }
    if (out->ballot_meta) {
        c.ballot_meta = out->ballot_meta + gi; c.ballot_term = out->ballot_term + gi; c.ballot_last = out->ballot_last + gi;
        *c.ballot_meta = 0;
    }
    if (out->rep_meta) { out->rep_meta[gi] = 0; }
    /* ---- group op (or sweep) ---- */
    int64_t sweep = in->row_now ? in->row_now[r] : 0;
    uint32_t kind = RAFTING_OP_NONE, meta = 0, entoff = 0;
    if (sweep != 0) {
        /* timer sweep row: implied TIMEOUT for groups whose timer is due (RaftRoutine.java:53-77) */
        if (g->alive) {
            int due = (g->role == RAFTING_ROLE_LEADER) ? (g->hbDue <= sweep)
                      : (g->deadline > 0 && g->deadline != I64_MAX && g->deadline <= sweep);
            if (due) { kind = RAFTING_OP_TIMEOUT; c.now = sweep; c.draw = 0; }
        }
    } else if (in->op_meta) {
        uint64_t m = in->op_meta[gi];
        meta = (uint32_t)m; entoff = (uint32_t)(m >> 32);
        kind = RAFTING_OP_KIND(meta);
        if (kind != RAFTING_OP_NONE) { c.now = in->op_nr[gi].x; c.draw = in->op_nr[gi].y; }
    }
    if (kind != RAFTING_OP_NONE) {
        (*events)++;
        int err = 0; oreply_t rep = {0, 0, 0};
        int64_t a = 0, b = 0, cc = 0, d = 0;
        if (sweep == 0) {
            if (in->op_ab) { a = in->op_ab[gi].x; b = in->op_ab[gi].y; }
            if (in->op_cd) { cc = in->op_cd[gi].x; d = in->op_cd[gi].y; }
        }
        int peer = (int)RAFTING_OP_PEER(meta); uint32_t count = RAFTING_OP_COUNT(meta);
        if (!g->alive) err = RAFTING_ERR_CLOSED_GROUP;
        /* the caller promised no inbound requests: one found anyway is refused (rafting_b200.h, RAFTING_INBOX_NO_REQUESTS) */
        else if (kind > RAFTING_OP_TIMEOUT && (in->flags & RAFTING_INBOX_NO_REQUESTS)) err = RAFTING_ERR_BAD_EVENT;
        else switch (kind) {
        case RAFTING_OP_SUBMIT:  err = op_submit(&c, count, (uint64_t)a); break;
        case RAFTING_OP_TIMEOUT: err = op_timeout(&c, (uint64_t)a); break;
        case RAFTING_OP_AE_REQUEST: {
            int64_t first = in->op_e ? in->op_e[gi] : (int64_t)((uint64_t)b + 1u);
            const int64_t* terms = in->ent_terms ? in->ent_terms + entoff : NULL;
            if (count > 0 && (!terms || (uint64_t)entoff + count > in->ent_count)) { err = RAFTING_ERR_BAD_EVENT; break; }
            err = op_append_entries(&c, peer, a, b, cc, first, count, terms, d, &rep);
            break;
        }
        case RAFTING_OP_PREVOTE_REQ: err = op_pre_vote(&c, peer, a, b, cc, &rep); break;
        case RAFTING_OP_VOTE_REQ:    err = op_request_vote(&c, peer, a, b, cc, &rep); break;
        case RAFTING_OP_IS_REQUEST:  err = op_install_snapshot(&c, peer, a, d != 0, &rep); break;
        case RAFTING_OP_FLUSH:       err = log_flush(&g->log, b, cc); break;
        default: err = RAFTING_ERR_BAD_EVENT;
        }
        if (err) { if (g->alive) flag_err(g, err); rep.valid = 0; }
        if (out->rep_meta) {
            out->rep_meta[gi] = (uint32_t)(rep.valid ? 1 : 0) | ((uint32_t)(rep.success ? 1 : 0) << 1) | ((uint32_t)err << 8);
            out->rep_term[gi] = rep.valid ? rep.term : 0;
        }
    }
    /* ---- lane events f = 0..F-1 ---- */
    if (in->ev_meta) {
        for (uint32_t f = 0; f < F; f++) {
            size_t li = gi * F + f;
            uint64_t m = in->ev_meta[li];
            uint32_t ek = RAFTING_EVM_KIND(m);
            if (ek == RAFTING_EV_NONE) continue;
            (*events)++;
            if (!g->alive) continue;
            c.now = in->ev_tn[li].y; c.draw = 0;
            int64_t respTerm = in->ev_tn[li].x;
            int outcome = (int)RAFTING_EVM_OUTCOME(m), success = (int)RAFTING_EVM_SUCCESS(m);
            uint32_t inc = RAFTING_EVM_INC(m);
            int err = 0;
            switch (ek) {
            case RAFTING_EV_AE_ACK: case RAFTING_EV_IS_ACK:
                err = ev_ack(&c, f, (int)ek, outcome, success, respTerm,
                             in->ev_el ? in->ev_el[li].x : 0, in->ev_el ? in->ev_el[li].y : 0, inc);
                break;
            case RAFTING_EV_PV_REPLY: err = ev_prevote_reply(&c, f, outcome, success, respTerm, inc); break;
            case RAFTING_EV_RV_REPLY: err = ev_vote_reply(&c, f, outcome, success, respTerm, inc); break;
            default: err = RAFTING_ERR_BAD_EVENT;
            }
            if (err) flag_err(g, err);
        }
    }
}
/* end-of-step snapshot columns: by gid, or by position in the active list (RAFTING_INBOX_COMPACT_GROUPS) */
static void step_end(const rafting_inbox_t* in, const rafting_outbox_t* out, uint32_t i, uint32_t gid, ogroup_t* g) {
    const uint32_t go = (in->gids && (in->flags & RAFTING_INBOX_COMPACT_GROUPS)) ? i : gid;
    if (out->commit_index) out->commit_index[go] = g->log.commitIndex;
    if (out->current_term) out->current_term[go] = g->term;
    if (out->role_word)    out->role_word[go] = role_word(g);
    if (out->incarnation)  out->incarnation[go] = g->incarnation;
    if (out->err_word)     out->err_word[go] = g->errWord;
    if (out->last_entry)   last_or_epoch(&g->log, &out->last_entry[go].x, &out->last_entry[go].y);
}
/* A chunk of consecutive positions, ROW-major: every column of the batch is [row][group], so walking a row across the
   chunk streams contiguous memory, while one group's rows lie rows * n * 8 bytes apart (a different page per access).  The
   per-group order of rows — the only order the semantics fix — is unchanged; the 64 contexts of a chunk stay in L1/L2. */
static void step_chunk(orc_engine_t* e, const rafting_inbox_t* in, const rafting_outbox_t* out,
                       uint32_t c0, uint32_t c1, uint32_t n, uint64_t* events) {
    for (uint32_t i = c0; i < c1; i++) {
        uint32_t gid = in->gids ? in->gids[i] : i;
        if (gid < e->cfg.max_groups) { e->groups[gid].persistDirty = 0; e->groups[gid].commitDirty = 0; }
    }
    for (uint32_t r = 0; r < in->rows; r++)
        for (uint32_t i = c0; i < c1; i++) {
            uint32_t gid = in->gids ? in->gids[i] : i;
            if (gid < e->cfg.max_groups) step_row(e, in, out, i, n, gid, &e->groups[gid], r, events);
        }
    for (uint32_t i = c0; i < c1; i++) {
        uint32_t gid = in->gids ? in->gids[i] : i;
        if (gid < e->cfg.max_groups) step_end(in, out, i, gid, &e->groups[gid]);
    }
}

/* The loop threads live as long as the engine (the reference's ContextLoop-k threads do, too): a step hands every
   thread its share and waits for all of them — no thread creation inside the timed region of the CPU baseline. */
typedef struct orc_pool {
    pthread_t th[256]; int T;
    pthread_mutex_t mu; pthread_cond_t go, done;
    uint64_t gen; int pending, quit;
    uint32_t next_chunk;     /* work queue of the step in flight: chunks of 64 consecutive groups, taken with an atomic add */
    orc_engine_t* e; const rafting_inbox_t* in; const rafting_outbox_t* out; uint32_t n;
    uint64_t events[256];
    int ids[256];
    struct orc_pool* self[256];
} orc_pool_t;
typedef struct { orc_pool_t* p; int t; } pool_arg_t;

static void run_share(orc_pool_t* p, int t) {
    /* groups are bound to loops round-robin (EventLoopGroup.next(), EventLoopGroup.java:77-80) — here in chunks of 64
       consecutive groups, so that two loop threads never write the same cache line of a batch column (in the JVM every
       context is its own heap object; strict per-group round-robin over SoA columns would charge the CPU baseline for
       false sharing the reference does not have).  Results do not depend on the binding. */
    /* round 2: the chunks are handed out dynamically (one atomic add per 64 groups) instead of by a fixed stride, so a loop
       thread that lost its core for a while (hyper-thread sibling, remote NUMA node, another tenant) no longer sets the
       step time: a faster and steadier CPU baseline than the reference's fixed binding would give. */
    uint64_t ev = 0;
    const uint32_t nchunks = (p->n + 63u) / 64u;
    for (;;) {
        const uint32_t c = __atomic_fetch_add(&p->next_chunk, 1u, __ATOMIC_RELAXED);
        if (c >= nchunks) break;
        const uint32_t c0 = c * 64u, c1 = c0 + 64u < p->n ? c0 + 64u : p->n;
        step_chunk(p->e, p->in, p->out, c0, c1, p->n, &ev);
    }
    p->events[t] = ev;
}
static void* pool_main(void* a) {
    pool_arg_t* pa = (pool_arg_t*)a; orc_pool_t* p = pa->p; const int t = pa->t; free(pa);
    uint64_t seen = 0;
    for (;;) {
        pthread_mutex_lock(&p->mu);
        while (p->gen == seen && !p->quit) pthread_cond_wait(&p->go, &p->mu);
        if (p->quit) { pthread_mutex_unlock(&p->mu); return NULL; }
        seen = p->gen;
        pthread_mutex_unlock(&p->mu);
        run_share(p, t);
        pthread_mutex_lock(&p->mu);
        if (--p->pending == 0) pthread_cond_signal(&p->done);
        pthread_mutex_unlock(&p->mu);
    }
}
static orc_pool_t* pool_create(int T) {
    orc_pool_t* p = (orc_pool_t*)calloc(1, sizeof(*p));
    if (!p) return NULL;
    p->T = T;
    pthread_mutex_init(&p->mu, NULL); pthread_cond_init(&p->go, NULL); pthread_cond_init(&p->done, NULL);
    /* loop thread t is pinned to the t-th CPU this process may run on (wrapping): no migrations inside the timed region */
    cpu_set_t allowed; int ncpu = 0, cpus[1024];
    if (sched_getaffinity(0, sizeof(allowed), &allowed) == 0)
        for (int c = 0; c < CPU_SETSIZE && ncpu < 1024; c++) if (CPU_ISSET(c, &allowed)) cpus[ncpu++] = c;
    for (int t = 0; t < T; t++) {
        pool_arg_t* a = (pool_arg_t*)malloc(sizeof(*a)); a->p = p; a->t = t;
        pthread_create(&p->th[t], NULL, pool_main, a);
        if (ncpu > 0 && !getenv("ORACLE_NO_PIN")) {
            cpu_set_t one; CPU_ZERO(&one); CPU_SET(cpus[t % ncpu], &one);
            pthread_setaffinity_np(p->th[t], sizeof(one), &one);
        }
    }
    return p;
}
static void pool_destroy(struct orc_pool* p) {
    if (!p) return;
    pthread_mutex_lock(&p->mu); p->quit = 1; pthread_cond_broadcast(&p->go); pthread_mutex_unlock(&p->mu);
    for (int t = 0; t < p->T; t++) pthread_join(p->th[t], NULL);
    pthread_mutex_destroy(&p->mu); pthread_cond_destroy(&p->go); pthread_cond_destroy(&p->done);
    free(p);
}
int orc_step(orc_engine_t* e, const rafting_inbox_t* in, const rafting_outbox_t* out, int threads) {
    if (!e || !in || !out) return RAFTING_E_INVAL;
    uint32_t n = in->gids ? in->n_active : e->cfg.max_groups;
    if (threads <= 1) {
        uint64_t ev = 0;
        for (uint32_t c0 = 0; c0 < n; c0 += 64u) step_chunk(e, in, out, c0, c0 + 64u < n ? c0 + 64u : n, n, &ev);
        e->events += ev;
        return 0;
    }
    if (threads > 256) threads = 256;
    if (e->pool && e->pool->T != threads) { pool_destroy(e->pool); e->pool = NULL; }
    if (!e->pool) { e->pool = pool_create(threads); if (!e->pool) return RAFTING_E_NOMEM; }
    orc_pool_t* p = e->pool;
    pthread_mutex_lock(&p->mu);
    p->e = e; p->in = in; p->out = out; p->n = n; p->pending = threads; p->next_chunk = 0; p->gen++;
    pthread_cond_broadcast(&p->go);
    while (p->pending) pthread_cond_wait(&p->done, &p->mu);
    pthread_mutex_unlock(&p->mu);
    for (int t = 0; t < threads; t++) e->events += p->events[t];
    return 0;
}
uint64_t orc_events_processed(orc_engine_t* e) { return e ? e->events : 0; }

static uint64_t fnv1a(uint64_t h, uint64_t v) {
    for (int i = 0; i < 8; i++) { h ^= (v >> (8 * i)) & 0xff; h *= 0x100000001B3ull; }
    return h;
}
int orc_state_export(orc_engine_t* e, uint32_t gid, rafting_group_state_t* o) {
    if (!e || gid >= e->cfg.max_groups || !o) return RAFTING_E_INVAL;
    const ogroup_t* g = &e->groups[gid]; const olog_t* l = &g->log;
    memset(o, 0, sizeof(*o));
    o->alive = (uint32_t)g->alive; o->role = (uint32_t)g->role; o->current_term = g->term;
    o->voted_for = g->ballot; o->current_leader = g->currentLeader; o->incarnation = g->incarnation;
    o->timeout_detected = (uint32_t)g->timeoutDetected; o->leader_prepared = (uint32_t)g->prepared;
    o->votes = g->votes; o->elected_inc = g->electedInc; o->elected_aborted = (uint32_t)g->electedAborted;
    o->elected_term = g->electedTerm;
    o->timer = (g->role == RAFTING_ROLE_LEADER) ? g->hbDue : g->deadline;
    o->commit_index = l->commitIndex; o->epoch_index = l->epochIndex; o->epoch_term = l->epochTerm;
    int64_t li = 0, lt = 0;
    if (log_last(l, &li, &lt)) { o->first_index = l->lo; o->last_index = li; o->last_term = lt; }
    else { o->first_index = 1; o->last_index = 0; o->last_term = 0; }
    o->term_runs = log_runs(l);
    o->err_word = g->errWord;
    /* digest over the run-length form: (start, term) oldest -> newest, then last index */
    uint64_t h = 0xCBF29CE484222325ull;
    if (!log_empty(l)) {
        int64_t start = l->lo, t = l->terms[l->lo - l->base];
        for (int64_t i = l->lo + 1; i <= l->hi; i++) {
            int64_t ti = l->terms[i - l->base];
            if (ti != t) { h = fnv1a(h, (uint64_t)start); h = fnv1a(h, (uint64_t)t); start = i; t = ti; }
        }
        h = fnv1a(h, (uint64_t)start); h = fnv1a(h, (uint64_t)t); h = fnv1a(h, (uint64_t)l->hi);
    }
    o->log_digest = h;
    o->n_followers = e->F;
    if (g->role == RAFTING_ROLE_LEADER && g->prepared) {
        for (uint32_t f = 0; f < e->F; f++) {
            const ostate_t* s = &g->st[f]; rafting_follower_state_t* d = &o->followers[f];
            d->last_request = s->lastRequest; d->request_success = s->requestSuccess; d->request_failure = s->requestFailure;
            d->request_in_flight = s->requestInFlight; d->recent_rejection = s->recentRejection; d->recent_failure = s->recentFailure;
            d->pending_installation = s->pendingInstallation;
            d->last_epoch = s->lastEpoch; d->next_index = s->nextIndex; d->match_index = s->matchIndex;
        }
    }
    return 0;
}
int orc_log_term(orc_engine_t* e, uint32_t gid, int64_t index, int64_t* term) {
    if (!e || gid >= e->cfg.max_groups || !term) return RAFTING_E_INVAL;
    int64_t t;
    *term = log_get(&e->groups[gid].log, index, &t) ? t : -1;
    return 0;
}
