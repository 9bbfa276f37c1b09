/*
 * rafting_b200.h — C ABI of the H100-native batched Multi-Raft hot path.
 *
 * Drop-in boundary for curioloop/rafting's per-context EventLoop path
 * (reference: src/main/java/io/lubricant/consensus/raft/, abbreviated M/ below).
 * The reference has no FFI of its own (100 % Java); every entry point below names the
 * Java surface it replaces.  Plain pointers and sizes only: no torch / C++ types.
 *
 *   Java surface replaced                                   entry point here
 *   ------------------------------------------------------  ---------------------------
 *   ContextManager.start / RaftRoutine ctor                 rafting_engine_create
 *     (M/context/ContextManager.java:46-55, RaftRoutine.java:44-50)
 *   ContextManager.close                                     rafting_engine_destroy
 *   ContextManager.buildContext + RaftContext.initialize    rafting_group_open[_bulk]
 *     (ContextManager.java:57-106, RaftContext.java:91-113)
 *   ContextManager.exitContext / RaftContext.close          rafting_group_close
 *   ContextEventLoop.execute(event[,urgent])                rafting_lease + rafting_step
 *     (M/support/EventLoop.java:41-101) — one step == the event loops of ALL groups
 *     draining one batch, in the canonical serial order described in DESIGN.md §3
 *   RaftParticipant.{appendEntries,preVote,requestVote,     group-op kinds RAFTING_OP_*
 *     installSnapshot,onTimeout} (M/RaftParticipant.java:14-49)
 *   RaftStub.process -> Leader.acceptCommand                RAFTING_OP_SUBMIT
 *     (M/command/RaftStub.java:79-91, Leader.java:128-140)
 *   Async callbacks registered by Leader.replicateLog,      lane-event kinds RAFTING_EV_*
 *     Follower.prepareElection, Candidate.startElection
 *     (Leader.java:174-188,218-237; Follower.java:258-270; Candidate.java:112-134)
 *   RaftService.{appendEntries,installSnapshot,preVote,     outbox plan / ballot records
 *     requestVote} *outbound* calls (M/RaftService.java:22-61)
 *   RaftLog.{epoch,last,lastCommitted,get(i).term()}        rafting_state_export / rafting_log_term
 *     (M/command/RaftLog.java:72-132, storage/RocksLog.java:92-128)
 *   RaftLog.flush (compaction / snapshot epoch move)        RAFTING_OP_FLUSH
 *   (new, north_star) cross-shard commitIndex summary       rafting_commit_slice / rafting_allgather_commit
 *
 * All functions return 0 (RAFTING_OK) or a negative rafting_status_t; they never throw and never
 * call back into the caller.  Per-event protocol errors (the reference's AssertionError /
 * AbstractMethodError / IllegalStateException, which its event loop logs and drops —
 * M/support/EventLoopGroup.java:40-44) are reported per event in the outbox and in the group's
 * sticky error word, never as the call's return value.
 */
#ifndef RAFTING_B200_H
#define RAFTING_B200_H

#include <stdint.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

#define RAFTING_ABI_VERSION 2u

/* ------------------------------------------------------------------------------------------ */
/* status codes (call level)                                                                  */
/* ------------------------------------------------------------------------------------------ */
typedef enum rafting_status {
    RAFTING_OK            =  0,
    RAFTING_E_INVAL       = -1,  /* bad argument (IllegalArgumentException)                    */
    RAFTING_E_NOMEM       = -2,
    RAFTING_E_CUDA        = -3,  /* CUDA runtime failure; rafting_last_error() has the text    */
    RAFTING_E_CLOSED      = -4,  /* engine/group closed (IllegalStateException "log closed")   */
    RAFTING_E_CAPACITY    = -5,  /* max_groups / max_rows / entry pool exceeded                */
    RAFTING_E_NODEVICE    = -6,  /* no CUDA device: the product path has no CPU fallback       */
    RAFTING_E_BUSY        = -7,  /* lease outstanding / step in flight                         */
    RAFTING_E_NCCL        = -8
} rafting_status_t;

/* ------------------------------------------------------------------------------------------ */
/* per-event error codes (outbox + sticky per-group word). One code per throw site.           */
/* ------------------------------------------------------------------------------------------ */
enum {
    RAFTING_EV_OK                    = 0,
    RAFTING_ERR_MATCH_ROLLBACK       = 1,  /* AbstractMethodError, Leadership.java:76-81          */
    RAFTING_ERR_IMPOSSIBLE_REPL      = 2,  /* AssertionError, Leader.java:251-253                  */
    RAFTING_ERR_COMMIT_ROLLBACK      = 3,  /* AssertionError, RocksLog.java:101-103                */
    RAFTING_ERR_TRY_COMMIT_FAILED    = 4,  /* NPE on get(major)==null, caught+logged Leader.java:277 */
    RAFTING_ERR_LEADER_SELF_AE       = 5,  /* Leader.java:71-73                                    */
    RAFTING_ERR_TWO_LEADERS          = 6,  /* Leader.java:79-81                                    */
    RAFTING_ERR_LEADER_VOTE_SELF     = 7,  /* Leader.java:104                                      */
    RAFTING_ERR_FOLLOWER_TWO_LEADERS = 8,  /* Follower.java:48-50                                  */
    RAFTING_ERR_INDEX_TERM_ZERO      = 9,  /* Follower.java:179-181                                */
    RAFTING_ERR_EPOCH_TERM_MISMATCH  = 10, /* Follower.java:184-186                                */
    RAFTING_ERR_IMPOSSIBLE_LOG       = 11, /* Follower.java:199-204                                */
    RAFTING_ERR_CANDIDATE_SELF_RV    = 12, /* Candidate.java:53-55                                 */
    RAFTING_ERR_CANDIDATE_VOTE_SELF  = 13, /* Candidate.java:64-66                                 */
    RAFTING_ERR_IS_BEFORE_AE         = 14, /* RaftMember.java:62-64, Follower.java:138-139         */
    RAFTING_ERR_LEADER_UNCHANGED     = 15, /* Membership.java:89                                   */
    RAFTING_ERR_BALLOT_MISMATCH      = 16, /* Membership.java:103-105                              */
    RAFTING_ERR_LOG_NOT_FOLLOW_EPOCH = 17, /* RocksLog.java:175-177                                */
    RAFTING_ERR_LOG_NOT_CONTINUOUS   = 18, /* RocksLog.java:185-187                                */
    RAFTING_ERR_LOG_START            = 19, /* Leader.java:202-204                                  */
    RAFTING_ERR_LOG_VACANCY          = 20, /* RocksLog.java:161-163                                */
    RAFTING_ERR_FLUSH_RANGE          = 21, /* IndexOutOfBoundsException, RocksLog.java:230-233     */
    RAFTING_ERR_TERM_RUNS_OVERFLOW   = 22, /* engine capacity: > RAFTING_TERM_RUNS term changes    */
    RAFTING_ERR_LOG_SHAPE            = 23, /* degenerate store shape outside the engine's domain   */
    RAFTING_ERR_NOT_LEADER           = 24, /* NotLeaderException, RaftStub.java:88-90              */
    RAFTING_ERR_NOT_READY            = 25, /* NotReadyException, RaftStub.java:83-87               */
    RAFTING_ERR_BAD_EVENT            = 26, /* malformed event (unknown kind / lane)                */
    RAFTING_ERR_CLOSED_GROUP         = 27  /* ObsoleteContextException / !stillRunning             */
};

/* ------------------------------------------------------------------------------------------ */
/* constants mirrored from the reference                                                      */
/* ------------------------------------------------------------------------------------------ */
#define RAFTING_REPLICATE_LIMIT 50   /* Leadership.java:10 */
#define RAFTING_IN_FLIGHT_LIMIT 20   /* Leadership.java:11 */
#define RAFTING_TIMER_TIMEOUT  (-1)  /* TimerTicket.java:13 */
#define RAFTING_TIMER_FENCING  (-2)  /* TimerTicket.java:14 */
#define RAFTING_TIMER_INVALID  (-3)  /* TimerTicket.java:15 */
#define RAFTING_TERM_RUNS        8   /* engine: run-length term table depth per group          */
#define RAFTING_MAX_REPLICAS    33   /* follower lanes per group <= 32 (one warp)              */

enum { RAFTING_ROLE_FOLLOWER = 0, RAFTING_ROLE_CANDIDATE = 1, RAFTING_ROLE_LEADER = 2 };

/* ------------------------------------------------------------------------------------------ */
/* config — mirrors M/support/RaftConfig.java:187-198 + the hard-coded constants              */
/* ------------------------------------------------------------------------------------------ */
typedef struct rafting_cfg {
    uint32_t struct_size;           /* sizeof(rafting_cfg_t), ABI guard                        */
    uint32_t replicas;              /* R = RaftCluster.size(); follower lanes F = R-1          */
    uint32_t local_slot;            /* this node's slot in the sorted node table, 0..R-1       */
    uint32_t max_groups;            /* capacity G                                              */
    uint32_t max_rows;              /* rows per step                                           */
    uint32_t entry_pool_cap;        /* int64 term slots for inbound AE entries, per step       */
    int32_t  pre_vote;              /* RaftConfig.preVote()                                    */
    int32_t  avail_critical_point;  /* metrics/avail-critical-point                            */
    int64_t  recovery_cool_down_ms; /* metrics/recovery-cool-down                              */
    int64_t  heartbeat_ms;          /* RaftConfig.heartbeatInterval()                          */
    int64_t  broadcast_ms;          /* RaftConfig.broadcastTimeout() (informational)           */
    int64_t  election_ms;           /* E = round(election*tick); timeouts are drawn in [E, 2E]  */
    uint64_t timer_seed;            /* seed of the counter-based draw used when an event carries none */
    int32_t  device;                /* CUDA ordinal                                            */
    uint32_t flags;                 /* RAFTING_CFG_* ; 0 = bit-identical to the reference      */
} rafting_cfg_t;
/* Opt-in departures from the reference that close the two flaws DESIGN.md §2 documents.  Specified and tested in the
   oracle (tests/test_cluster_cpu.py); the CUDA engine of this version REJECTS a non-zero cfg.flags (RAFTING_E_INVAL). */
#define RAFTING_CFG_STRICT_CANDIDATE_VOTE   1u   /* a Candidate applies logUpToDate before it votes (Candidate.java:68-71 does not) */
#define RAFTING_CFG_LENIENT_FOLLOWER_COMMIT 2u   /* leaderCommit below the follower's commitIndex is ignored instead of asserted */

/*
 * Election-timeout draws.  The reference draws ThreadLocalRandom.nextInt(E, 2E+1) at every
 * non-muted resetTimer (RaftConfig.java:187-190), which makes its output non-deterministic; for a
 * bit-exact batch semantics the draw is an INPUT.  Group ops carry one draw (op_nr.y, used for every
 * reset inside that op; 0 = use the counter-based draw); role changes triggered by lane events and
 * by timer sweeps use the counter-based draw below, keyed by (seed, gid, incarnation of the new role).
 */
#if defined(__CUDACC__)
#define RAFTING_HD __host__ __device__
#else
#define RAFTING_HD
#endif
RAFTING_HD static inline uint64_t rafting_splitmix64(uint64_t x) {
    x += 0x9E3779B97F4A7C15ull;
    uint64_t z = x;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}
RAFTING_HD static inline int64_t rafting_draw(uint64_t seed, uint32_t gid, uint32_t incarnation, int64_t election_ms) {
    uint64_t h = rafting_splitmix64(seed ^ ((uint64_t)gid * 0xD6E8FEB86659FD93ull) ^ ((uint64_t)incarnation << 32));
    if (election_ms <= 0) return 1;
    return election_ms + (int64_t)(h % (uint64_t)(election_ms + 1));
}

/* ------------------------------------------------------------------------------------------ */
/* batch layout                                                                               */
/*                                                                                            */
/* A step carries `rows` rows over `n` groups (n = n_active, or every open group when         */
/* gids == NULL).  Row r holds, per group, at most ONE group op followed by at most ONE lane  */
/* event per follower lane f = 0..F-1.  Canonical serial order per group (DESIGN.md §3):      */
/*     for r in rows: [timer sweep if row_now[r] != 0]; op(r); ev(r,0); ev(r,1); ... ev(r,F-1) */
/* Follower lane f stands for node slot (f < local_slot ? f : f + 1).                         */
/* ------------------------------------------------------------------------------------------ */
typedef struct rafting_i64x2 { int64_t x, y; } rafting_i64x2_t;

/* group-op kinds (op_meta bits 0..7) */
enum {
    RAFTING_OP_NONE         = 0,
    RAFTING_OP_SUBMIT       = 1,  /* RaftStub.process: isReady -> newEntry x count -> replicateLog(false)
                                     count = bits 16..31 (>=1; count==1 is exactly Leader.acceptCommand;
                                     count>1 is the batched-submit extension, one replicateLog at the end).
                                     a = bitmask of follower lanes whose RaftService is unavailable      */
    RAFTING_OP_TIMEOUT      = 2,  /* timer fired: electionTimeout / keepAlive (RaftRoutine.java:53-77).
                                     a = unavailable-lane mask (used by heartbeat / vote broadcast)      */
    RAFTING_OP_AE_REQUEST   = 3,  /* inbound appendEntries: peer=leader slot, a=term, b=prevLogIndex,
                                     c=prevLogTerm, d=leaderCommit, count=n entries, ent=pool offset;
                                     entries are (prevLogIndex_first + i, ent_terms[ent+i]) with
                                     first index = e (see op_e): contiguous by construction            */
    RAFTING_OP_PREVOTE_REQ  = 4,  /* inbound preVote: peer=candidate, a=term, b=lastLogIndex, c=lastLogTerm */
    RAFTING_OP_VOTE_REQ     = 5,  /* inbound requestVote: same fields                                    */
    RAFTING_OP_IS_REQUEST   = 6,  /* inbound installSnapshot: peer=leader, a=term, b=lastIncludedIndex,
                                     c=lastIncludedTerm, d=host result of RaftContext.installSnapshot   */
    RAFTING_OP_FLUSH        = 7,  /* RaftLog.flush(b=index, c=term) — compaction / snapshot epoch move  */
    RAFTING_OP_KIND_MAX     = 8
};
#define RAFTING_OP_KIND(m)   ((uint32_t)(m) & 0xffu)
#define RAFTING_OP_PEER(m)   (((uint32_t)(m) >> 8) & 0xffu)
#define RAFTING_OP_COUNT(m)  (((uint32_t)(m) >> 16) & 0xffffu)
#define RAFTING_OP_MAKE(kind, peer, count) \
    ((uint32_t)(kind) | ((uint32_t)(peer) << 8) | ((uint32_t)(count) << 16))

/* lane-event kinds (ev_meta bits 0..3) */
enum {
    RAFTING_EV_NONE     = 0,
    RAFTING_EV_AE_ACK   = 1,  /* AE-Echo,  Leader.java:218-237 */
    RAFTING_EV_IS_ACK   = 2,  /* IS-Echo,  Leader.java:174-188 */
    RAFTING_EV_PV_REPLY = 3,  /* PV-Echo,  Follower.java:258-270 */
    RAFTING_EV_RV_REPLY = 4   /* RV-Echo,  Candidate.java:112-134 */
};
/* outcome taxonomy of Async callbacks (M/transport/rpc/Async.java:239-254) */
enum { RAFTING_OUT_OK = 0, RAFTING_OUT_ERROR = 1, RAFTING_OUT_CANCELED = 2 };
/* ev_meta: bits 0..3 kind | 4..5 outcome | 6 success | 32..63 incarnation of the role object that sent the RPC */
#define RAFTING_EVM_MAKE(kind, outcome, success, incarnation) \
    ((uint64_t)(kind) | ((uint64_t)(outcome) << 4) | ((uint64_t)((success) ? 1 : 0) << 6) | \
     ((uint64_t)(uint32_t)(incarnation) << 32))
#define RAFTING_EVM_KIND(m)     ((uint32_t)((m) & 0xfu))
#define RAFTING_EVM_OUTCOME(m)  ((uint32_t)(((m) >> 4) & 0x3u))
#define RAFTING_EVM_SUCCESS(m)  ((uint32_t)(((m) >> 6) & 0x1u))
#define RAFTING_EVM_INC(m)      ((uint32_t)((m) >> 32))

/*
 * Inbox: SoA columns.  Index of group column = r * n + i ; of lane column = (r * n + i) * F + f.
 * Any op_* pointer may be NULL when op_meta is NULL (no group ops in the step); ev_* likewise.
 */
/* inbox flags: NO_REQUESTS promises the step holds no inbound-request ops (AE/PREVOTE/VOTE/IS
   requests, FLUSH); the engine then runs the leaner kernel variant, and any such op found anyway is
   answered with RAFTING_ERR_BAD_EVENT */
#define RAFTING_INBOX_NO_REQUESTS 1u
/* COMPACT_GROUPS (only with an active list): the per-group outbox columns (commit_index ... last_entry)
   are indexed by POSITION in gids[] and hold n_active entries instead of max_groups — a step over a few
   hundred busy groups then moves kilobytes, not the whole per-group snapshot, across PCIe */
#define RAFTING_INBOX_COMPACT_GROUPS 2u

typedef struct rafting_inbox {
    uint32_t rows;                 /* rows in this step (<= cfg.max_rows)                        */
    uint32_t n_active;             /* 0 = dense over gid 0..G-1, else length of gids[]           */
    const uint32_t* gids;          /* optional compacted active list (strictly increasing)       */
    const int64_t*  row_now;       /* [rows] optional: != 0 => SWEEP ROW: the row's group-op slot is the
                                      implied TIMEOUT of every group whose timer is due at that time
                                      (op_* of that row are ignored); its lane events still run     */
    /* group ops */
    const uint64_t*        op_meta; /* lo32 RAFTING_OP_MAKE(...), hi32 entry-pool offset          */
    const rafting_i64x2_t* op_nr;   /* (now_ms, election-timeout draw ms)                         */
    const rafting_i64x2_t* op_ab;   /* (a, b)                                                     */
    const rafting_i64x2_t* op_cd;   /* (c, d)                                                     */
    const int64_t*         op_e;    /* AE request: index of entries[0]                            */
    const int64_t*         ent_terms; /* entry-term pool                                          */
    uint32_t               ent_count;
    uint32_t               flags;   /* RAFTING_INBOX_* promises about the batch content              */
    /* lane events */
    const uint64_t*        ev_meta; /* RAFTING_EVM_MAKE(...)                                      */
    const rafting_i64x2_t* ev_tn;   /* (respTerm, now_ms)                                         */
    const rafting_i64x2_t* ev_el;   /* AE/IS ack: (epochAtSend, lastIndexAtSend); votes: unused   */
} rafting_inbox_t;

/* plan kinds (plan_meta bits 0..3) */
enum { RAFTING_PLAN_NONE = 0, RAFTING_PLAN_AE = 1, RAFTING_PLAN_IS = 2,
       RAFTING_PLAN_SKIP_INFLIGHT = 3, RAFTING_PLAN_UNAVAILABLE = 4 };
/* plan_meta: bits 0..3 kind | 4 heartbeat | 16..31 entry count | 32..63 incarnation */
#define RAFTING_PLM_KIND(m)   ((uint32_t)((m) & 0xfu))
#define RAFTING_PLM_HB(m)     ((uint32_t)(((m) >> 4) & 1u))
#define RAFTING_PLM_COUNT(m)  ((uint32_t)(((m) >> 16) & 0xffffu))
#define RAFTING_PLM_INC(m)    ((uint32_t)((m) >> 32))

/* ballot kinds (ballot_meta bits 0..3) */
enum { RAFTING_BALLOT_NONE = 0, RAFTING_BALLOT_PREVOTE = 1, RAFTING_BALLOT_VOTE = 2 };

/* reply: rep_meta bit 0 valid | bit 1 success | bits 8..15 per-event error code (reply suppressed if != 0) */
#define RAFTING_REP_VALID(m)   ((uint32_t)((m) & 1u))
#define RAFTING_REP_SUCCESS(m) ((uint32_t)(((m) >> 1) & 1u))
#define RAFTING_REP_ERR(m)     ((uint32_t)(((m) >> 8) & 0xffu))

/*
 * Outbox: what the Java pump thread turns back into Netty writes / fsyncs / applies.
 * Row-indexed columns mirror the inbox; group-indexed columns are end-of-step snapshots.
 */
typedef struct rafting_outbox {
    /* per (row, group): reply to an inbound RPC, or op status                                   */
    uint32_t*        rep_meta;
    int64_t*         rep_term;     /* RaftResponse.term()                                        */
    /* per (row, group, lane): outbound AppendEntries / InstallSnapshot (Leader.replicateLog)    */
    uint64_t*        plan_meta;
    rafting_i64x2_t* plan_pp;      /* AE: (prevLogIndex, prevLogTerm); IS: (epoch.index, epoch.term) */
    rafting_i64x2_t* plan_lc;      /* (lastIndex == lastIndexAtSend, leaderCommit)               */
    int64_t*         plan_epoch;   /* epoch.index at send == epochAtSend                          */
    /* per (row, group): outbound PreVote / RequestVote broadcast                                */
    uint64_t*        ballot_meta;  /* bits 0..3 kind | 32..63 incarnation of the asking role object */
    int64_t*         ballot_term;  /* term argument of the RPC                                    */
    rafting_i64x2_t* ballot_last;  /* (lastLogIndex, lastLogTerm)                                 */
    /* per group, end of step: [max_groups] indexed by gid, or [n_active] indexed by position in
       gids[] under RAFTING_INBOX_COMPACT_GROUPS                                                  */
    int64_t*         commit_index; /* RaftLog.lastCommitted()                                     */
    int64_t*         current_term; /* RaftParticipant.currentTerm()                               */
    uint32_t*        role_word;    /* bits 0..1 role | 8..15 votedFor+1 | 16..23 currentLeader+1 |
                                      bit 24 timeoutDetected | bit 25 leader isReady(now of last op) |
                                      bit 30 persist-dirty | bit 31 commit-dirty                  */
    uint32_t*        incarnation;
    uint32_t*        err_word;     /* lo16 last per-event error code, hi16 error count (sticky)   */
    rafting_i64x2_t* last_entry;   /* RaftLog.last(): (index, term); (epoch.index, epoch.term) when the store is empty
                                      — what Follower.prepareElection / Candidate.startElection would send */
} rafting_outbox_t;

/* restored per-group state handed to group_open (StableLock.restore + RaftLog state)            */
typedef struct rafting_group_init {
    int64_t term;          /* Persistence.term                                                   */
    int32_t ballot;        /* Persistence.ballot as node slot, -1 = null                         */
    int32_t _pad;
    int64_t epoch_index, epoch_term;   /* RaftLog.epoch()                                         */
    int64_t first_index;   /* lowest stored key (epoch_index or epoch_index+1), ignored if empty */
    int64_t last_index;    /* RaftLog.last().index, or < first_index for an empty store           */
    int64_t last_term;     /* every restored entry is given this term (single run)                */
    int64_t commit_index;  /* volatile in the reference (RocksLog.java:50): 0 after restart       */
    int64_t now_ms;        /* time of RaftContext.initialize                                      */
    int64_t rand_ms;       /* election-timeout draw for the initial resetTimer                    */
} rafting_group_init_t;

/* full per-group state for parity checks / checkpoint (RaftContext.initialize restores from it) */
typedef struct rafting_follower_state {   /* Leadership.State, Leadership.java:26-38 */
    int64_t last_request, request_success, request_failure;
    int32_t request_in_flight, recent_rejection, recent_failure;
    int32_t pending_installation;
    int64_t last_epoch, next_index, match_index;
} rafting_follower_state_t;

typedef struct rafting_group_state {
    uint32_t alive;
    uint32_t role;
    int64_t  current_term;
    int32_t  voted_for;            /* node slot or -1 */
    int32_t  current_leader;       /* node slot or -1 */
    uint32_t incarnation;
    uint32_t timeout_detected;
    uint32_t leader_prepared;      /* Leader.followerStatus != null */
    int32_t  votes;                /* tally of the live election / pre-vote round */
    uint32_t elected_inc;          /* incarnation of the last elected Candidate (0 = none) */
    uint32_t elected_aborted;
    int64_t  elected_term;
    int64_t  timer;                /* TimerTicket deadline (non-leader) / next heartbeat due (leader) */
    int64_t  commit_index;
    int64_t  epoch_index, epoch_term;
    int64_t  first_index, last_index;   /* stored key range; empty when last_index < first_index */
    int64_t  last_term;
    uint32_t term_runs;            /* number of term runs in the stored range */
    uint32_t err_word;
    uint64_t log_digest;           /* FNV-1a over (index, term) of every stored entry */
    uint32_t n_followers;
    uint32_t _pad;
    rafting_follower_state_t followers[RAFTING_MAX_REPLICAS - 1];
} rafting_group_state_t;

typedef struct rafting_engine rafting_engine_t;

/* lease: pinned host staging columns sized for (rows x n groups); valid until the matching step */
typedef struct rafting_lease {
    rafting_inbox_t  in;    /* const-cast to fill; pointers are into pinned host memory */
    rafting_outbox_t out;   /* filled by rafting_step */
    uint32_t generation;    /* set by rafting_lease: a stale copy of an ended lease is rejected, even if a later lease
                               was carved at the same addresses */
    uint32_t _pad;
} rafting_lease_t;

/* ------------------------------------------------------------------------------------------ */
/* entry points                                                                               */
/* ------------------------------------------------------------------------------------------ */
uint32_t    rafting_abi_version(void);
const char* rafting_last_error(void);                         /* thread-local text of the last failure */

int rafting_engine_create (const rafting_cfg_t* cfg, rafting_engine_t** out);
int rafting_engine_destroy(rafting_engine_t* e);

/* open group(s): gid is caller-chosen (dense 0..max_groups-1) so shards keep group order */
int rafting_group_open     (rafting_engine_t* e, uint32_t gid, const rafting_group_init_t* init);
int rafting_group_open_bulk(rafting_engine_t* e, uint32_t first_gid, uint32_t count,
                            const rafting_group_init_t* inits /* [count] */);
int rafting_group_close    (rafting_engine_t* e, uint32_t gid);
/* group_open / group_open_bulk / group_close / group_load_runs edit the tables from the host: they drain the engine's step
   stream first and return RAFTING_E_BUSY while a host-path step (step_begin / step_begin_host) has not been waited for.
   Steps enqueued on a CALLER's stream through rafting_step_device must be synchronised by the caller. */
/* Restart with a log that spans several terms (RaftContext.initialize over an existing RocksLog, RaftContext.java:91-113):
 * after rafting_group_open, hand over the stored log's index->term map as runs, oldest first — runs[k] = (first index of
 * the run, its term); runs[0].x must be the group's first stored index, the last run's term its last_term.  At most
 * RAFTING_TERM_RUNS runs (RAFTING_E_CAPACITY beyond: compact the log first). */
int rafting_group_load_runs(rafting_engine_t* e, uint32_t gid, const rafting_i64x2_t* runs, uint32_t n_runs);

/* Open, restart and close groups in step-stream order, while steps are in flight (ContextManager.buildContext / exitContext
 * issued by a pipelined pump between two step begins).
 *   Ordering: the edits are enqueued on the engine's step stream.  Every step, due query and edit begun before the call sees
 *     the tables without them, everything begun after it sees them.  Host, compact, active, sweep and due steps may be in
 *     flight: the call never returns RAFTING_E_BUSY for that and never synchronises the step stream.  Steps enqueued on a
 *     CALLER's stream through rafting_step_device must be ordered by the caller, as for rafting_group_open.
 *   Effect: at its place in the stream an OPEN leaves the gid exactly as rafting_group_open(init), followed by
 *     rafting_group_load_runs(runs, n_runs) when n_runs > 0, would after a drain; an OPEN of an alive gid replaces it (a
 *     restart).  A CLOSE leaves the gid as rafting_group_close would; a CLOSE of a closed gid changes nothing but the tags.
 *   Tags: both kinds free every tag of the gid's F lanes in the compact path's in-flight table, if that table exists.
 *   Pump contract: incarnations restart at 1 (RaftMember.java:20-26), so the engine cannot tell a reply to the old life from
 *     one to the new.  After an edit of gid g the caller must not put a reply to an RPC planned before the edit into any later
 *     step, dense or compact: it drops those RPCs from its pending table, as the reference drops the callbacks of a closed
 *     context.
 *   Validation: every record is checked on the host before anything is enqueued (RAFTING_E_INVAL / RAFTING_E_CAPACITY, with
 *     nothing enqueued): gid < max_groups and gids strictly increasing within the call, a known kind, every check
 *     group_open_bulk makes on init, and for n_runs > 0 every check load_runs makes, against the record's own init.
 *     n == 0 is a no-op.
 *   Buffers: `edits` may be reused as soon as the call returns.  The records travel from pinned staging of the engine's own,
 *     reused under an event: the call blocks only to reuse a staging buffer whose edit has not yet run, or to grow one. */
enum { RAFTING_EDIT_OPEN = 1, RAFTING_EDIT_CLOSE = 2 };
typedef struct rafting_group_edit {
    uint32_t gid, kind;
    rafting_group_init_t init;                 /* OPEN: exactly what rafting_group_open takes; CLOSE: ignored */
    uint32_t n_runs, _pad;                     /* OPEN: 0 = the single run init describes (rafting_group_open);
                                                  1..RAFTING_TERM_RUNS = runs[] as rafting_group_load_runs takes them */
    rafting_i64x2_t runs[RAFTING_TERM_RUNS];   /* (first index, term), oldest first */
} rafting_group_edit_t;
int rafting_group_edit_begin(rafting_engine_t* e, uint32_t n, const rafting_group_edit_t* edits /* host */);

/* host path: fill lease->in (pinned), call step; H2D + kernels + D2H happen inside the call */
int rafting_lease(rafting_engine_t* e, uint32_t rows, uint32_t n_active, uint32_t ent_count,
                  rafting_lease_t* out);
/* same, with the inbox flags the step will carry: RAFTING_INBOX_COMPACT_GROUPS sizes the per-group outbox
   columns for n_active entries.  Every column of a lease lives in one pinned block per direction, so a leased
   step is one copy up (two with an active list) and one copy down */
int rafting_lease_ex(rafting_engine_t* e, uint32_t rows, uint32_t n_active, uint32_t ent_count, uint32_t flags,
                     rafting_lease_t* out);
int rafting_step (rafting_engine_t* e, rafting_lease_t* lease);          /* synchronous         */
int rafting_step_begin(rafting_engine_t* e, rafting_lease_t* lease);     /* async: enqueue      */
int rafting_step_wait (rafting_engine_t* e, rafting_lease_t* lease);     /* async: outbox ready; ends the lease (on error the lease stays) */
int rafting_lease_release(rafting_engine_t* e, rafting_lease_t* lease);  /* give back a lease that will not be stepped */
/* Up to RAFTING_HOST_SLOTS (4) leases may be outstanding: begin(A); fill B; begin(B); wait(A); ... overlaps
   the H2D of one step, the kernel of another and the D2H of a third.
   Caller-owned buffers (e.g. the transport's pinned receive pool, north_star "Netty feeds pinned
   staging buffers"): same pipeline, host pointers supplied by the caller; pin them for real overlap. */
int rafting_step_begin_host(rafting_engine_t* e, uint32_t slot /* 0..3 */, const rafting_inbox_t* in_host,
                            const rafting_outbox_t* out_host);
int rafting_step_wait_slot (rafting_engine_t* e, uint32_t slot);

/* ---------------------------------------------------------------------------------------------------------------------
 * COMPACT host path (round 2): the same step, an eighth of the PCIe bytes.
 *
 * The dense host path moves 65 B up and 69 B down per AppendEntries ack and is PCIe-bound.  Most of those bytes are
 * redundant in leader steady state: every time of a row lies within 65 s of the row's base time; a reply's term is the
 * term its request was sent with; (epochAtSend, lastIndexAtSend) — which the reference keeps in the callback closure of
 * Leader.replicateLog (Leader.java:216-237) — only travel down to be sent up again; a plan's prevLogIndex / leaderCommit
 * lie close to the group's end-of-step snapshot.  The compact format drops them LOSSLESSLY: whatever does not fit its rules
 * travels in full through an escape list, and two device kernels (unpack before, pack after the step kernel) convert
 * between the compact wire columns and the dense SoA batch the step kernel works on.
 *   * the (epochAtSend, lastIndexAtSend) echo stays in an HBM in-flight table: pack gives every AE / IS plan a TAG (a free
 *     slot 0..31 of its (group, follower) lane), the reply echoes the tag, unpack looks the pair up and frees the slot.
 *     No free slot (more than 32 RPCs of one lane outstanding): tag 255, and the reply must come back as an escape record.
 *   * whole-shard steps (every column sized by max_groups), or steps over an active list through
 *     rafting_step_begin_compact_active (every column sized by n_active, below).  op_c carries SUBMIT / TIMEOUT ops, ev_c
 *     AE / IS acks; vote replies and anything irregular use the escape lists (vote replies, ballots and vote requests travel
 *     compact under RAFTING_COMPACT_ELECTIONS, below).  Inbound requests ride beside the inbox in a request list (rafting_creqs_t, below):
 *     AppendEntries as 32-byte records, every other request kind as an op escape.  A step without requests runs as
 *     RAFTING_INBOX_NO_REQUESTS.
 *   * wire words are 32 bits: 4 B per lane slot + 4 B per group row up, 4 B per lane slot + 1 B per group row down.
 *   * a tag is freed by the compact reply that echoes it (every RPC completes exactly once: reply, error or cancellation,
 *     Async.java:239-254).  Dense and compact steps can be mixed slot by slot, but the reply to a compact-planned RPC should come
 *     back through the compact path; if it comes back dense (or never), its tag stays taken and, once a lane has none left,
 *     that lane's plans are simply untagged (their replies travel as escape records): slower, never wrong.
 * ------------------------------------------------------------------------------------------------------------------- */
/* ev_c (32 bits per lane slot):
 *        bits 0..3 kind (RAFTING_EV_NONE / _AE_ACK / _IS_ACK, or 15 = "see the escape list") | 4..5 outcome | 6 success |
 *        7 term-as-sent (RaftResponse.term() == the term the request carried; required for outcome OK, else escape) |
 *        8..15 tag echoed from plan_c | 16..31 now - row_base[row] (ms, unsigned)
 *        The incarnation of the role object that sent the RPC is NOT on the wire: it waits in the in-flight table with the echo
 *        pair and comes back under the tag (a reply without a tag must be escaped).
 * op_c (32 bits per group row):
 *        bits 0..3 kind (NONE / SUBMIT / TIMEOUT) | 4..15 count (1..4095 commands of a SUBMIT) | 16..31 now - row_base[row];
 *        unavailable-follower masks travel in their own optional column op_unavail (16 bits per group row)                  */
#define RAFTING_CEV_ESCAPED 15u
#define RAFTING_CEV_MAKE(kind, outcome, success, term_as_sent, tag, dt)                                                \
    ((uint32_t)(kind) | ((uint32_t)(outcome) << 4) | ((uint32_t)((success) ? 1 : 0) << 6) |                            \
     ((uint32_t)((term_as_sent) ? 1 : 0) << 7) | ((uint32_t)((tag) & 0xffu) << 8) | ((uint32_t)((dt) & 0xffffu) << 16))
#define RAFTING_COP_MAKE(kind, count, dt) ((uint32_t)(kind) | ((uint32_t)((count) & 0xfffu) << 4) | ((uint32_t)((dt) & 0xffffu) << 16))
#define RAFTING_CTAG_NONE 63u    /* in ev_c (8-bit field) any value >= 32 means "no tag" */
typedef struct rafting_cesc_in {     /* a lane event in full: overwrites slot (row * G + gid) * F + lane after unpacking */
    uint32_t slot, _pad;
    uint64_t ev_meta;                /* RAFTING_EVM_MAKE(...) */
    int64_t  term, now_ms, epoch_at_send, last_at_send;
} rafting_cesc_in_t;
typedef struct rafting_cinbox {
    uint32_t rows, n_esc;
    const int64_t*           row_base;   /* [rows] */
    const uint32_t*          op_c;       /* [rows][G], may be NULL (no group ops) */
    const uint16_t*          op_unavail; /* [rows][G] unavailable-follower lanes 0..15 of the op, may be NULL (nobody unavailable) */
    const uint32_t*          ev_c;       /* [rows][G][F], may be NULL (no lane events) */
    const rafting_cesc_in_t* esc;        /* [n_esc] */
} rafting_cinbox_t;
/* plan_c (ONE 32-bit word per lane slot): bits 0..2 kind | 3 heartbeat | 4 escaped | 5..10 tag (0..31, 63 = none) |
 *          11..16 entry count (0..50, Leadership.REPLICATE_LIMIT) | 17..24 dprev | 25..31 dcommit.  Not escaped means:
 *          the plan's incarnation == incarnation[g] (end of step), and
 *          AE  prevLogIndex = last_entry[g].x - dprev, prevLogTerm = current_term[g], lastIndex = prevLogIndex + count,
 *              leaderCommit = commit_index[g] - dcommit, epochAtSend = epoch[g].x          (dprev < 256, dcommit < 128)
 *          IS  (epoch.index, epoch.term) = epoch[g], leaderCommit as above
 *          SKIP_INFLIGHT / UNAVAILABLE: no payload
 * rep_c  : bits 0..5 per-event error code of the row's group op (rafting_outbox_t.rep_meta bits 8..15) | 6 success |
 *          7 compact reply: a valid reply whose RaftResponse.term() equals current_term[g] at the end of the step.
 *          Bits 6 and 7 are set only by steps begun with a request list (rafting_step_begin_compact_req with reqs != NULL);
 *          every other valid reply travels as a RAFTING_CESC_REPLY escape record                                         */
#define RAFTING_CPLAN_KIND(w)    ((uint32_t)(w) & 7u)
#define RAFTING_CPLAN_HB(w)      (((uint32_t)(w) >> 3) & 1u)
#define RAFTING_CPLAN_ESCAPED(w) (((uint32_t)(w) >> 4) & 1u)
#define RAFTING_CPLAN_TAG(w)     (((uint32_t)(w) >> 5) & 63u)
#define RAFTING_CPLAN_COUNT(w)   (((uint32_t)(w) >> 11) & 63u)
#define RAFTING_CPLAN_DPREV(w)   (((uint32_t)(w) >> 17) & 255u)
#define RAFTING_CPLAN_DCOMMIT(w) (((uint32_t)(w) >> 25) & 127u)
enum { RAFTING_CESC_PLAN = 1, RAFTING_CESC_BALLOT = 2, RAFTING_CESC_REPLY = 3 };
typedef struct rafting_cesc_out {
    uint32_t kind, slot;             /* PLAN: lane slot; BALLOT / REPLY: row * G + gid */
    uint64_t meta;                   /* plan_meta | tag << 8 (the full 64-bit plan word, incarnation included; tag 255 = none) / ballot_meta / rep_meta */
    int64_t  a, b, c, d, e;          /* PLAN: plan_pp.x, .y, plan_lc.x, .y, plan_epoch; BALLOT: term, last.x, last.y; REPLY: rep_term */
} rafting_cesc_out_t;
typedef struct rafting_coutbox {
    uint32_t* plan_c;                /* [rows][G][F] */
    uint8_t*  rep_c;                 /* [rows][G]    */
    int64_t*  commit_index; int64_t* current_term; uint32_t* role_word; uint32_t* incarnation; uint32_t* err_word;
    rafting_i64x2_t* last_entry;     /* [G] each, as in rafting_outbox_t */
    rafting_i64x2_t* epoch;          /* [G] RaftLog.epoch() at the end of the step */
    rafting_cesc_out_t* esc;         /* [esc_cap] */
    uint32_t  esc_cap, _pad;
    uint32_t* counts;                /* [4] escape records produced (may exceed esc_cap: then use rafting_step_fetch_dense),
                                        ballots, valid replies, and for rafting_step_begin_compact_due the number of due groups
                                        outside the host's list (0 for every other step) */
} rafting_coutbox_t;
/* Byte offsets of the wire columns inside ONE block per direction, as the engine lays them out on the device.  A caller that
   carves its pinned inbox / outbox out of one block with these offsets gets ONE copy up and ONE copy down per launch instead
   of one per column (the engine recognises the arrangement from the pointers; any other arrangement works column by column).
     in_off : row_base, op_c, op_unavail, ev_c, esc, total
     out_off: plan_c, rep_c, commit_index, current_term, role_word, incarnation, err_word, last_entry, epoch, counts, esc, total */
int rafting_compact_layout(uint32_t rows, uint32_t max_groups, uint32_t followers, uint32_t n_esc_in, uint32_t esc_cap,
                           uint64_t in_off[6], uint64_t out_off[12]);
int rafting_step_begin_compact(rafting_engine_t* e, uint32_t slot /* 0..3 */, const rafting_cinbox_t* in_host,
                               const rafting_coutbox_t* out_host);
/* Inbound requests of a compact step.  Every slot (row * G + gid) takes at most ONE group op: a non-NONE op_c word, a
 * record or an op escape.
 * rafting_creq_t: one inbound AppendEntries in 32 bytes.  It fits when
 *          the election-timeout draw is 0, op_e == prevLogIndex + 1, every entry term equals the request's term,
 *          0 <= term - prevLogTerm < 2^32, leaderCommit - prevLogIndex fits an int32, 0 <= now - row_base[row] <= 65535,
 *          count <= 63 and the peer slot < 32.
 *        meta bits 0..4 peer slot | 5..10 entry count | 11..15 zero (else malformed) | 16..31 now - row_base[row] (ms, unsigned)
 *        The step sees: kind AE, a = term, b = prev_index, c = term - d_prev_term, d = prev_index + d_commit,
 *        e = prev_index + 1, and `count` entries of term `term`, which the engine writes into the entry pool itself.
 *        Every field is relative to the request itself or to row_base, never to engine state: a pump encodes a step while
 *        earlier ones are still in flight.
 * rafting_cesc_op_t: any other request (PreVote / RequestVote / InstallSnapshot / FLUSH, an AppendEntries that breaks a
 *        rule above) or a SUBMIT / TIMEOUT with an explicit draw, in full.  Its entry terms sit at ent_terms[ent ...].
 * Both lists are strictly increasing in slot; slots >= rows * G are ignored.  A slot claimed twice (an op_c word and a
 * record or op escape, a record and an op escape, the same slot twice in one list) is answered with RAFTING_ERR_BAD_EVENT:
 * unpack gives it the op kind RAFTING_COP_MALFORMED with now = row_base[row] and every other field 0.  A list that
 * decreases anywhere makes every op of both lists malformed.
 * Entry pool of the step: ent_terms[0 .. ent_count) then the records' terms in list order, req_entries in all;
 * ent_count + req_entries > cfg.entry_pool_cap is RAFTING_E_CAPACITY.  A record whose entries would end past the pool gets
 * an entry offset past it, so the step answers it with RAFTING_ERR_BAD_EVENT.                                          */
#define RAFTING_CREQ_MAKE(peer, count, dt) \
    ((uint32_t)((peer) & 0x1fu) | ((uint32_t)((count) & 0x3fu) << 5) | ((uint32_t)((dt) & 0xffffu) << 16))
#define RAFTING_CREQ_PEER(m)  ((uint32_t)(m) & 0x1fu)
#define RAFTING_CREQ_COUNT(m) (((uint32_t)(m) >> 5) & 0x3fu)
#define RAFTING_CREQ_DT(m)    ((uint32_t)(m) >> 16)
#define RAFTING_COP_MALFORMED 0xffu
typedef struct rafting_creq {
    uint32_t slot;                   /* row * G + gid */
    uint32_t meta;                   /* RAFTING_CREQ_MAKE(peer, count, now - row_base[row]) */
    int64_t  term;                   /* the RPC's term; every entry of the request carries it */
    int64_t  prev_index;             /* prevLogIndex */
    uint32_t d_prev_term;            /* term - prevLogTerm */
    int32_t  d_commit;               /* leaderCommit - prevLogIndex */
} rafting_creq_t;
typedef struct rafting_cesc_op {
    uint32_t slot, ent;              /* row * G + gid; offset of its entry terms in ent_terms */
    uint64_t op_meta;                /* lo32 RAFTING_OP_MAKE(kind, peer, count); hi32 ignored */
    int64_t  now_ms, draw, a, b, c, d, e;
} rafting_cesc_op_t;
typedef struct rafting_creqs {
    uint32_t n_req, n_op_esc;
    const rafting_creq_t*    req;       /* [n_req] */
    const rafting_cesc_op_t* op_esc;    /* [n_op_esc] */
    const int64_t*           ent_terms; /* [ent_count] entry terms of the escaped AppendEntries */
    uint32_t ent_count;
    uint32_t req_entries;               /* sum of the records' counts */
} rafting_creqs_t;
/* Byte offsets of req, op_esc and ent_terms inside ONE pinned block, and its size: carved this way the request list goes
   up in one copy (none when both lists are empty).  off: req, op_esc, ent_terms, total */
int rafting_compact_req_layout(uint32_t n_req, uint32_t n_op_esc, uint32_t ent_count, uint64_t off[4]);
/* rafting_step_begin_compact with a request list.  reqs == NULL is exactly rafting_step_begin_compact; with a list (even
   an empty one) rep_c carries compact replies.  rafting_step_wait_compact / rafting_step_fetch_dense serve both. */
int rafting_step_begin_compact_req(rafting_engine_t* e, uint32_t slot /* 0..3 */, const rafting_cinbox_t* in_host,
                                   const rafting_creqs_t* reqs, const rafting_coutbox_t* out_host);
/* ELECTIONS on the compact path (flag RAFTING_COMPACT_ELECTIONS of rafting_step_begin_compact_ex; flags == 0 is exactly
 * rafting_step_begin_compact_req).  Election traffic comes in storms (a node restarts, a partition heals, every group that
 * had its leader there elects at once); under the flag a ballot, its replies and inbound vote requests travel compact too.
 *   * ballot (down): a PreVote / RequestVote broadcast of (row, group) becomes one plan_c word per lane of the group, kind
 *     RAFTING_CPLAN_PREVOTE (5) / RAFTING_CPLAN_VOTE (6), a tag in bits 5..10 (63 = none), no payload.  It stands for
 *          ballot_meta = BALLOT_PREVOTE / BALLOT_VOTE | incarnation[g] << 32, ballot_term = current_term[g] + 1 (PreVote) /
 *          current_term[g] (RequestVote), ballot_last = last_entry[g]      (end-of-step columns, as for plans)
 *     and is used only when exactly that holds and no lane of the (row, group) also holds a plan; every other ballot stays a
 *     RAFTING_CESC_BALLOT escape record and takes no tag.  counts[1] counts both.  Each lane's word takes the lowest free tag
 *     of its lane and parks (ballot term, 0) and the incarnation under it: a vote RPC completes exactly once, like an AE / IS.
 *   * vote reply (up), an ev_c word of kind RAFTING_EV_PV_REPLY / RAFTING_EV_RV_REPLY:
 *        bits 0..3 kind | 4..5 outcome | 6 granted | 7 reserved (0) | 8..12 tag (0..31) | 13..15 c | 16..31 now - row_base[row]
 *        Bit 7 is reserved: a writer sets it to 0, and unpack ignores it (it does not reach ev_meta; unlike an ack word, a vote
 *        word has no term-as-sent bit, the term comes from c).
 *        The step sees: the incarnation and ballot term parked under the tag (the tag is freed), respTerm = ballotTerm - c for
 *        outcome OK and 0 otherwise (c must then be 0), ev_el = (0, 0).  A reply with no tag, respTerm > ballotTerm,
 *        ballotTerm - respTerm > 7, a non-zero respTerm without outcome OK, or a time out of range is an escape record.
 *   * escaped word: RAFTING_CEV_ESCAPED | tag << 8 carries the tag of the RPC the escaped event answers (any value >= 32 = none);
 *     unpack frees it, so escaped replies (AE / IS acks included) do not leak tags.  Unflagged steps ignore bits 8..31.
 *   * vote record (rafting_creq_t, request list): meta bits 11..12 = 1 PreVote / 2 RequestVote (RAFTING_CREQ_VOTE_*),
 *        prev_index = lastLogIndex, d_prev_term = term - lastLogTerm, entry count 0, d_commit 0.  The step sees kind
 *        PREVOTE_REQ / VOTE_REQ, a = term, b = prev_index, c = term - d_prev_term, d = e = 0, entry offset 0.  A vote record
 *        with a non-zero count or d_commit, or bits 11..12 == 3, is malformed, like a record with bits 13..15 set.  Without
 *        the flag any non-zero bit 11..15 stays malformed.
 *   Replies to inbound vote requests need nothing new: rep_c bit 7 already covers a valid reply with the end-of-step term. */
#define RAFTING_COMPACT_ELECTIONS 1u
#define RAFTING_CPLAN_PREVOTE 5u
#define RAFTING_CPLAN_VOTE    6u
#define RAFTING_CEV_VOTE_MAKE(kind, outcome, granted, tag, c, dt)                                                      \
    ((uint32_t)(kind) | ((uint32_t)(outcome) << 4) | ((uint32_t)((granted) ? 1 : 0) << 6) | ((uint32_t)((tag) & 0x1fu) << 8) | \
     ((uint32_t)((c) & 7u) << 13) | ((uint32_t)((dt) & 0xffffu) << 16))
#define RAFTING_CEV_VOTE_TAG(w)  (((uint32_t)(w) >> 8) & 0x1fu)
#define RAFTING_CEV_VOTE_C(w)    (((uint32_t)(w) >> 13) & 7u)
#define RAFTING_CREQ_VOTE_PRE 1u
#define RAFTING_CREQ_VOTE_RV  2u
#define RAFTING_CREQ_VOTE(m)  (((uint32_t)(m) >> 11) & 3u)
/* PREV_TERM on the compact path (flag RAFTING_COMPACT_PREV_TERM of rafting_step_begin_compact_ex; it combines freely with
 * RAFTING_COMPACT_ELECTIONS, so flags is 0, 1, 4 or 5, and every other bit is refused).  The first heartbeats of a newly
 * elected leader, and AppendEntries that follow an older term or catch a follower up after a rejection, carry a prevLogTerm
 * below the group's term: under kind 1 each is a RAFTING_CESC_PLAN record.  Under the flag such a plan is one plan_c word:
 *        bits 0..2 RAFTING_CPLAN_AE_PREV_TERM (7) | 3 heartbeat | 4 zero (an escaped AE keeps kind 1) | 5..10 tag (as kind 1) |
 *        11..16 count | 17..24 dprev | 25..27 dterm - 1 | 28..31 dcommit
 *     prevLogIndex = last_entry[g].x - dprev      prevLogTerm  = current_term[g] - dterm      (dterm 1..8)
 *     lastIndex    = prevLogIndex + count         leaderCommit = commit_index[g] - dcommit    (dcommit 0..15)
 *     epochAtSend  = epoch[g].x                   incarnation  = incarnation[g]               (end-of-step columns, as kind 1)
 *   It is used only when every other kind-1 condition holds (incarnation, epochAtSend, lastIndex == prevLogIndex + count,
 *   count < 64, dprev < 256), 1 <= current_term[g] - prevLogTerm <= 8 and dcommit < 16.  A plan that fits kind 1 stays kind
 *   1; any other plan stays a RAFTING_CESC_PLAN record.  The plan takes its tag and parks (epochAtSend, lastIndex) and the
 *   incarnation exactly as kind 1 does, so its ack or failure is an ordinary AE ev_c word: nothing else of the step changes. */
#define RAFTING_COMPACT_PREV_TERM 4u
#define RAFTING_CPLAN_AE_PREV_TERM 7u
#define RAFTING_CPLAN_DTERM(w)    ((((uint32_t)(w) >> 25) & 7u) + 1u)    /* current_term[g] - prevLogTerm, 1..8 */
#define RAFTING_CPLAN_DCOMMIT7(w) (((uint32_t)(w) >> 28) & 15u)           /* the dcommit of a kind-7 word */
int rafting_step_begin_compact_ex(rafting_engine_t* e, uint32_t slot /* 0..3 */, const rafting_cinbox_t* in_host,
                                  const rafting_creqs_t* reqs, const rafting_coutbox_t* out_host, uint32_t flags);
/* ACTIVE LISTS on the compact path.  A node hosts 64 K - 1 M groups and most of them are idle in any one tick; a step over
 * the n_active busy groups gids[0 .. n_active) moves columns of n_active entries instead of max_groups.  flags and reqs mean
 * what they mean for rafting_step_begin_compact_ex (flags 0, 1, 4 or 5; reqs == NULL: no request list).
 *   * position i stands for gids[i].  Every wire column is sized by n = n_active in place of max_groups: op_c and op_unavail
 *     [rows][n], ev_c and plan_c [rows][n][F], rep_c [rows][n], and the group columns commit_index ... epoch [n] by position
 *     (the RAFTING_INBOX_COMPACT_GROUPS shape).  Every slot is positional too: row * n + i in the request list and in
 *     ballot / reply escape records, (row * n + i) * F + f in lane escape records, both ways.  rafting_compact_layout(rows,
 *     n_active, F, ...) and rafting_compact_req_layout give the block offsets.  gids travels in a copy of its own (pin it,
 *     and keep it until the wait, for overlap).
 *   * gids must be strictly increasing, every id < max_groups, 1 <= n_active <= max_groups; anything else is refused
 *     (RAFTING_E_INVAL, RAFTING_E_CAPACITY for n_active > max_groups) before anything is enqueued, and the slot stays free.
 *   * the in-flight table stays indexed by gid: a plan packed at position i of one step is found by its ack at whatever
 *     position its gid holds in a later step's list, or in a whole-shard step.  Active and whole-shard compact steps, dense
 *     steps and leased steps mix slot by slot.  Groups not in the list are untouched.
 *   * rafting_step_wait_compact serves the step; after it, rafting_step_fetch_dense returns the dense outbox in the
 *     COMPACT_GROUPS shape: row columns [rows][n], group columns [n] by position. */
int rafting_step_begin_compact_active(rafting_engine_t* e, uint32_t slot /* 0..3 */, uint32_t n_active, const uint32_t* gids /* host */,
                                      const rafting_cinbox_t* in_host, const rafting_creqs_t* reqs, const rafting_coutbox_t* out_host,
                                      uint32_t flags);
/* TIMERS on the compact path.  Raft's timers (RaftRoutine's TimerTicket: a follower's / candidate's election timeout, a leader's
 * keepAlive, RaftRoutine.java:53-130) fire on a SWEEP ROW: row r of a step with row_now[r] = t != 0 gives every group of the
 * step whose timer is due at t the implied RAFTING_OP_TIMEOUT in that row's op slot, where due means
 *        alive && (leader ? timer <= t : timer > 0 && timer != INT64_MAX && timer <= t)
 * The deadlines live in HBM and move inside steps (resetTimer on AppendEntries, votes and role changes, counter-based draws,
 * muted timers), so a pump does not track them; it asks the engine which groups are due and lists those.
 *
 * rafting_step_begin_compact_sweep: the compact step (whole shard when gids == NULL, else over the active list gids[0 .. n_active),
 *   checked as rafting_step_begin_compact_active checks it) that stands for the dense step with row_now = sweep (host, [rows];
 *   0 = not a sweep row; NULL = no sweep row).  Its wire columns, flags (0, 1, 4 or 5), request list and outbox mean what they mean
 *   for rafting_step_begin_compact_ex / _active; rafting_step_wait_compact and rafting_step_fetch_dense serve it.
 *   * a sweep row's op slot belongs to the sweep: its op_c words are ignored, as the dense step ignores op_meta there, and a
 *     request record or op escape whose slot lies on a sweep row is refused (RAFTING_E_INVAL, nothing enqueued, slot free).
 *   * a step that holds only a sweep (no op_c, no ev_c, no request) is legal: its heartbeats, ballots and replies come back in
 *     plan_c / rep_c and the escape list like those of any op.
 *   * the sweep column travels up in the same copy as the active list (alone for a whole-shard step).
 *
 * rafting_timers_due_begin / _wait: the gids a sweep row at t = until_ms would fire, over the whole shard, as of every step begun
 *   before the query (it is enqueued on the engine's step stream, behind them; begin does not synchronise).
 *   * gids_out receives the due gids in strictly increasing order.  n_due is the full count: when n_due > cap only the first cap
 *     gids are written (the lowest ones) — never silently, the count says so; query again with a larger buffer, or list the
 *     first cap now and the rest after the next query.  cap == 0 asks for the count and the next deadline only.
 *   * gids_out should be pinned (cudaHostAlloc / registered): the device then writes it directly.  Any other host memory works
 *     through a pinned staging block of the query slot, copied into gids_out at the wait.  It must stay valid until the wait.
 *   * next_deadline_ms: the earliest deadline after until_ms that a later sweep would fire (the least timer > until_ms of an
 *     alive leader, or of an alive follower / candidate whose timer is armed: > 0 and != INT64_MAX); INT64_MAX if there is none.
 *     An idle pump sleeps until then.
 *   * query slots 0..RAFTING_HOST_SLOTS-1 are independent of the step slots; each holds one query until its wait
 *     (RAFTING_E_BUSY otherwise).  The table is the engine's, so the query serves whole-shard and active, dense and compact steps.
 *
 * PIPELINING RULE.  A pump encodes step k+1 while steps k-d+1 .. k (d >= 0) are in flight, its sweep times never decrease.  With
 * Q = the due list of a query begun after step k-d, at until = the last sweep time of step k+1, the list
 *        Q  u  event gids of steps k-d+1 .. k+1        (event gid: a group op outside the sweep rows, or a lane event)
 * holds every group that a whole-shard sweep would fire in step k+1, and listing exactly those groups leaves the shard as the
 * whole-shard step would.  For a group g outside it:
 *   * g has no event in steps k-d+1 .. k+1, and Q says it is not due at until; the predicate is monotone in t, so it was not due
 *     at any earlier sweep time of those steps either;
 *   * a group without events whose timer is not due is left untouched by a step (listed or not, a sweep row passes it by), so
 *     step by step g keeps the state Q was computed from, and is not due at step k+1.
 * Listing more is always safe: a listed group that is not due is left untouched by a sweep row.  So the lists of the steps in
 * flight may be added as well, but they need not be, and should not: each list would then contain the one before it.
 * (A whole-shard in-flight step counts as an event of every group.) */
int rafting_step_begin_compact_sweep(rafting_engine_t* e, uint32_t slot /* 0..3 */, uint32_t n_active, const uint32_t* gids /* NULL = whole shard */,
                                     const int64_t* sweep /* [rows], host; 0 = not a sweep row */,
                                     const rafting_cinbox_t* in_host, const rafting_creqs_t* reqs, const rafting_coutbox_t* out_host,
                                     uint32_t flags);
int rafting_timers_due_begin(rafting_engine_t* e, uint32_t slot /* 0..3 */, int64_t until_ms, uint32_t* gids_out /* host [cap] */, uint32_t cap);
int rafting_timers_due_wait (rafting_engine_t* e, uint32_t slot, uint32_t* n_due, int64_t* next_deadline_ms);
/* DUE STEPS: the step finds its own due groups, so a pump lists only the groups it has events for, at any depth of pipelining.
 * rafting_step_begin_compact_due is a sweep step over a list of n = n_host + cap positions:
 *   * positions 0 .. n_host-1 are gids, checked as an active list is (strictly increasing, each < max_groups), except that
 *     n_host = 0 is allowed (a pure timer tick);
 *   * positions n_host .. n-1, the TAIL, are chosen on the device on the step stream right before the step, from the state the
 *     step itself sees (whatever is in flight): first the groups outside gids that a sweep at t = max(sweep[r]) would fire, lowest
 *     gids first, up to cap of them; then FILLERS, groups outside gids that are not due at t, lowest first, until the tail holds
 *     cap entries.  Each of the two parts is strictly increasing; the tail and the whole list are not, and need not be: no
 *     kernel of a step depends on the order of its list, only on its uniqueness (one owner per lane's tag bitmap).
 *     Fillers keep n a host-known number, and they are exact: a listed group with no event whose timer is not due is left
 *     untouched by a sweep row.
 *   * counts[3] of the outbox is the full number of due groups outside gids.  If counts[3] <= cap, tail positions n_host ..
 *     n_host + counts[3] - 1 hold due groups and the rest fillers, and the step leaves the shard exactly as the whole-shard
 *     compact sweep step with the same events would.  If counts[3] > cap it is exactly the sweep step over gids u tail; the due
 *     groups left over stay due, untouched, and the next step finds them (raise cap).
 *   * tail_out (host [cap]) receives the tail; it is valid after rafting_step_wait_compact.
 *   * every column and slot is positional with n = n_host + cap, both ways, as for rafting_step_begin_compact_active
 *     (rafting_compact_layout(rows, n_host + cap, F, ...)); the host leaves the tail positions of op_c, op_unavail and ev_c empty.
 *     flags is 0, 1, 4 or 5; rafting_step_fetch_dense returns the COMPACT_GROUPS-shaped dense outbox with n = n_host + cap.
 *   * refused with nothing enqueued and the slot free: a request record or op escape at a position >= n_host or on a sweep row,
 *     a lane escape record at a tail position, no sweep row, cap = 0, and n_host + cap > max_groups (RAFTING_E_CAPACITY: there
 *     would not be enough fillers).
 * Use it rather than rafting_step_begin_compact_sweep over the PIPELINING RULE's list when steps are in flight: the rule must
 * list every event gid of the steps in flight as well, and at d = 3 that covers most of a heartbeat-driven shard. */
int rafting_step_begin_compact_due(rafting_engine_t* e, uint32_t slot /* 0..3 */, uint32_t n_host, const uint32_t* gids /* host, [n_host] */,
                                   uint32_t cap, const int64_t* sweep /* [rows], host */,
                                   const rafting_cinbox_t* in_host, const rafting_creqs_t* reqs,
                                   const rafting_coutbox_t* out_host, uint32_t* tail_out /* host [cap] */, uint32_t flags);
int rafting_step_wait_compact (rafting_engine_t* e, uint32_t slot);
/* the dense outbox of the compact step last waited for in `slot` (every column that is non-NULL in out_host): the lossless
   fallback when the escape list overflowed */
int rafting_step_fetch_dense  (rafting_engine_t* e, uint32_t slot, const rafting_outbox_t* out_host);

/* device path: inbox/outbox columns already resident in HBM (pointers are device pointers).
   `stream` is a cudaStream_t (0 = engine's stream). No host copies, no sync. */
int rafting_step_device(rafting_engine_t* e, const rafting_inbox_t* in_dev,
                        const rafting_outbox_t* out_dev, void* stream);

/* parity / checkpoint */
int rafting_state_export(rafting_engine_t* e, uint32_t gid, rafting_group_state_t* out);
int rafting_state_export_bulk(rafting_engine_t* e, uint32_t first_gid, uint32_t count,
                              rafting_group_state_t* out /* [count], host */);
int rafting_state_digest(rafting_engine_t* e, uint32_t first_gid, uint32_t count,
                         uint64_t* digests /* [count], host */);
int rafting_log_term    (rafting_engine_t* e, uint32_t gid, int64_t index, int64_t* term /* -1 = null */);
/* in-HBM checkpoint of every table (RaftContext.initialize restores from StableLock + RaftLog; here
   the whole shard is snapshotted / rolled back at once).  One shadow copy per engine. */
int rafting_checkpoint(rafting_engine_t* e);
int rafting_restore   (rafting_engine_t* e);
int rafting_restore_async(rafting_engine_t* e);   /* the same, enqueued on the step stream without a host synchronisation */
/* the same state as ONE file that survives the process (planned restart / move of a shard): header + checksummed blocks,
   written to <path>.tmp, fdatasync'ed and renamed.  Load needs an engine created with the same max_groups / replicas; it
   verifies every block before touching the tables.  Drains the step stream; RAFTING_E_BUSY while a host step is in flight. */
int rafting_state_save(rafting_engine_t* e, const char* path);
int rafting_state_load(rafting_engine_t* e, const char* path);

/* ---- HBM-resident segmented entry buffer with async pinned-host spill (rafting_b200/csrc/seglog.cuh) ----
   Payload side of RaftLog (M/command/RaftLog.java:72-132; RocksLog.java:82-242): newEntry/append ->
   rafting_log_append; get/batch -> rafting_log_read / rafting_log_gather.  truncate/flush need no call:
   a record is visible iff its index lies in the group's stored key range kept by the step kernel. */
typedef struct rafting_entry_ref {
    uint32_t gid;
    uint32_t len;        /* payload bytes; 0xffffffff in gather output = not stored */
    int64_t  index, term;
    uint64_t blob_off;   /* offset of the payload inside the accompanying blob (8-byte aligned on output) */
} rafting_entry_ref_t;
int rafting_log_config(rafting_engine_t* e, uint32_t segment_bytes, uint32_t hbm_segments, uint32_t ring_slots /* pow2 */);
int rafting_log_append(rafting_engine_t* e, const rafting_entry_ref_t* refs, uint32_t n, const void* blob, size_t blob_bytes);
int rafting_log_read  (rafting_engine_t* e, uint32_t gid, int64_t first_index, uint32_t max_n,
                       rafting_entry_ref_t* refs_out, void* blob_out, size_t blob_cap, uint32_t* n_out);
int rafting_log_gather(rafting_engine_t* e, uint32_t n_ranges, const uint32_t* gids, const int64_t* firsts,
                       const uint32_t* counts, rafting_entry_ref_t* refs_out, uint32_t refs_cap,
                       void* blob_out, size_t blob_cap, uint32_t* n_out, size_t* bytes_out);
/* garbage collection behind RaftLog.flush (RocksLog.java:228-242): drops the index entries below each group's lowest
   stored key and frees cold (pinned host) segments that hold no live record any more */
int rafting_log_trim  (rafting_engine_t* e, uint32_t first_gid, uint32_t count, uint64_t* dropped_entries, uint64_t* freed_cold_bytes);
/* PAYLOADS OF A COMPACT STEP'S PLANS, gathered on the device: what rafting_log_gather returns for the step's AppendEntries
 * ranges, without decoding plan_c words or escape records on the host.
 *   * Which plans: those of the compact step last waited for in `slot`, whatever its shape (whole shard, active, sweep or due;
 *     flags 0, 1, 4 or 5; escaped plans included); the precondition of rafting_step_fetch_dense.  A plan of kind AE with entry
 *     count c > 0 asks for indices plan_pp.x + 1 ... plan_pp.x + c of its group; heartbeats without entries, IS, SKIP_INFLIGHT
 *     and UNAVAILABLE plans ask for nothing, and so does a step with no op and no sweep row (it has no plan columns).  Plans are
 *     walked in lane-slot order (row * n + position) * F + lane; positions map to gids through the step's list, a due step's
 *     device-chosen tail included.
 *   * refs_out: one record per asked-for entry, plan after plan in that order: exactly the gid, index, term and len that
 *     rafting_log_gather returns for the same ranges in the same order (len 0xffffffff: never appended).
 *     plans_out: one record per plan with entries (its lane slot, its first ref, its count).
 *     blob_out: the payloads at blob_off, 16-byte aligned; entries served on the device first, in ref order, then the entries
 *     the host serves.
 *   * Semantics: the payloads are what rafting_log_gather over those ranges returns at the point in the entry buffer's stream
 *     where the begin is enqueued.  Visibility stays the caller's, as for rafting_log_gather.
 *   * Ordering: the work runs on the entry buffer's stream, behind every rafting_log_append made before the begin (the payloads
 *     of the SUBMITs that created the step's entries included); the step stream never waits for it.  rafting_log_append,
 *     rafting_log_trim and rafting_log_store_open return RAFTING_E_BUSY while a gather is not waited for.
 *   * Host-served entries: an entry the device ring does not hold (the ring slot caches a newer index, the record is in the
 *     pinned cold tier or the entry file, or it was never appended) goes to a miss list, which the wait serves through the host
 *     index; host work is proportional to misses.  *host_served is their number.
 *   * Capacity: nothing past refs_cap, plans_cap or blob_cap is written; when one is exceeded the wait returns
 *     RAFTING_E_CAPACITY with the sizes needed in *n_refs, *bytes, *n_plans.  The slot's plans stay resident: begin again.
 *   * Slot lifetime: a slot holds at most one gather (a second begin is RAFTING_E_BUSY); while it is not waited for, every step
 *     begin on the slot returns RAFTING_E_BUSY with nothing enqueued.  A begin without a finished compact step in the slot, or
 *     without rafting_log_config, is RAFTING_E_INVAL.
 *   * Output memory: pinned or registered outputs (blob_out 16-byte aligned) are written by the device directly, so only the
 *     gathered bytes cross PCIe; any other host memory goes through pinned staging of the slot, copied at the wait.  Outputs
 *     stay valid until the wait; nothing synchronises the host between begin and wait. */
typedef struct rafting_plan_ref { uint32_t slot, first, count, _pad; } rafting_plan_ref_t;   /* lane slot, first ref, refs */
int rafting_log_gather_step_begin(rafting_engine_t* e, uint32_t slot /* 0..3 */,
                                  rafting_entry_ref_t* refs_out, uint32_t refs_cap,
                                  void* blob_out, size_t blob_cap,
                                  rafting_plan_ref_t* plans_out, uint32_t plans_cap);
int rafting_log_gather_step_wait (rafting_engine_t* e, uint32_t slot,
                                  uint32_t* n_refs, size_t* bytes, uint32_t* n_plans, uint32_t* host_served);
int rafting_log_stats (rafting_engine_t* e, uint64_t* out /* appended, head, spilled_bytes, hbm_hits, cold_hits, indexed,
                                                              last gather kernels ns, last gather bytes, trimmed entries,
                                                              cold bytes freed, spills skipped (dead segments) */, uint32_t n);

/* Durable tier of the entry buffer (SURVEY.md §8(f)-1; what flushWal(true) gives RocksLog, RocksLog.java:87,195).  With an
   entry file open every rafting_log_append is framed into it first (write-ahead) and rafting_log_sync is the ONE durability
   barrier per step (fdatasync) — issue it before the step's replies are released.  The stored key range is metadata of the
   step kernel, so the pump logs truncations / compactions with rafting_log_mark; rafting_log_store_open replays the file
   (torn tail cut) and rafting_log_recovered summarises a group for rafting_group_open + rafting_group_load_runs.  The file
   is also the coldest read tier, which bounds the pinned-host pool to cold_max_segments (0 = unbounded).
   rafting_log_append / gather / read run on the entry buffer's own stream: the step kernel's stream never waits for them.
   Visibility of gathered entries is the CALLER's: pass ranges taken from this step's plans (rafting_log_read checks the
   group's stored key range itself). */
int rafting_log_store_open(rafting_engine_t* e, const char* path, uint32_t cold_max_segments, uint64_t* recovered_records);
int rafting_log_sync      (rafting_engine_t* e);
int rafting_log_mark      (rafting_engine_t* e, uint32_t gid, int64_t lowest_key, int64_t highest_key /* lo > hi: empty */,
                           int64_t epoch_index, int64_t epoch_term);
int rafting_log_recovered (rafting_engine_t* e, uint32_t gid, rafting_group_init_t* init /* epoch, key range, last term */,
                           rafting_i64x2_t* runs /* [cap] (first index, term), oldest first */, uint32_t cap, uint32_t* n_runs);
/* one stored entry in the reference's RocksDB layout (RocksLog.java:82-89,259-280): key = 8-byte BE index,
   value = 8-byte BE term || payload — what the reference's LogChecker iterates over */
int rafting_log_export_kv (rafting_engine_t* e, uint32_t gid, int64_t index, uint8_t key_out[8], void* val_out, size_t val_cap,
                           size_t* val_len);
int rafting_log_store_stats(rafting_engine_t* e, uint64_t out[6] /* file bytes, synced bytes, fdatasync calls, file-tier reads,
                                                                    cold segments evicted, cold segments resident */);
/* multi-GPU summary (SURVEY.md §8(e), BASELINE config #4): groups shard by contiguous gid blocks, rank r owns global groups
   [r*G, (r+1)*G); the ONLY exchange is one ncclAllGather of commitIndex[G] (int64) per step into a [world * G] device
   buffer every rank keeps (two, alternating).  The gather runs on its own stream behind the kernel that produced the column.
     rafting_comm_init          one process per GPU: every rank passes the same 128-byte NCCL unique id (world == 1: no NCCL)
     rafting_comm_init_all      ONE process owning n shards on n devices (the reference's host is a single JVM,
                                ContextManager.java:46): engines[r] becomes rank r; the n ncclCommInitRank calls are grouped
     rafting_allgather_commit_from   source = a device column the caller names, normally the step's outbox commit_index
                                column (an end-of-step snapshot): the gathered vector is exactly the state after that step
                                on every rank, and the next step kernel does not wait for the gather (the step stream waits
                                for the gather issued one call EARLIER, so rotate at least two outboxes)
     rafting_allgather_commit   source = the live table column; the next step kernel waits for the gather
     rafting_allgather_commit_all    the same for every shard of a rafting_comm_init_all communicator, issued as one NCCL group
   host_out != NULL: the call synchronises and copies the [world * G] vector to the host. */
int rafting_commit_slice(rafting_engine_t* e, void** dev_ptr, uint32_t* count);
int rafting_comm_init   (rafting_engine_t* e, int rank, int world, const void* nccl_unique_id, size_t id_len);
int rafting_comm_init_all(rafting_engine_t** engines, int n);
int rafting_comm_unique_id(void* out, size_t* len);
int rafting_allgather_commit(rafting_engine_t* e, int64_t* host_out /* [world*G], may be NULL */, void** dev_out);
int rafting_allgather_commit_from(rafting_engine_t* e, const int64_t* dev_src /* [G] device, NULL = table column */,
                                  int64_t* host_out, void** dev_out);
int rafting_allgather_commit_all(rafting_engine_t** engines, int n, const int64_t* const* dev_srcs /* may be NULL */,
                                 int64_t* const* host_outs /* may be NULL */, void** dev_outs /* [n], may be NULL */);
int rafting_allgather_join  (rafting_engine_t* e);  /* the step stream waits for the gathers enqueued so far */
int rafting_allgather_last  (rafting_engine_t* e, int64_t* host_out /* [world*G] */);  /* the most recently gathered vector */
/* n device-resident steps enqueued by one call (ins[k] -> outs[k], in order): what a pump thread with a queue of decoded
   batches does, without n trips through the binding.  gather != 0: each step is followed by
   rafting_allgather_commit_from(outs[k].commit_index). */
int rafting_step_device_seq(rafting_engine_t* e, const rafting_inbox_t* ins_dev, const rafting_outbox_t* outs_dev, uint32_t n,
                            int gather, void* stream);

/* introspection used by bench/tests */
int rafting_engine_stream(rafting_engine_t* e, void** cuda_stream);
int rafting_engine_counters(rafting_engine_t* e, uint64_t* kernel_launches,
                            uint64_t* events_processed /* reserved: always 0 in this version */);
int64_t rafting_backoff_step(int32_t recent_rejection);   /* integer form of round(ln(e + r)), Leadership.java:105 */
int rafting_abi_sizes(uint32_t* out, uint32_t n);   /* sizeof of the ABI structs as compiled, for binding self-checks */

#ifdef __cplusplus
}
#endif
#endif /* RAFTING_B200_H */
