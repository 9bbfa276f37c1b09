// tables.cuh — HBM-resident SoA state of the batched Multi-Raft engine (sm_90a).
//
// Group-major layout: every per-group scalar is its own column (index = gid); every per-follower
// field lives in a 16-byte "plane" (index = gid * F + lane) so that a sub-warp of W lanes reads one
// group's replica table with consecutive 128-bit loads.  DESIGN.md §4 has the byte budget.
//
// What each column restates in the reference (M/ = src/main/java/io/lubricant/consensus/raft/):
//   g_meta   lo32 word: role (class of RaftContext.participant()), alive (stillRunning),
//            timeoutDetected (Follower.java:23), prepared (Leader.followerStatus != null, Leader.java:24),
//            votedFor / currentLeader (RaftMember.lastCandidate, Follower.currentLeader), nruns;
//            hi32 incarnation = number of RaftMember constructions (RaftMember.java:20-26)
//   g_term   RaftMember.currentTerm
//   g_commit RocksLog.commitIndex (RocksLog.java:50) — lives inside the all-gather buffer
//   g_lo/g_hi lowest / highest stored log key (RocksLog keys; empty when nruns == 0)
//   g_timer  TimerTicket deadline (non-leader) or the Leader's next keepAlive time (RaftRoutine.java:86-130)
//   g_epoch  RocksLog.epochEntry (index, term)
//   g_elect  Candidate.elected bookkeeping: (term of the elected Candidate, its incarnation | votes << 32)
//   g_runs   run-length index->term map, newest run first: replaces RocksLog.get(i).term()
//   l_*      Leadership.State (Leadership.java:26-38), one slot per (group, follower)
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "../../include/rafting_b200.h"

namespace rafting {

struct __align__(16) i64x2 { int64_t x, y; };

// internal g_meta word bits
constexpr uint32_t W_ROLE_MASK   = 3u;
constexpr uint32_t W_ALIVE       = 1u << 2;
constexpr uint32_t W_TIMEOUT_DET = 1u << 3;
constexpr uint32_t W_PREPARED    = 1u << 4;
constexpr uint32_t W_ELECT_ABORT = 1u << 5;
constexpr uint32_t W_READY       = 1u << 6;
constexpr int      W_BALLOT_SH   = 8;    // 8 bits, ballot + 1
constexpr int      W_LEADER_SH   = 16;   // 8 bits, currentLeader + 1
constexpr int      W_NRUNS_SH    = 24;   // 4 bits

struct Tables {
    uint64_t* g_meta;
    int64_t*  g_term;
    int64_t*  g_commit;
    int64_t*  g_lo;
    int64_t*  g_hi;
    int64_t*  g_timer;
    i64x2*    g_epoch;
    i64x2*    g_elect;
    uint32_t* g_err;
    i64x2*    g_runs;     // [RAFTING_TERM_RUNS][G]
    i64x2*    l_nm;       // (nextIndex, matchIndex)
    i64x2*    l_es;       // (lastEpoch, requestSuccess)
    i64x2*    l_fr;       // (requestFailure, lastRequest)
    int4*     l_cnt;      // (requestInFlight, recentRejection, recentFailure, pendingInstallation)
    uint32_t  G;          // capacity (max_groups)
    uint32_t  F;          // follower lanes
};

// device views of the batch (same field meaning as rafting_inbox_t / rafting_outbox_t)
struct InboxD {
    uint32_t rows, n;
    const uint32_t* gids;
    const int64_t*  row_now;
    const uint64_t* op_meta;
    const i64x2*    op_nr;
    const i64x2*    op_ab;
    const i64x2*    op_cd;
    const int64_t*  op_e;
    const int64_t*  ent_terms;
    uint32_t        ent_count;
    uint32_t        flags;
    const uint64_t* ev_meta;
    const i64x2*    ev_tn;
    const i64x2*    ev_el;
    // engine-internal (launch_step): positions sorted by class — perm[c * n ..) the positions of class c, perm_cnt[c]
    // their number (classify_kernel, step_kernel.cuh)
    const uint32_t* perm;
    const uint32_t* perm_cnt;
};
struct OutboxD {
    uint32_t* rep_meta; int64_t* rep_term;
    uint64_t* plan_meta; i64x2* plan_pp; i64x2* plan_lc; int64_t* plan_epoch;
    uint64_t* ballot_meta; int64_t* ballot_term; i64x2* ballot_last;
    int64_t* commit_index; int64_t* current_term; uint32_t* role_word; uint32_t* incarnation; uint32_t* err_word;
    i64x2* last_entry;
    uint32_t* flags;          // engine-internal: [0] += ballots emitted, [1] += valid replies (host path's sparse D2H)
};
struct CfgD {
    uint32_t replicas, local_slot;
    int32_t  pre_vote, avail_critical_point;
    int64_t  recovery_cool_down_ms, heartbeat_ms, election_ms;
    uint64_t timer_seed;
    uint32_t flags, _pad;           // rafting_cfg_t.flags: read only by the FIX instantiations of the step kernels
};

}  // namespace rafting
