"""Known-answer tests that pin the CPU oracle to the reference, branch by branch.

Upstream holds no test of this path (SURVEY.md §4); the only upstream known-answer material is the
comment table at M/context/member/Leadership.java:120-126, checked first.  Every other case is
hand-derived from the cited reference lines (M/ = src/main/java/io/lubricant/consensus/raft/).
"""
import math
import os

import numpy as np
import pytest

from oracle import binding
from rafting_b200 import abi
from rafting_b200.abi import (ERR, OUT_CANCELED, OUT_ERROR, OUT_OK, ROLE_CANDIDATE, ROLE_FOLLOWER, ROLE_LEADER,
                              I64_MAX)

T0 = 1_700_000_000_000


# --------------------------------------------------------------------------------------------
# Leadership.java:116-130 — majorIndices and the comment table :120-126
# --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n_nodes,major_pos", [(2, 0), (3, 1), (4, 1), (5, 2), (6, 2), (7, 3)])
def test_major_position_table(n_nodes, major_pos):
    """|x|o|*| table: with N nodes there are N-1 followers; the 'o' cell is sorted[(N-1)/2]."""
    followers = n_nodes - 1
    match = list(range(10, 10 + followers))          # already sorted, distinct
    full, major = binding.major_indices(match[::-1])
    assert full == match[0]
    assert major == match[major_pos]
    # majority property: leader + followers with matchIndex >= major form a majority of N
    assert 1 + sum(m >= major for m in match) >= n_nodes // 2 + 1
    # and it is the largest such index
    bigger = [m for m in match if m > major]
    if bigger:
        assert 1 + sum(m >= min(bigger) for m in match) < n_nodes // 2 + 1


def test_major_indices_random():
    rng = np.random.default_rng(7)
    for _ in range(200):
        n = int(rng.integers(1, 33))
        m = rng.integers(0, 50, size=n).tolist()
        s = sorted(m)
        assert binding.major_indices(m) == (s[0], s[n // 2])


# --------------------------------------------------------------------------------------------
# Leadership.java:105 — round(ln(e + r)) as the JVM computes it
# --------------------------------------------------------------------------------------------
def test_backoff_step_matches_double_math():
    L = binding.lib()
    for r in list(range(0, 3000)) + [4912, 4913, 13357, 13358, 36312, 36313, 98713, 98714, 2**31 - 1]:
        assert L.orc_backoff_step(r) == math.floor(math.log(math.e + r) + 0.5)


# --------------------------------------------------------------------------------------------
# Membership.java:74-108 — isBetter
# --------------------------------------------------------------------------------------------
F_, C_, L_ = ROLE_FOLLOWER, ROLE_CANDIDATE, ROLE_LEADER


@pytest.mark.parametrize("new,cur,expect", [
    ((F_, 5, 0), None, 1),                       # :75-77 null
    ((F_, 6, 0), (L_, 5, 0), 1),                 # :80-82 higher term wins
    ((L_, 4, 0), (F_, 5, 0), 0),                 # lower term loses
    ((L_, 5, 0), (C_, 5, 0), 1),                 # :86-87 candidate wins the election
    ((L_, 5, 0), (F_, 5, 1), -ERR["LEADER_UNCHANGED"]),   # :89
    ((F_, 5, 1), (C_, 5, 0), 1),                 # :92 follower beats candidate
    ((F_, 5, 1), (L_, 5, 0), 1),                 # :92 follower "beats" leader (Leader.appendEntries path)
    ((C_, 5, 0), (F_, 5, 1), 0),                 # :92
    ((C_, 5, 0), (L_, 5, 0), 0),
    ((L_, 5, 0), (L_, 5, 0), 0),                 # :95-97
    ((F_, 5, 2), (F_, 5, 1), 1),                 # :98-100 same-term follower is always re-created
    ((C_, 5, 0), (C_, 5, 0), 0),                 # :107
    ((C_, 5, 0), (C_, 5, 1), -ERR["BALLOT_MISMATCH"]),    # :103-105
])
def test_is_better(new, cur, expect):
    L = binding.lib()
    if cur is None:
        got = L.orc_is_better(new[0], new[1], new[2], 0, 0, 0, 1)
    else:
        got = L.orc_is_better(new[0], new[1], new[2], cur[0], cur[1], cur[2], 0)
    assert got == expect


# --------------------------------------------------------------------------------------------
# helpers: drive one group through the batch interface
# --------------------------------------------------------------------------------------------
SUT_FACTORY = binding.Oracle     # tests/test_engine_gpu.py re-runs every scenario below with the CUDA engine


class One:
    """One group, R replicas, local slot 0; each call is a one-row step."""

    def __init__(self, replicas=3, pre_vote=True, **init):
        self.cfg = abi.make_cfg(replicas=replicas, local_slot=0, max_groups=1, max_rows=1, pre_vote=pre_vote,
                                heartbeat_ms=300, election_ms=900, entry_pool_cap=64)
        self.F = replicas - 1
        self.o = SUT_FACTORY(self.cfg)
        init.setdefault("now_ms", T0)
        init.setdefault("rand_ms", 1000)
        self.o.open_group(0, **init)
        self.now = T0

    def inbox(self):
        return abi.Inbox(1, 1, self.F, ent_cap=64)

    def run(self, ib):
        out = self.o.step(ib)
        self.out = out
        return out

    @property
    def st(self):
        return self.o.export(0)

    # shortcuts
    def timeout(self, rand=1000, unavail=0):
        ib = self.inbox(); ib.timeout(0, 0, self.now, rand=rand, unavail=unavail); return self.run(ib)

    def submit(self, count=1):
        ib = self.inbox(); ib.submit(0, 0, self.now, count=count); return self.run(ib)

    def votes(self, replies, pre):
        """replies: {lane: (resp_term, granted[, outcome])}"""
        ib = self.inbox()
        inc = self.st.incarnation
        for f, rep in replies.items():
            outcome = rep[2] if len(rep) > 2 else OUT_OK
            ib.vote_reply(0, 0, f, self.now, inc, rep[0], rep[1], outcome=outcome, pre=pre)
        return self.run(ib)

    def acks(self, acks):
        """acks: {lane: dict(resp_term, success, epoch, last[, outcome, snapshot, inc])}"""
        ib = self.inbox()
        for f, a in acks.items():
            ib.ack(0, 0, f, self.now, a.get("inc", self.st.incarnation), a["resp_term"], a["success"], a["epoch"],
                   a["last"], outcome=a.get("outcome", OUT_OK), snapshot=a.get("snapshot", False))
        return self.run(ib)

    def elect(self):
        """Follower -> (pre-vote) -> Candidate -> Leader with unanimous grants."""
        self.timeout()
        if self.cfg.pre_vote:
            t = self.st.current_term
            self.votes({f: (t, True) for f in range(self.F)}, pre=True)
        t = self.st.current_term
        self.votes({f: (t, True) for f in range(self.F)}, pre=False)
        assert self.st.role == ROLE_LEADER
        return self


def err_code(word):
    return word & 0xFFFF


# --------------------------------------------------------------------------------------------
# RaftContext.initialize + RaftRoutine.resetTimer
# --------------------------------------------------------------------------------------------
def test_initialize_becomes_follower_with_armed_timer():
    g = One(term=7, ballot=2, now_ms=T0, rand_ms=1234)
    s = g.st
    assert (s.role, s.current_term, s.voted_for, s.incarnation) == (ROLE_FOLLOWER, 7, 2, 1)
    assert s.timer == T0 + 1234           # max(0 + 1, now + timeout), RaftRoutine.java:105-107
    assert s.current_leader == -1 and s.timeout_detected == 0


# --------------------------------------------------------------------------------------------
# election: Follower.onTimeout / prepareElection / PV-Echo / Candidate / RV-Echo
# --------------------------------------------------------------------------------------------
def test_prevote_round_then_candidate_then_leader():
    g = One(replicas=5, term=3, ballot=-1)
    out = g.timeout(rand=1111)
    s = g.st
    # Follower.java:159: same-term Follower re-created, then prepareElection on the new object
    assert (s.role, s.current_term, s.incarnation, s.timeout_detected, s.votes) == (ROLE_FOLLOWER, 3, 2, 1, 1)
    assert s.timer == T0 + 1111
    assert int(out.ballot_meta[0, 0]) & 0xF == abi.BALLOT_PREVOTE
    assert int(out.ballot_meta[0, 0]) >> 32 == 2
    assert out.ballot_term[0, 0] == 4                      # nextTerm, Follower.java:246
    assert tuple(out.ballot_last[0, 0]) == (0, 0)          # empty log -> epoch (0,0)
    # one grant: votes 2 < majority 3
    g.votes({0: (3, True)}, pre=True)
    assert (g.st.role, g.st.votes) == (ROLE_FOLLOWER, 2)
    # a refusal and a second grant -> Candidate(term 4) which immediately broadcasts RequestVote
    out = g.votes({1: (3, False), 2: (4, True)}, pre=True)
    s = g.st
    assert (s.role, s.current_term, s.voted_for, s.votes, s.incarnation) == (ROLE_CANDIDATE, 4, 0, 1, 3)
    assert int(out.ballot_meta[0, 0]) & 0xF == abi.BALLOT_VOTE and out.ballot_term[0, 0] == 4
    # stale pre-vote reply for the dead Follower object is ignored
    ib = g.inbox(); ib.vote_reply(0, 0, 3, g.now, 2, 9, True, pre=True); g.run(ib)
    assert (g.st.role, g.st.current_term) == (ROLE_CANDIDATE, 4)
    # RV grants: 2 more -> Leader
    g.votes({0: (4, True)}, pre=False)
    assert g.st.role == ROLE_CANDIDATE
    g.votes({1: (4, True)}, pre=False)
    s = g.st
    assert (s.role, s.current_term, s.voted_for, s.incarnation) == (ROLE_LEADER, 4, 0, 4)
    assert (s.elected_inc, s.elected_term, s.elected_aborted) == (3, 4, 0)
    assert s.timer == g.now                                # first heartbeat is due immediately (delay 0)


def test_prevote_reply_with_term_equal_to_next_term_does_not_step_down():
    g = One(term=3)
    g.timeout()
    g.votes({0: (4, False)}, pre=True)                     # result.term() > nextTerm is false, Follower.java:261
    assert (g.st.role, g.st.current_term, g.st.incarnation) == (ROLE_FOLLOWER, 3, 2)
    g.votes({1: (5, False)}, pre=True)                     # 5 > 4 -> Follower(5, ballot = responder)
    s = g.st
    assert (s.role, s.current_term, s.voted_for, s.incarnation) == (ROLE_FOLLOWER, 5, 2, 3)


def test_no_prevote_goes_straight_to_candidate():
    g = One(pre_vote=False, term=3)
    out = g.timeout()
    s = g.st
    assert (s.role, s.current_term, s.voted_for) == (ROLE_CANDIDATE, 4, 0)
    assert int(out.ballot_meta[0, 0]) & 0xF == abi.BALLOT_VOTE
    out = g.timeout()                                      # Candidate.onTimeout: new election at term 5
    assert (g.st.role, g.st.current_term, g.st.incarnation) == (ROLE_CANDIDATE, 5, 3)


def test_vote_reply_errors_and_cancels_are_ignored():
    g = One(pre_vote=False, term=1)
    g.timeout()
    g.votes({0: (9, True, OUT_ERROR), 1: (9, True, OUT_CANCELED)}, pre=False)
    assert (g.st.role, g.st.current_term, g.st.votes) == (ROLE_CANDIDATE, 2, 1)


def test_elected_candidate_late_replies():
    """Candidate.onFencing skips the abort when elected (Candidate.java:75-80): late replies still run."""
    g = One(replicas=5, pre_vote=False, term=1)
    g.timeout()
    cand_inc = g.st.incarnation
    g.votes({0: (2, True), 1: (2, True)}, pre=False)
    assert g.st.role == ROLE_LEADER
    # late grant: trySwitchTo(Leader) is "not better" -> nothing
    ib = g.inbox(); ib.vote_reply(0, 0, 2, g.now, cand_inc, 2, True); g.run(ib)
    assert (g.st.role, g.st.incarnation, err_code(g.st.err_word)) == (ROLE_LEADER, cand_inc + 1, 0)
    # late higher-term reply: the live Leader steps down, ballot = responder (lane 3 -> slot 4)
    ib = g.inbox(); ib.vote_reply(0, 0, 3, g.now, cand_inc, 7, False); g.run(ib)
    s = g.st
    assert (s.role, s.current_term, s.voted_for, s.elected_aborted) == (ROLE_FOLLOWER, 7, 4, 1)
    # the zombie head is now aborted: further replies are dropped
    ib = g.inbox(); ib.vote_reply(0, 0, 2, g.now, cand_inc, 99, False); g.run(ib)
    assert g.st.current_term == 7


# --------------------------------------------------------------------------------------------
# Leader: prepareReplication / replicateLog / acks / tryCommit
# --------------------------------------------------------------------------------------------
def test_first_heartbeat_prepares_replication_and_submit_needs_ready():
    g = One(term=1).elect()
    t = g.st.current_term
    out = g.submit()
    assert out.rep_meta[0, 0] >> 8 == ERR["NOT_READY"]     # followerStatus == null -> isReady false
    out = g.timeout()                                      # keepAlive -> replicateLog(true)
    s = g.st
    assert s.leader_prepared == 1 and s.timer == g.now + 300
    for f in range(2):
        assert int(out.plan_meta[0, 0, f]) & 0xF == abi.PLAN_AE
        assert (int(out.plan_meta[0, 0, f]) >> 4) & 1 == 1            # heartbeat
        assert tuple(out.plan_pp[0, 0, f]) == (0, 0) and tuple(out.plan_lc[0, 0, f]) == (0, 0)
        assert s.followers[f].next_index == 1 and s.followers[f].request_in_flight == 1
        assert s.followers[f].last_request == g.now
    out = g.submit()
    assert out.rep_meta[0, 0] >> 8 == ERR["NOT_READY"]     # requestSuccess == 0 still
    g.acks({0: dict(resp_term=t, success=True, epoch=0, last=0)})
    out = g.submit()                                       # 1 + 1 ready > 2/2 -> ready
    assert out.rep_meta[0, 0] >> 8 == 0
    s = g.st
    assert (s.last_index, s.last_term, s.term_runs) == (1, t, 1)
    # nextIndex is still 1 -> batch(0, 51): prev = epoch(0,0), entries = [1]
    assert tuple(out.plan_pp[0, 0, 0]) == (0, 0) and tuple(out.plan_lc[0, 0, 0]) == (1, 0)
    assert (int(out.plan_meta[0, 0, 0]) >> 16) & 0xFFFF == 1


def test_ack_advances_match_and_commit_r3():
    g = One(term=1).elect(); t = g.st.current_term
    g.timeout()
    g.acks({0: dict(resp_term=t, success=True, epoch=0, last=0), 1: dict(resp_term=t, success=True, epoch=0, last=0)})
    g.submit(count=3)
    assert g.st.last_index == 3
    g.now += 5
    g.acks({0: dict(resp_term=t, success=True, epoch=0, last=3)})
    s = g.st
    assert (s.followers[0].match_index, s.followers[0].next_index) == (3, 4)
    assert s.commit_index == 3                             # R=3: major = max(3, 0) = 3, term matches
    assert s.followers[0].request_success == g.now and s.followers[0].request_in_flight == 0  # hb + submit sent, both acked
    g.acks({1: dict(resp_term=t, success=True, epoch=0, last=2)})
    assert g.st.commit_index == 3                          # unchanged: commitIndex == lastCommitted


def test_commit_needs_current_term_entry_r5():
    """Leader.java:257-261: an entry of an older term commits only when replicated everywhere."""
    g = One(replicas=5, term=1, first_index=1, last_index=4, last_term=1)
    g.elect(); t = g.st.current_term
    assert t == 2
    g.timeout()
    for f in range(4):
        assert g.st.followers[f].next_index == 5
    # three followers hold index 4 (term 1 != 2): major = sorted[2]; full = min
    g.acks({0: dict(resp_term=t, success=True, epoch=0, last=4), 1: dict(resp_term=t, success=True, epoch=0, last=4),
            2: dict(resp_term=t, success=True, epoch=0, last=2)})
    assert g.st.commit_index == 0                          # full index is 0 (lane 3 unmatched)
    g.acks({3: dict(resp_term=t, success=True, epoch=0, last=1)})
    assert g.st.commit_index == 1                          # commit the fully replicated prefix
    # now the leader appends in its own term and a majority acks it
    g.acks({})
    g.submit()                                             # index 5 @ term 2
    g.acks({0: dict(resp_term=t, success=True, epoch=0, last=5), 1: dict(resp_term=t, success=True, epoch=0, last=5)})
    assert g.st.commit_index == 5                          # sorted = [1,2,5,5] -> [2] = 5, term(5) == 2


def test_reject_backoff_and_pending_installation():
    g = One(term=1, first_index=1, last_index=10, last_term=1).elect(); t = g.st.current_term
    g.timeout()
    assert g.st.followers[0].next_index == 11
    # first reject: recentRejection=1 -> step = round(ln(e+1)) = 1 -> next = min(10, max(10, 1)) = 10
    g.acks({0: dict(resp_term=t, success=False, epoch=0, last=10)})
    s = g.st.followers[0]
    assert (s.next_index, s.recent_rejection, s.match_index, s.pending_installation) == (10, 1, 0, 0)
    # second: r=2 -> step 2 -> 8 ; third: r=3 -> step 2 -> 6
    g.acks({0: dict(resp_term=t, success=False, epoch=0, last=10)})
    assert g.st.followers[0].next_index == 8
    g.acks({0: dict(resp_term=t, success=False, epoch=0, last=10)})
    assert g.st.followers[0].next_index == 6
    # success resets recentRejection and jumps nextIndex
    g.acks({0: dict(resp_term=t, success=True, epoch=0, last=7)})
    s = g.st.followers[0]
    assert (s.next_index, s.match_index, s.recent_rejection) == (8, 7, 0)
    # reject with matchIndex != 0 leaves nextIndex alone (:103)
    g.acks({0: dict(resp_term=t, success=False, epoch=0, last=7)})
    assert g.st.followers[0].next_index == 8


def test_flush_triggers_install_snapshot_and_recovery():
    g = One(term=1, first_index=1, last_index=10, last_term=1).elect(); t = g.st.current_term
    g.timeout()
    g.acks({0: dict(resp_term=t, success=True, epoch=0, last=10), 1: dict(resp_term=t, success=False, epoch=0, last=10)})
    assert g.st.followers[1].next_index == 10
    ib = g.inbox(); ib.flush(0, 0, g.now, 10, 1); g.run(ib)
    s = g.st
    assert (s.epoch_index, s.epoch_term, s.first_index, s.last_index) == (10, 1, 10, 10)   # entry 10 survives the flush
    out = g.timeout()                                      # plans carry the new epoch
    assert out.plan_epoch[0, 0, 1] == 10
    # lane 1's ack for that plan: epoch 10 > lastEpoch 0 -> nextIndex = max(10,10)=10, then reject at matchIndex==0:
    # step=round(ln(e+2))=2: next = max(10-2, 11) = 11 -> min(9, 11) = 9 -> 9 <= epoch -> pending
    g.acks({1: dict(resp_term=t, success=False, epoch=10, last=10)})
    s = g.st.followers[1]
    assert (s.last_epoch, s.next_index, s.pending_installation) == (10, 9, 1)
    out = g.timeout()
    assert int(out.plan_meta[0, 0, 1]) & 0xF == abi.PLAN_IS and tuple(out.plan_pp[0, 0, 1]) == (10, 1)
    assert int(out.plan_meta[0, 0, 0]) & 0xF == abi.PLAN_AE
    # an AE ack while pending is ignored by updateIndex (:90) but still counts as success stat
    g.acks({1: dict(resp_term=t, success=True, epoch=10, last=10)})
    assert g.st.followers[1].pending_installation == 1
    # IS-Echo false keeps pending; true clears it and sets nextIndex = epoch + 1
    g.acks({1: dict(resp_term=t, success=False, epoch=10, last=10, snapshot=True)})
    assert g.st.followers[1].pending_installation == 1
    g.acks({1: dict(resp_term=t, success=True, epoch=10, last=10, snapshot=True)})
    s = g.st.followers[1]
    assert (s.pending_installation, s.next_index) == (0, 11)


def test_match_rollback_throws_after_stat_success():
    g = One(term=1, first_index=1, last_index=5, last_term=1).elect(); t = g.st.current_term
    g.timeout()
    g.acks({0: dict(resp_term=t, success=True, epoch=0, last=5)})
    g.now += 7
    g.acks({0: dict(resp_term=t, success=False, epoch=0, last=3)})    # index 3 < matchIndex 5
    s = g.st
    assert err_code(s.err_word) == ERR["MATCH_ROLLBACK"]
    assert s.followers[0].request_success == g.now                     # statSuccess already ran (Leader.java:228)
    assert s.followers[0].recent_rejection == 1
    assert (s.followers[0].match_index, s.followers[0].next_index) == (5, 6)


def test_ack_error_and_cancel_stats():
    g = One(term=1).elect(); t = g.st.current_term
    g.timeout()
    g.now += 3
    g.acks({0: dict(resp_term=0, success=False, epoch=0, last=0, outcome=OUT_ERROR),
            1: dict(resp_term=0, success=False, epoch=0, last=0, outcome=OUT_CANCELED)})
    s = g.st
    assert (s.followers[0].request_failure, s.followers[0].recent_failure, s.followers[0].request_in_flight) == (g.now, 1, 0)
    assert (s.followers[1].request_failure, s.followers[1].recent_failure, s.followers[1].request_in_flight) == (g.now, 0, 0)


def test_ack_with_higher_term_steps_down():
    g = One(term=1).elect(); t = g.st.current_term
    g.timeout()
    g.acks({1: dict(resp_term=t + 3, success=False, epoch=0, last=0)})
    s = g.st
    assert (s.role, s.current_term, s.voted_for) == (ROLE_FOLLOWER, t + 3, 2)   # ballot = responder (lane 1 -> slot 2)
    inc = s.incarnation
    # acks addressed to the dead Leader object change nothing
    ib = g.inbox(); ib.ack(0, 0, 0, g.now, inc - 1, t, True, 0, 0); g.run(ib)
    assert g.st.raw() == s.raw()


def test_in_flight_limit_and_unavailable():
    g = One(term=1).elect(); t = g.st.current_term
    for _ in range(3):
        g.now += 300
        out = g.timeout()
    # heartbeat limit = 20/10 = 2: third heartbeat finds inFlight == 2 (not > 2) -> still sent; fourth is skipped
    assert g.st.followers[0].request_in_flight == 3
    g.now += 300
    out = g.timeout()
    assert int(out.plan_meta[0, 0, 0]) & 0xF == abi.PLAN_SKIP_INFLIGHT
    assert g.st.followers[0].request_in_flight == 3
    g.now += 300
    out = g.timeout(unavail=0b10)
    assert int(out.plan_meta[0, 0, 1]) & 0xF == abi.PLAN_UNAVAILABLE
    s = g.st.followers[1]
    assert (s.recent_failure, s.request_failure) == (1, g.now)


# --------------------------------------------------------------------------------------------
# Follower.appendEntries and the log model
# --------------------------------------------------------------------------------------------
def ae(g, leader, term, prev, prev_term, terms=(), commit=0, first=None, rand=1000):
    ib = g.inbox(); ib.ae_request(0, 0, g.now, leader, term, prev, prev_term, terms, commit, first_index=first, rand=rand)
    return g.run(ib)


def rep(out):
    m = int(out.rep_meta[0, 0])
    return (m & 1, (m >> 1) & 1, m >> 8, int(out.rep_term[0, 0]))


def test_append_entries_basic_and_passive_commit():
    g = One(term=2)
    out = ae(g, 1, 1, 0, 0)
    assert rep(out) == (1, 0, 0, 2)                        # stale term, Follower.java:39-41
    out = ae(g, 1, 2, 0, 0, [2, 2, 2], commit=2, rand=1500)
    assert rep(out) == (1, 1, 0, 2)
    s = g.st
    assert (s.last_index, s.last_term, s.commit_index, s.current_leader) == (3, 2, 2, 1)
    assert s.timer == g.now + 1500                         # unmuted with a fresh draw
    out = ae(g, 1, 2, 3, 2, [2], commit=9)
    assert g.st.commit_index == 4                          # min(leaderCommit, last.index)
    out = ae(g, 1, 2, 7, 2, [2])
    assert rep(out) == (1, 0, 0, 2)                        # prev not contained
    out = ae(g, 2, 2, 4, 2)                                # another leader in the same term
    assert rep(out)[2] == ERR["FOLLOWER_TWO_LEADERS"]
    assert g.st.timer == I64_MAX                           # timer left muted (Follower.java:43,48-50)


def test_append_entries_higher_term_recreates_follower():
    g = One(term=2, ballot=1)
    inc = g.st.incarnation
    ae(g, 2, 5, 0, 0, [5])
    s = g.st
    assert (s.current_term, s.voted_for, s.incarnation, s.current_leader) == (5, 1, inc + 1, 2)


def test_conflict_truncates_and_appends():
    g = One(term=3)
    ae(g, 1, 3, 0, 0, [1, 1, 2, 2, 3])
    assert g.o.log_term(0, 4) == 2
    out = ae(g, 1, 3, 2, 1, [3, 3])                        # conflict at index 3 (2 != 3): truncate 3.. then append
    assert rep(out) == (1, 1, 0, 3)
    s = g.st
    assert (s.last_index, s.last_term, s.term_runs) == (4, 3, 2)
    assert [g.o.log_term(0, i) for i in range(1, 6)] == [1, 1, 3, 3, -1]
    # identical resend is idempotent
    d = s.log_digest
    ae(g, 1, 3, 2, 1, [3, 3])
    assert g.st.log_digest == d
    # gap after the end: RocksLog.append "log index is not continuous"
    out = ae(g, 1, 3, 4, 3, [3], first=7)
    assert rep(out)[2] == ERR["LOG_NOT_CONTINUOUS"]


def test_purge_entries_below_epoch_and_epoch_checks():
    g = One(term=3, epoch_index=10, epoch_term=2, first_index=10, last_index=12, last_term=2)
    out = ae(g, 1, 3, 8, 2, [2, 2, 2, 2, 3])               # entries 9..13; 9,10 purged; 11,12 match; 13 new
    assert rep(out) == (1, 1, 0, 3)
    assert (g.st.last_index, g.st.last_term) == (13, 3)
    out = ae(g, 1, 3, 10, 1)                               # index == epoch.index but term differs
    assert rep(out)[2] == ERR["EPOCH_TERM_MISMATCH"]
    out = ae(g, 1, 3, 0, 5)
    assert rep(out)[2] == ERR["INDEX_TERM_ZERO"]
    out = ae(g, 1, 3, 5, 9, [9, 9])                        # prev and all entries below the epoch
    assert rep(out) == (1, 1, 0, 3) and g.st.last_index == 13


def test_passive_commit_rollback_is_an_assertion():
    g = One(term=2)
    ae(g, 1, 2, 0, 0, [2, 2, 2], commit=3)
    out = ae(g, 1, 2, 3, 2, [], commit=1)
    assert rep(out)[2] == ERR["COMMIT_ROLLBACK"] and g.st.commit_index == 3


def test_term_runs_overflow_is_rejected_before_mutation():
    g = One(term=20)
    out = ae(g, 1, 20, 0, 0, list(range(1, 9)))
    assert rep(out)[2] == 0 and g.st.term_runs == 8
    d = g.st.log_digest
    out = ae(g, 1, 20, 8, 8, [9])
    assert rep(out)[2] == ERR["TERM_RUNS_OVERFLOW"] and g.st.log_digest == d


def test_candidate_and_leader_receive_append_entries():
    g = One(pre_vote=False, term=1)
    g.timeout()                                            # Candidate(2)
    out = ae(g, 1, 2, 0, 0)                                # same term: becomes Follower(2) keeping its own ballot
    s = g.st
    assert rep(out) == (1, 1, 0, 2) and (s.role, s.voted_for, s.current_leader) == (ROLE_FOLLOWER, 0, 1)
    g = One(term=1).elect(); t = g.st.current_term; inc = g.st.incarnation
    assert rep(ae(g, 1, t, 0, 0))[2] == ERR["TWO_LEADERS"]
    assert rep(ae(g, 0, t + 1, 0, 0))[2] == ERR["LEADER_SELF_AE"]
    assert rep(ae(g, 1, t - 1, 0, 0)) == (1, 0, 0, t)
    out = ae(g, 2, t + 2, 0, 0)
    s = g.st
    assert rep(out) == (1, 1, 0, t + 2)
    assert (s.role, s.current_term, s.incarnation) == (ROLE_FOLLOWER, t + 2, inc + 2)   # Follower(t) then Follower(t+2)


# --------------------------------------------------------------------------------------------
# votes: Follower / Candidate / Leader request handlers
# --------------------------------------------------------------------------------------------
def vote(g, cand, term, li, lt, pre=False, rand=1000):
    ib = g.inbox()
    (ib.prevote_request if pre else ib.vote_request)(0, 0, g.now, cand, term, li, lt, rand=rand)
    return g.run(ib)


def test_follower_request_vote():
    g = One(term=3, ballot=1, first_index=1, last_index=5, last_term=3)
    assert rep(vote(g, 2, 2, 9, 9)) == (1, 0, 0, 3)
    assert rep(vote(g, 2, 3, 9, 9)) == (1, 0, 0, 3)        # same term, voted for 1
    assert rep(vote(g, 1, 3, 0, 0)) == (1, 1, 0, 3)        # same term, same candidate: no log check
    out = vote(g, 2, 4, 4, 3)                              # higher term, log NOT up to date: refuse but adopt term
    s = g.st
    assert rep(out) == (1, 0, 0, 4) and (s.current_term, s.voted_for) == (4, -1)
    out = vote(g, 2, 5, 5, 3)
    assert rep(out) == (1, 1, 0, 5) and g.st.voted_for == 2
    out = vote(g, 1, 6, 1, 4)                              # higher last term wins regardless of index
    assert rep(out) == (1, 1, 0, 6)


def test_follower_prevote_needs_timeout_detected():
    g = One(term=3)
    assert rep(vote(g, 1, 4, 0, 0, pre=True)) == (1, 0, 0, 3)          # !timeoutDetected
    g.timeout()
    assert rep(vote(g, 1, 3, 0, 0, pre=True)) == (1, 0, 0, 3)          # term <= currentTerm
    out = vote(g, 1, 4, 0, 0, pre=True, rand=1777)
    assert rep(out) == (1, 1, 0, 3) and g.st.current_term == 3         # pre-vote never changes the term
    assert g.st.timer == g.now + 1777


def test_candidate_prevote_is_request_vote():
    g = One(pre_vote=False, term=1)
    g.timeout()                                            # Candidate(2)
    out = vote(g, 2, 5, 0, 0, pre=True)                    # Candidate.preVote == requestVote: adopts the term, votes
    s = g.st
    assert rep(out) == (1, 1, 0, 5) and (s.role, s.current_term, s.voted_for) == (ROLE_FOLLOWER, 5, 2)
    g = One(pre_vote=False, term=1); g.timeout()
    assert rep(vote(g, 2, 2, 0, 0)) == (1, 0, 0, 2)        # same term, other candidate
    assert rep(vote(g, 0, 2, 0, 0))[2] == ERR["CANDIDATE_SELF_RV"]


def test_leader_vote_handlers():
    g = One(term=1).elect(); t = g.st.current_term
    assert rep(vote(g, 1, t + 5, 0, 0, pre=True)) == (1, 0, 0, t)      # Leader refuses every pre-vote
    assert rep(vote(g, 1, t, 0, 0)) == (1, 0, 0, t)
    out = vote(g, 2, t + 1, 0, 0)
    s = g.st
    assert rep(out) == (1, 1, 0, t + 1) and (s.role, s.voted_for) == (ROLE_FOLLOWER, 2)


def test_install_snapshot_request():
    g = One(term=3)
    ib = g.inbox(); ib.is_request(0, 0, g.now, 1, 2, 10, 2, True); out = g.run(ib)
    assert rep(out) == (1, 0, 0, 3) and g.st.timer == I64_MAX          # muted before the term check, stays muted
    ib = g.inbox(); ib.is_request(0, 0, g.now, 1, 4, 10, 2, True); out = g.run(ib)
    assert rep(out)[2] == ERR["IS_BEFORE_AE"]
    ib = g.inbox(); ib.is_request(0, 0, g.now, 1, 3, 10, 2, True, rand=1300); out = g.run(ib)
    assert rep(out) == (1, 1, 0, 3) and g.st.timer == g.now + 1300
    g2 = One(term=1).elect(); t = g2.st.current_term
    ib = g2.inbox(); ib.is_request(0, 0, g2.now, 1, t, 10, 2, True); out = g2.run(ib)
    assert rep(out)[2] == ERR["IS_BEFORE_AE"]
    ib = g2.inbox(); ib.is_request(0, 0, g2.now, 1, t - 1, 10, 2, True); out = g2.run(ib)
    assert rep(out) == (1, 0, 0, t)


def test_requests_refused_in_a_step_promising_none():
    """rafting_b200.h, RAFTING_INBOX_NO_REQUESTS: a step flagged to hold no inbound requests answers any request op
    found anyway with BAD_EVENT and an invalid reply, and leaves term, ballot, timer and log as they were.  SUBMIT and
    TIMEOUT still run in such a step."""
    g = One(term=3, ballot=1, first_index=1, last_index=5, last_term=3)
    g.timeout()                                            # timeoutDetected: a pre-vote would otherwise be granted
    before = g.st
    requests = [
        lambda ib: ib.ae_request(0, 0, g.now, 2, 7, 5, 3, [7, 7], leader_commit=6, rand=1300),
        lambda ib: ib.prevote_request(0, 0, g.now, 2, 4, 9, 3, rand=1300),
        lambda ib: ib.vote_request(0, 0, g.now, 2, 8, 9, 3, rand=1300),
        lambda ib: ib.is_request(0, 0, g.now, 2, 9, 40, 3, True, rand=1300),
        lambda ib: ib.flush(0, 0, g.now, 2, 3),
    ]
    for k, put in enumerate(requests):
        ib = g.inbox(); put(ib); ib.flags = abi.INBOX_NO_REQUESTS
        out = g.run(ib)
        assert rep(out)[:3] == (0, 0, ERR["BAD_EVENT"]), k
        s = g.st
        assert err_code(s.err_word) == ERR["BAD_EVENT"] and s.err_word >> 16 == k + 1
        for name in ("role", "current_term", "voted_for", "current_leader", "incarnation", "timer", "commit_index",
                     "epoch_index", "first_index", "last_index", "last_term", "log_digest"):
            assert getattr(s, name) == getattr(before, name), (k, name)
        assert int(out.current_term[0]) == 3 and int(out.ballot_meta[0, 0]) == 0
    g.now += 10
    ib = g.inbox(); ib.timeout(0, 0, g.now, rand=1200); ib.flags = abi.INBOX_NO_REQUESTS
    out = g.run(ib)
    assert rep(out)[2] == 0 and int(out.ballot_meta[0, 0]) & 0xF == abi.BALLOT_PREVOTE and g.st.timer == g.now + 1200


def test_restart_over_a_log_with_several_terms():
    """RaftContext.initialize over an existing RocksLog (RaftContext.java:91-113): the index->term map of the stored log
    comes back as runs; AppendEntries consistency checks must then see the right term at every index."""
    g = One(term=5, first_index=1, last_index=10, last_term=3)
    g.o.load_runs(0, [(1, 1), (4, 2), (8, 3)])
    assert [g.o.log_term(0, i) for i in (1, 3, 4, 7, 8, 10)] == [1, 1, 2, 2, 3, 3]
    # prev (7, 2) matches, (7, 3) does not (Follower.logContains, Follower.java:177-191)
    ib = g.inbox(); ib.ae_request(0, 0, g.now, 1, 5, 7, 3, [], leader_commit=0); out = g.run(ib)
    assert rep(out)[:2] == (1, 0)
    ib = g.inbox(); ib.ae_request(0, 0, g.now, 1, 5, 7, 2, [3, 3, 3, 5], leader_commit=9); out = g.run(ib)
    assert rep(out)[:2] == (1, 1)
    st = g.st
    assert (st.last_index, st.last_term, st.commit_index) == (11, 5, 9)
    assert g.o.log_term(0, 11) == 5 and g.o.log_term(0, 6) == 2
    # a conflicting suffix is cut at the first index whose stored term differs (RocksLog.conflict, RocksLog.java:199-216)
    ib = g.inbox(); ib.ae_request(0, 0, g.now, 1, 5, 9, 3, [4, 4], leader_commit=9); out = g.run(ib)
    assert rep(out)[:2] == (1, 1) and g.st.last_index == 11 and g.o.log_term(0, 10) == 4 and g.o.log_term(0, 9) == 3
    for bad in ([(2, 1), (8, 3)], [(1, 1), (4, 1), (8, 3)], [(1, 1), (4, 2)], [(1, 1), (12, 3)]):
        h = One(term=5, first_index=1, last_index=10, last_term=3)
        with pytest.raises(Exception):
            h.o.load_runs(0, bad)


# --------------------------------------------------------------------------------------------
# timers
# --------------------------------------------------------------------------------------------
def test_reset_timer_monotonic_guard_and_sweep():
    g = One(term=1, now_ms=T0, rand_ms=1000)
    assert g.st.timer == T0 + 1000
    g.now = T0 - 500                                       # clock went backwards: deadline must still advance by 1
    ae(g, 1, 1, 0, 0, rand=100)
    assert g.st.timer == g.now + 100                       # muted (MAX) resets the guard: max(0, now + timeout)
    # sweep row: not due -> nothing; due -> TIMEOUT with the counter-based draw
    ib = abi.Inbox(1, 1, 2, sweep=True); ib.row_now[0] = g.now + 50
    inc = g.st.incarnation
    g.run(ib)
    assert g.st.incarnation == inc
    ib = abi.Inbox(1, 1, 2, sweep=True); ib.row_now[0] = g.now + 100
    g.run(ib)
    s = g.st
    assert (s.incarnation, s.timeout_detected) == (inc + 1, 1)
    draw = binding.lib().orc_draw(g.cfg.timer_seed, 0, inc + 1, g.cfg.election_ms)
    assert 900 <= draw <= 1800 and s.timer == g.now + 100 + draw


# ---------------------------------------------------------------------------------------------------------------------
# upstream golden vectors (oracle/java/GoldenGen.java drives the reference's own, unmodified Leadership.State and
# Membership classes).  The build needs no JDK, so the vector file is
# produced by a maintainer with `make -C oracle/java`; until it is committed the replay test skips and parity stays
# "unpinned by upstream" (DESIGN.md §2).  The replay code itself is exercised on the one upstream table that exists in
# source form: the majority-position comment table, Leadership.java:120-126.
# ---------------------------------------------------------------------------------------------------------------------
UPSTREAM = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "upstream_leadership.json")
_OPS = {"statSuccess": 0, "statFailure": 1, "isReady": 2, "updateIndex": 3}


def replay_upstream(doc):
    """Replays a GoldenGen document through the oracle; returns the number of checks made."""
    import ctypes as C
    L = binding.lib()
    checks = 0
    for seq in doc.get("state", []):
        st = (C.c_int64 * 10)(*seq["init"])
        for call in seq["calls"]:
            name, args = call["c"][0], list(call["c"][1:])
            if name == "updateIndex":
                st[4] = args.pop()                     # recentRejection as the generator set it before the call
            a = (C.c_int64 * 4)(*(args + [0] * (4 - len(args))))
            ret = (C.c_int64 * 2)(0, 0)
            err = L.orc_state_apply(st, _OPS[name], a, ret)
            assert (err != 0) == (call["err"] != 0), (name, args, err)
            assert list(st) == call["s"], (name, args, list(st), call["s"])
            if call["r"] is not None:
                assert [ret[0], ret[1]] == call["r"], (name, args)
            checks += 1
    for m in doc.get("major", []):
        assert binding.major_indices(m["match"]) == (m["full"], m["major"]), m
        checks += 1
    for nr, nt, nb, cr, cb, want in doc.get("better", []):
        got = L.orc_is_better(nr, nt, nb, cr, 10, cb, 0)
        assert ("T" if got > 0 else "F" if got == 0 else "E") == want, (nr, nt, nb, cr, cb, got, want)
        checks += 1
    return checks


def test_upstream_replay_plumbing_on_the_source_comment_table():
    # Leadership.java:120-126: N = 2..7 nodes, position of the majority element among the N-1 sorted follower indices
    rows = []
    for n_nodes, major_pos in ((2, 0), (3, 1), (4, 1), (5, 2), (6, 2), (7, 3)):
        match = list(range(10, 10 + n_nodes - 1))
        rows.append({"match": match[::-1], "full": match[0], "major": match[major_pos]})
    doc = {"state": [{"init": [0, 0, 0, 0, 0, 0, 0, 8, 0, 0],
                      "calls": [{"c": ["statSuccess", 5, 0], "r": None, "err": 0, "s": [0, 5, 0, 0, 0, 0, 0, 8, 0, 0]},
                                {"c": ["updateIndex", 0, 7, 1, 0, 0], "r": None, "err": 0, "s": [0, 5, 0, 0, 0, 0, 0, 8, 7, 0]},
                                {"c": ["updateIndex", 0, 3, 1, 0, 0], "r": None, "err": 1, "s": [0, 5, 0, 0, 0, 0, 0, 8, 7, 0]},
                                {"c": ["isReady", 0, 0, 9], "r": [1, 0], "err": 0, "s": [0, 5, 0, 0, 0, 0, 0, 8, 7, 0]}]}],
           "major": rows, "better": [[2, 10, 0, 1, 0, "T"], [2, 10, 0, 0, 0, "E"], [1, 10, 0, 1, 1, "E"], [0, 9, 0, 0, 0, "F"]]}
    assert replay_upstream(doc) == 4 + 6 + 4


@pytest.mark.skipif(not os.path.exists(UPSTREAM), reason="tests/golden/upstream_leadership.json absent: no JDK here (make -C oracle/java)")
def test_upstream_golden_vectors():
    import json
    with open(UPSTREAM) as f:
        doc = json.load(f)
    assert replay_upstream(doc) > 6000
