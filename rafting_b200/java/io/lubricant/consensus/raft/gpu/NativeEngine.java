/*
 * NativeEngine.java — the Java half of the JNI boundary (glue: rafting_b200/csrc/jni/rafting_jni.c; C ABI: include/*.h).
 * Kept identical to the listing in INTEGRATION.md §1 and checked, native by native, against the glue's parameter lists by
 * tests/test_jni_glue_cpu.py (there is no JDK in this project's images, so this file is never compiled here).
 */
package io.lubricant.consensus.raft.gpu;

import java.nio.ByteBuffer;

/** Thin binding of the C ABI.  Every buffer is a direct ByteBuffer over memory the ENGINE owns (pinned). */
final class NativeEngine {
    static { System.loadLibrary("rafting_b200"); System.loadLibrary("rafting_jni"); }

    static native long create(ByteBuffer cfg);                                   // rafting_engine_create
    static native void destroy(long h);                                          // rafting_engine_destroy
    static native void groupOpen(long h, int gid, ByteBuffer init);              // rafting_group_open
    static native void groupClose(long h, int gid);                              // rafting_group_close
    static native void lease(long h, int rows, int nActive, int entCount, int flags, ByteBuffer leaseStruct);   // rafting_lease_ex
    static native ByteBuffer wrap(long address, long bytes);                     // view of one leased column
    static native void stepBegin(long h, ByteBuffer leaseStruct);                // rafting_step_begin
    static native void stepWait(long h, ByteBuffer leaseStruct);                 // rafting_step_wait
    static native void stateExport(long h, int gid, ByteBuffer out);             // rafting_state_export
    static native long logTerm(long h, int gid, long index);                     // rafting_log_term == RaftLog.get(i).term()
    static native void allgatherCommit(long h, ByteBuffer hostOut);              // rafting_allgather_commit
    // ---- round 2 ----
    static native void groupOpenBulk(long h, int first, int count, ByteBuffer inits);            // rafting_group_open_bulk
    static native void groupLoadRuns(long h, int gid, ByteBuffer runs, int n);                   // rafting_group_load_runs (restart, §4)
    static native void groupEditBegin(long h, ByteBuffer edits, int n);                          // rafting_group_edit_begin: opens / restarts / closes between steps
    static native void leaseRelease(long h, ByteBuffer leaseStruct);                             // rafting_lease_release
    static native void stepBeginHost(long h, int slot, ByteBuffer inboxStruct, ByteBuffer outboxStruct);   // rafting_step_begin_host: Netty's pinned receive pool
    static native void stepWaitSlot(long h, int slot);                                           // rafting_step_wait_slot
    static native void stepBeginCompact(long h, int slot, ByteBuffer cinbox, ByteBuffer coutbox); // rafting_step_begin_compact (§7)
    static native void stepBeginCompactReq(long h, int slot, ByteBuffer cinbox, ByteBuffer creqs, ByteBuffer coutbox);   // rafting_step_begin_compact_req: with inbound requests
    static native void stepBeginCompactEx(long h, int slot, ByteBuffer cinbox, ByteBuffer creqs, ByteBuffer coutbox, int flags);   // rafting_step_begin_compact_ex: RAFTING_COMPACT_ELECTIONS
    static native void stepBeginCompactActive(long h, int slot, int nActive, ByteBuffer gids, ByteBuffer cinbox, ByteBuffer creqs, ByteBuffer coutbox, int flags);   // rafting_step_begin_compact_active: over an active list
    static native void stepBeginCompactSweep(long h, int slot, int nActive, ByteBuffer gids, ByteBuffer sweep, ByteBuffer cinbox, ByteBuffer creqs, ByteBuffer coutbox, int flags);   // rafting_step_begin_compact_sweep: with sweep rows (timers)
    static native void stepBeginCompactDue(long h, int slot, int nHost, ByteBuffer gids, int cap, ByteBuffer sweep, ByteBuffer cinbox, ByteBuffer creqs, ByteBuffer coutbox, ByteBuffer tailOut, int flags);   // rafting_step_begin_compact_due: the device lists the due groups
    static native void timersDueBegin(long h, int slot, long untilMs, ByteBuffer gidsOut, int cap);   // rafting_timers_due_begin: the groups a sweep would fire
    static native void timersDueWait(long h, int slot, long[] nDueAndNextDeadline);              // rafting_timers_due_wait
    static native void stepWaitCompact(long h, int slot);                                        // rafting_step_wait_compact
    static native void stepFetchDense(long h, int slot, ByteBuffer outboxStruct);                // rafting_step_fetch_dense (escape overflow)
    static native void checkpoint(long h);                                                       // rafting_checkpoint
    static native void restore(long h);                                                          // rafting_restore
    static native void logConfig(long h, int segmentBytes, int hbmSegments, int ringSlots);      // rafting_log_config
    static native long logStoreOpen(long h, String path, int coldMaxSegments);                   // rafting_log_store_open (recovery)
    static native void logAppend(long h, ByteBuffer refs, int n, ByteBuffer blob, long blobBytes);   // rafting_log_append
    static native void logSync(long h);                                                          // rafting_log_sync: the step's flushWal(true)
    static native void logMark(long h, int gid, long lo, long hi, long epochIndex, long epochTerm);   // rafting_log_mark
    static native int  logRead(long h, int gid, long first, int maxN, ByteBuffer refsOut, ByteBuffer blobOut, long blobCap);   // RaftLog.batch
    static native int  logGather(long h, int nRanges, ByteBuffer gids, ByteBuffer firsts, ByteBuffer counts,
                                 ByteBuffer refsOut, int refsCap, ByteBuffer blobOut, long blobCap);  // the AE plans of a step at once
    static native void logGatherStepBegin(long h, int slot, ByteBuffer refsOut, int refsCap, ByteBuffer blobOut, long blobCap,
                                          ByteBuffer plansOut, int plansCap);                     // rafting_log_gather_step_begin: a step's AE payloads
    static native void logGatherStepWait(long h, int slot, long[] nRefsBytesNPlansHostServed);   // rafting_log_gather_step_wait
    static native void logGatherBegin(long h, int ticket, int nRanges, ByteBuffer gids, ByteBuffer firsts, ByteBuffer counts,
                                      ByteBuffer refsOut, int refsCap, ByteBuffer blobOut, long blobCap);   // rafting_log_gather_begin: ranges' payloads, async
    static native void logGatherWait(long h, int ticket, long[] nRefsBytesHostServed);           // rafting_log_gather_wait
    static native void logTrim(long h, int first, int count);                                    // rafting_log_trim (behind RaftLog.flush)
    static native int  logRecovered(long h, int gid, ByteBuffer initOut, ByteBuffer runsOut, int cap);   // rafting_log_recovered
    static native void commInitAll(long[] engines);                                              // rafting_comm_init_all: ONE JVM, n shards
    static native void commInit(long h, int rank, int world, ByteBuffer ncclUniqueId);           // rafting_comm_init: one process per GPU
    static native void allgatherCommitFrom(long h, long devColumn, ByteBuffer hostOut);          // rafting_allgather_commit_from
    static native long journalOpen(String dir, int maxGroups);                                   // rafting_journal_open (StableLock, batched)
    static native void journalClose(long j);
    static native long journalCommitStep(long j, ByteBuffer gids, int n, boolean compact, ByteBuffer roleWord, ByteBuffer currentTerm);
    static native void journalMilestone(long j, int gid, long index, long term);                 // StableLock.persist(Snapshot)
    static native void journalRestore(long j, int gid, ByteBuffer stableOut);                    // StableLock.restore()
    static native void journalCheckpoint(long j);
    static native int  frameScan(ByteBuffer buf, long len, ByteBuffer framesOut, int cap, ByteBuffer consumedTransparentRc);   // rafting_frame_scan
    static native long ctxmapCreate();                                                           // rafting_ctxmap_create: contextId -> gid registry
    static native void ctxmapPut(long m, String contextId, int gid);
    static native void ctxmapDestroy(long m);
    static native int  acksDecode(ByteBuffer buf, ByteBuffer frames, int n, long m, ByteBuffer ackRecsOut);   // rafting_ack_frames_decode: ACK frames -> (gid, kind, sequence, term, success)
    static native long pendingCreate(int capacityHint);                                          // (peer, sequence) -> gid, lane, tag, term, echo pair
    static native void pendingDestroy(long p);
    static native void pendingPut(long p, int peer, int sequence, int evKind, int gid, int lane, int tag, int incarnation, long term, long epochAtSend, long lastAtSend);
    static native void failuresToCinbox(long p, int peer, ByteBuffer sequences, int n, int outcome, long nowMs, int row, ByteBuffer cinStruct, int nGroups, int followers,
                                        ByteBuffer esc, int escCap, ByteBuffer deferredOut, ByteBuffer counters);   // Async time-outs / cancellations -> ev_c words
    static native void failuresToCinboxEx(long p, int peer, ByteBuffer sequences, int n, int outcome, long nowMs, int row, ByteBuffer cinStruct, int nGroups,
                                          int followers, ByteBuffer esc, int escCap, ByteBuffer deferredOut, ByteBuffer counters, int flags);   // the same for a flagged step
    static native boolean pendingRemove(long p, int peer, int sequence);                         // the invocation timed out
    static native void acksToCinbox(long p, int peer, ByteBuffer ackRecs, int n, long nowMs, int row, ByteBuffer cinStruct, int nGroups, int followers,
                                    ByteBuffer esc, int escCap, ByteBuffer deferredOut, ByteBuffer counters);   // replies -> ev_c words / escape records
    static native void acksToCinboxEx(long p, int peer, ByteBuffer ackRecs, int n, long nowMs, int row, ByteBuffer cinStruct, int nGroups, int followers,
                                      ByteBuffer esc, int escCap, ByteBuffer deferredOut, ByteBuffer counters, int flags);   // the same for a flagged step: vote words
    static native long builderCreate(int nGroups, int followers);                                // the event loops' queues: per-group FIFOs -> rows of a step
    static native void builderDestroy(long b);
    static native void builderPushSubmit(long b, int gid, int count, int unavailableMask);       // RaftStub.submit: to the FRONT of the group's queue
    static native void builderPushRequest(long b, ByteBuffer reqRec, ByteBuffer entryTerms);     // an inbound appendEntries / preVote / requestVote
    static native void builderPushReply(long b, ByteBuffer replyRec);                            // a reply (or a failed invocation) for one follower lane
    static native void builderClearGroup(long b, int gid);
    static native int  builderBuild(long b, long nowMs, ByteBuffer inStruct, int entCap, ByteBuffer placedOut, ByteBuffer placedRowOut, int placedCap, ByteBuffer counters);
    static native int  applyRanges(ByteBuffer outStruct, ByteBuffer gids, int n, ByteBuffer applied, int nGroups, ByteBuffer rangesOut, int cap);   // commit-dirty groups -> (gid, first, last)
    static native long dispatchCreate(int nGroups, int followers, int localSlot);                // engine-to-engine peers: the dispatch loop of §4 in C
    static native void dispatchDestroy(long d);
    static native int  outboxToRequests(long d, ByteBuffer outStruct, int rows, ByteBuffer reqRecsOut, int cap);   // plans + vote broadcasts -> 64 B request records
    static native int  coutboxToRequests(long d, ByteBuffer coutStruct, int rows, int flags, ByteBuffer reqRecsOut, ByteBuffer tagsOut, int cap);   // the same from a compact outbox, + the pending tag per record
    static native int  requestToInbox(ByteBuffer rec, ByteBuffer entryTerms, int row, long nowMs, boolean hostResult, ByteBuffer inStruct, int nGroups, int entCap, int entCount);
    static native int  outboxToReplies(ByteBuffer outStruct, int nGroups, int localSlot, ByteBuffer placed, ByteBuffer placedRow, int n, ByteBuffer replyRecsOut);
    static native void requestToCreq(ByteBuffer rec, ByteBuffer entryTerms, int row, long nowMs, boolean hostResult, ByteBuffer cinStruct, int nGroups,
                                     ByteBuffer creqsStruct, int reqCap, int escCap, int entCap);   // a request record -> the compact step's request list
    static native void requestToCreqEx(ByteBuffer rec, ByteBuffer entryTerms, int row, long nowMs, boolean hostResult, ByteBuffer cinStruct, int nGroups,
                                       ByteBuffer creqsStruct, int reqCap, int escCap, int entCap, int flags);   // the same for a flagged step: vote records
    static native int  coutboxToReplies(ByteBuffer coutStruct, int nGroups, int localSlot, ByteBuffer placed, ByteBuffer placedRow, int n, ByteBuffer replyRecsOut);
}
