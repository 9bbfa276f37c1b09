/*
 * rafting_jni.c — JNI glue between io.lubricant.consensus.raft.gpu.NativeEngine and the C ABI
 * (include/rafting_b200.h).  It only marshals DirectByteBuffer addresses; no protocol logic.
 *
 * NOT COMPILED IN THIS IMAGE: there is no JDK (no jni.h).  The whole file is guarded so that the
 * build never depends on it; on a box with a JDK:
 *   gcc -shared -fPIC -I$JAVA_HOME/include -I$JAVA_HOME/include/linux -Iinclude \
 *       rafting_b200/csrc/jni/rafting_jni.c -Lrafting_b200 -lrafting_b200 -lrafting_durable -lrafting_ingest -o librafting_jni.so
 * The Java side is shown in INTEGRATION.md.
 */
#if defined(__has_include)
#if __has_include(<jni.h>)
#define RAFTING_HAVE_JNI 1
#endif
#endif

#ifdef RAFTING_HAVE_JNI
#include <jni.h>
#include <string.h>

#include "../../../include/rafting_b200.h"
#include "../../../include/rafting_durable.h"
#include "../../../include/rafting_ingest.h"

#define FN(name) Java_io_lubricant_consensus_raft_gpu_NativeEngine_##name

static void throw_status(JNIEnv* env, int rc) {
    /* status codes map 1:1 onto the reference's exception types (SURVEY.md §8b) */
    const char* cls = rc == RAFTING_E_INVAL ? "java/lang/IllegalArgumentException"
                    : rc == RAFTING_E_CLOSED ? "java/lang/IllegalStateException"
                    : "io/lubricant/consensus/raft/support/RaftException";
    jclass c = (*env)->FindClass(env, cls);
    if (c) (*env)->ThrowNew(env, c, rafting_last_error());
}

JNIEXPORT jlong JNICALL FN(create)(JNIEnv* env, jclass k, jobject cfgBuf) {
    rafting_engine_t* e = NULL;
    const rafting_cfg_t* cfg = (const rafting_cfg_t*)(*env)->GetDirectBufferAddress(env, cfgBuf);
    int rc = rafting_engine_create(cfg, &e);
    if (rc) { throw_status(env, rc); return 0; }
    return (jlong)(intptr_t)e;
}
JNIEXPORT void JNICALL FN(destroy)(JNIEnv* env, jclass k, jlong h) { rafting_engine_destroy((rafting_engine_t*)(intptr_t)h); }

JNIEXPORT void JNICALL FN(groupOpen)(JNIEnv* env, jclass k, jlong h, jint gid, jobject initBuf) {
    int rc = rafting_group_open((rafting_engine_t*)(intptr_t)h, (uint32_t)gid,
                                (const rafting_group_init_t*)(*env)->GetDirectBufferAddress(env, initBuf));
    if (rc) throw_status(env, rc);
}
JNIEXPORT void JNICALL FN(groupClose)(JNIEnv* env, jclass k, jlong h, jint gid) {
    int rc = rafting_group_close((rafting_engine_t*)(intptr_t)h, (uint32_t)gid);
    if (rc) throw_status(env, rc);
}

/* lease: fills `leaseBuf` (a direct buffer of sizeof(rafting_lease_t)) and returns the pinned columns as
   DirectByteBuffers the pump thread writes events into — see NativeEngine.Lease in INTEGRATION.md */
JNIEXPORT void JNICALL FN(lease)(JNIEnv* env, jclass k, jlong h, jint rows, jint nActive, jint entCount, jint flags, jobject leaseBuf) {
    rafting_lease_t* L = (rafting_lease_t*)(*env)->GetDirectBufferAddress(env, leaseBuf);
    int rc = rafting_lease_ex((rafting_engine_t*)(intptr_t)h, (uint32_t)rows, (uint32_t)nActive, (uint32_t)entCount, (uint32_t)flags, L);
    if (rc) throw_status(env, rc);
}
JNIEXPORT jobject JNICALL FN(wrap)(JNIEnv* env, jclass k, jlong addr, jlong bytes) {
    return (*env)->NewDirectByteBuffer(env, (void*)(intptr_t)addr, bytes);
}
JNIEXPORT void JNICALL FN(stepBegin)(JNIEnv* env, jclass k, jlong h, jobject leaseBuf) {
    int rc = rafting_step_begin((rafting_engine_t*)(intptr_t)h, (rafting_lease_t*)(*env)->GetDirectBufferAddress(env, leaseBuf));
    if (rc) throw_status(env, rc);
}
JNIEXPORT void JNICALL FN(stepWait)(JNIEnv* env, jclass k, jlong h, jobject leaseBuf) {
    int rc = rafting_step_wait((rafting_engine_t*)(intptr_t)h, (rafting_lease_t*)(*env)->GetDirectBufferAddress(env, leaseBuf));
    if (rc) throw_status(env, rc);
}
JNIEXPORT void JNICALL FN(stateExport)(JNIEnv* env, jclass k, jlong h, jint gid, jobject outBuf) {
    int rc = rafting_state_export((rafting_engine_t*)(intptr_t)h, (uint32_t)gid,
                                  (rafting_group_state_t*)(*env)->GetDirectBufferAddress(env, outBuf));
    if (rc) throw_status(env, rc);
}
JNIEXPORT jlong JNICALL FN(logTerm)(JNIEnv* env, jclass k, jlong h, jint gid, jlong index) {
    int64_t t = -1;
    int rc = rafting_log_term((rafting_engine_t*)(intptr_t)h, (uint32_t)gid, index, &t);
    if (rc) throw_status(env, rc);
    return t;
}
JNIEXPORT void JNICALL FN(allgatherCommit)(JNIEnv* env, jclass k, jlong h, jobject hostOut) {
    int rc = rafting_allgather_commit((rafting_engine_t*)(intptr_t)h,
                                      hostOut ? (int64_t*)(*env)->GetDirectBufferAddress(env, hostOut) : NULL, NULL);
    if (rc) throw_status(env, rc);
}

/* ---- round 2: the rest of the surface INTEGRATION.md uses -------------------------------------------------------- */
#define ENG(h) ((rafting_engine_t*)(intptr_t)(h))
#define BUF(b) ((b) ? (*env)->GetDirectBufferAddress(env, (b)) : NULL)
#define CHECK(call) do { int rc_ = (call); if (rc_) throw_status(env, rc_); } while (0)

/* restart over a log that spans several terms (INTEGRATION.md §4 "Restart") */
JNIEXPORT void JNICALL FN(groupOpenBulk)(JNIEnv* env, jclass k, jlong h, jint first, jint count, jobject inits) {
    CHECK(rafting_group_open_bulk(ENG(h), (uint32_t)first, (uint32_t)count, (const rafting_group_init_t*)BUF(inits)));
}
JNIEXPORT void JNICALL FN(groupLoadRuns)(JNIEnv* env, jclass k, jlong h, jint gid, jobject runs, jint n) {
    CHECK(rafting_group_load_runs(ENG(h), (uint32_t)gid, (const rafting_i64x2_t*)BUF(runs), (uint32_t)n));
}
/* opens, restarts and closes as rafting_group_edit_t records, in step-stream order while steps are in flight (INTEGRATION.md §4) */
JNIEXPORT void JNICALL FN(groupEditBegin)(JNIEnv* env, jclass k, jlong h, jobject edits, jint n) {
    CHECK(rafting_group_edit_begin(ENG(h), (uint32_t)n, (const rafting_group_edit_t*)BUF(edits)));
}
JNIEXPORT void JNICALL FN(leaseRelease)(JNIEnv* env, jclass k, jlong h, jobject leaseBuf) {
    CHECK(rafting_lease_release(ENG(h), (rafting_lease_t*)BUF(leaseBuf)));
}
/* caller-owned pinned buffers (the transport's receive pool): rafting_inbox_t / rafting_outbox_t structs in direct buffers */
JNIEXPORT void JNICALL FN(stepBeginHost)(JNIEnv* env, jclass k, jlong h, jint slot, jobject inStruct, jobject outStruct) {
    CHECK(rafting_step_begin_host(ENG(h), (uint32_t)slot, (const rafting_inbox_t*)BUF(inStruct), (const rafting_outbox_t*)BUF(outStruct)));
}
JNIEXPORT void JNICALL FN(stepWaitSlot)(JNIEnv* env, jclass k, jlong h, jint slot) { CHECK(rafting_step_wait_slot(ENG(h), (uint32_t)slot)); }
/* the compact host path: rafting_cinbox_t / rafting_coutbox_t structs in direct buffers */
JNIEXPORT void JNICALL FN(stepBeginCompact)(JNIEnv* env, jclass k, jlong h, jint slot, jobject cin, jobject cout) {
    CHECK(rafting_step_begin_compact(ENG(h), (uint32_t)slot, (const rafting_cinbox_t*)BUF(cin), (const rafting_coutbox_t*)BUF(cout)));
}
/* ... with the inbound requests of the step (a rafting_creqs_t struct in a direct buffer; null = none, as stepBeginCompact) */
JNIEXPORT void JNICALL FN(stepBeginCompactReq)(JNIEnv* env, jclass k, jlong h, jint slot, jobject cin, jobject creqs, jobject cout) {
    CHECK(rafting_step_begin_compact_req(ENG(h), (uint32_t)slot, (const rafting_cinbox_t*)BUF(cin), (const rafting_creqs_t*)BUF(creqs),
                                         (const rafting_coutbox_t*)BUF(cout)));
}
/* the same with RAFTING_COMPACT_ELECTIONS (or 0) in flags: ballots, vote replies and vote requests travel compact */
JNIEXPORT void JNICALL FN(stepBeginCompactEx)(JNIEnv* env, jclass k, jlong h, jint slot, jobject cin, jobject creqs, jobject cout, jint flags) {
    CHECK(rafting_step_begin_compact_ex(ENG(h), (uint32_t)slot, (const rafting_cinbox_t*)BUF(cin), (const rafting_creqs_t*)BUF(creqs),
                                        (const rafting_coutbox_t*)BUF(cout), (uint32_t)flags));
}
/* ... over an active list: nActive uint32 gids in a direct buffer, every column of cinbox / coutbox sized by nActive */
JNIEXPORT void JNICALL FN(stepBeginCompactActive)(JNIEnv* env, jclass k, jlong h, jint slot, jint nActive, jobject gids, jobject cin, jobject creqs,
                                                  jobject cout, jint flags) {
    CHECK(rafting_step_begin_compact_active(ENG(h), (uint32_t)slot, (uint32_t)nActive, (const uint32_t*)BUF(gids), (const rafting_cinbox_t*)BUF(cin),
                                            (const rafting_creqs_t*)BUF(creqs), (const rafting_coutbox_t*)BUF(cout), (uint32_t)flags));
}
/* ... with sweep rows: `sweep` holds rows int64 sweep times (0 = not a sweep row); gids null = the whole shard */
JNIEXPORT void JNICALL FN(stepBeginCompactSweep)(JNIEnv* env, jclass k, jlong h, jint slot, jint nActive, jobject gids, jobject sweep, jobject cin,
                                                 jobject creqs, jobject cout, jint flags) {
    CHECK(rafting_step_begin_compact_sweep(ENG(h), (uint32_t)slot, (uint32_t)nActive, (const uint32_t*)BUF(gids), (const int64_t*)BUF(sweep),
                                           (const rafting_cinbox_t*)BUF(cin), (const rafting_creqs_t*)BUF(creqs), (const rafting_coutbox_t*)BUF(cout),
                                           (uint32_t)flags));
}
/* ... over nHost listed gids (null when nHost = 0) and a tail of cap gids chosen on the device: every column of cinbox /
   coutbox sized by nHost + cap; tailOut (cap uint32, direct) receives the tail at stepWaitCompact, coutbox counts[3] the
   number of due groups outside the list */
JNIEXPORT void JNICALL FN(stepBeginCompactDue)(JNIEnv* env, jclass k, jlong h, jint slot, jint nHost, jobject gids, jint cap, jobject sweep,
                                               jobject cin, jobject creqs, jobject cout, jobject tailOut, jint flags) {
    CHECK(rafting_step_begin_compact_due(ENG(h), (uint32_t)slot, (uint32_t)nHost, (const uint32_t*)BUF(gids), (uint32_t)cap,
                                         (const int64_t*)BUF(sweep), (const rafting_cinbox_t*)BUF(cin), (const rafting_creqs_t*)BUF(creqs),
                                         (const rafting_coutbox_t*)BUF(cout), (uint32_t*)BUF(tailOut), (uint32_t)flags));
}
JNIEXPORT void JNICALL FN(stepWaitCompact)(JNIEnv* env, jclass k, jlong h, jint slot) { CHECK(rafting_step_wait_compact(ENG(h), (uint32_t)slot)); }
/* the groups a sweep at untilMs would fire: gidsOut (cap uint32) is filled at the wait; result = {nDue, nextDeadlineMs} */
JNIEXPORT void JNICALL FN(timersDueBegin)(JNIEnv* env, jclass k, jlong h, jint slot, jlong untilMs, jobject gidsOut, jint cap) {
    CHECK(rafting_timers_due_begin(ENG(h), (uint32_t)slot, (int64_t)untilMs, (uint32_t*)BUF(gidsOut), (uint32_t)cap));
}
JNIEXPORT void JNICALL FN(timersDueWait)(JNIEnv* env, jclass k, jlong h, jint slot, jlongArray result) {
    uint32_t n = 0; int64_t next = 0;
    int rc = rafting_timers_due_wait(ENG(h), (uint32_t)slot, &n, &next);
    if (rc) { throw_status(env, rc); return; }
    if (!result || (*env)->GetArrayLength(env, result) < 2) {
        jclass c = (*env)->FindClass(env, "java/lang/IllegalArgumentException");
        if (c) (*env)->ThrowNew(env, c, "timersDueWait: the result array needs 2 elements {nDue, nextDeadlineMs}");
        return;
    }
    jlong* r = (*env)->GetLongArrayElements(env, result, NULL);
    r[0] = (jlong)n; r[1] = (jlong)next;
    (*env)->ReleaseLongArrayElements(env, result, r, 0);
}
JNIEXPORT void JNICALL FN(stepFetchDense)(JNIEnv* env, jclass k, jlong h, jint slot, jobject outStruct) {
    CHECK(rafting_step_fetch_dense(ENG(h), (uint32_t)slot, (const rafting_outbox_t*)BUF(outStruct)));
}
JNIEXPORT void JNICALL FN(checkpoint)(JNIEnv* env, jclass k, jlong h) { CHECK(rafting_checkpoint(ENG(h))); }
JNIEXPORT void JNICALL FN(restore)(JNIEnv* env, jclass k, jlong h) { CHECK(rafting_restore(ENG(h))); }

/* payload side of RaftLog (GpuRaftLog, INTEGRATION.md §5) */
JNIEXPORT void JNICALL FN(logConfig)(JNIEnv* env, jclass k, jlong h, jint segBytes, jint hbmSegments, jint ringSlots) {
    CHECK(rafting_log_config(ENG(h), (uint32_t)segBytes, (uint32_t)hbmSegments, (uint32_t)ringSlots));
}
JNIEXPORT jlong JNICALL FN(logStoreOpen)(JNIEnv* env, jclass k, jlong h, jstring path, jint coldMax) {
    const char* p = (*env)->GetStringUTFChars(env, path, NULL);
    uint64_t n = 0;
    int rc = rafting_log_store_open(ENG(h), p, (uint32_t)coldMax, &n);
    (*env)->ReleaseStringUTFChars(env, path, p);
    if (rc) throw_status(env, rc);
    return (jlong)n;
}
JNIEXPORT void JNICALL FN(logAppend)(JNIEnv* env, jclass k, jlong h, jobject refs, jint n, jobject blob, jlong blobBytes) {
    CHECK(rafting_log_append(ENG(h), (const rafting_entry_ref_t*)BUF(refs), (uint32_t)n, BUF(blob), (size_t)blobBytes));
}
JNIEXPORT void JNICALL FN(logSync)(JNIEnv* env, jclass k, jlong h) { CHECK(rafting_log_sync(ENG(h))); }
JNIEXPORT void JNICALL FN(logMark)(JNIEnv* env, jclass k, jlong h, jint gid, jlong lo, jlong hi, jlong epochIndex, jlong epochTerm) {
    CHECK(rafting_log_mark(ENG(h), (uint32_t)gid, lo, hi, epochIndex, epochTerm));
}
JNIEXPORT jint JNICALL FN(logRead)(JNIEnv* env, jclass k, jlong h, jint gid, jlong first, jint maxN, jobject refsOut, jobject blobOut, jlong blobCap) {
    uint32_t n = 0;
    CHECK(rafting_log_read(ENG(h), (uint32_t)gid, first, (uint32_t)maxN, (rafting_entry_ref_t*)BUF(refsOut), BUF(blobOut), (size_t)blobCap, &n));
    return (jint)n;
}
JNIEXPORT jint JNICALL FN(logGather)(JNIEnv* env, jclass k, jlong h, jint nRanges, jobject gids, jobject firsts, jobject counts,
                                     jobject refsOut, jint refsCap, jobject blobOut, jlong blobCap) {
    uint32_t n = 0; size_t bytes = 0;
    CHECK(rafting_log_gather(ENG(h), (uint32_t)nRanges, (const uint32_t*)BUF(gids), (const int64_t*)BUF(firsts), (const uint32_t*)BUF(counts),
                             (rafting_entry_ref_t*)BUF(refsOut), (uint32_t)refsCap, BUF(blobOut), (size_t)blobCap, &n, &bytes));
    return (jint)n;
}
/* the payloads of the AppendEntries plans of the compact step last waited for in `slot`, gathered on the device (INTEGRATION.md §7) */
JNIEXPORT void JNICALL FN(logGatherStepBegin)(JNIEnv* env, jclass k, jlong h, jint slot, jobject refsOut, jint refsCap, jobject blobOut,
                                              jlong blobCap, jobject plansOut, jint plansCap) {
    CHECK(rafting_log_gather_step_begin(ENG(h), (uint32_t)slot, (rafting_entry_ref_t*)BUF(refsOut), (uint32_t)refsCap, BUF(blobOut),
                                        (size_t)blobCap, (rafting_plan_ref_t*)BUF(plansOut), (uint32_t)plansCap));
}
/* result = {nRefs, bytes, nPlans, hostServed}; they are written before RAFTING_E_CAPACITY is thrown, as the sizes needed */
JNIEXPORT void JNICALL FN(logGatherStepWait)(JNIEnv* env, jclass k, jlong h, jint slot, jlongArray result) {
    if (!result || (*env)->GetArrayLength(env, result) < 4) {
        jclass c = (*env)->FindClass(env, "java/lang/IllegalArgumentException");
        if (c) (*env)->ThrowNew(env, c, "logGatherStepWait: the result array needs 4 elements {nRefs, bytes, nPlans, hostServed}");
        return;
    }
    uint32_t n = 0, plans = 0, served = 0; size_t bytes = 0;
    int rc = rafting_log_gather_step_wait(ENG(h), (uint32_t)slot, &n, &bytes, &plans, &served);
    jlong* r = (*env)->GetLongArrayElements(env, result, NULL);
    r[0] = (jlong)n; r[1] = (jlong)bytes; r[2] = (jlong)plans; r[3] = (jlong)served;
    (*env)->ReleaseLongArrayElements(env, result, r, 0);
    if (rc) throw_status(env, rc);
}
/* the payloads of (gid, first, count) ranges, e.g. a step's apply ranges, gathered on the device under `ticket` (INTEGRATION.md §7) */
JNIEXPORT void JNICALL FN(logGatherBegin)(JNIEnv* env, jclass k, jlong h, jint ticket, jint nRanges, jobject gids, jobject firsts,
                                          jobject counts, jobject refsOut, jint refsCap, jobject blobOut, jlong blobCap) {
    CHECK(rafting_log_gather_begin(ENG(h), (uint32_t)ticket, (uint32_t)nRanges, (const uint32_t*)BUF(gids), (const int64_t*)BUF(firsts),
                                   (const uint32_t*)BUF(counts), (rafting_entry_ref_t*)BUF(refsOut), (uint32_t)refsCap, BUF(blobOut),
                                   (size_t)blobCap));
}
/* result = {nRefs, bytes, hostServed}; they are written before RAFTING_E_CAPACITY is thrown, bytes as the bytes needed */
JNIEXPORT void JNICALL FN(logGatherWait)(JNIEnv* env, jclass k, jlong h, jint ticket, jlongArray result) {
    if (!result || (*env)->GetArrayLength(env, result) < 3) {
        jclass c = (*env)->FindClass(env, "java/lang/IllegalArgumentException");
        if (c) (*env)->ThrowNew(env, c, "logGatherWait: the result array needs 3 elements {nRefs, bytes, hostServed}");
        return;
    }
    uint32_t n = 0, served = 0; size_t bytes = 0;
    int rc = rafting_log_gather_wait(ENG(h), (uint32_t)ticket, &n, &bytes, &served);
    jlong* r = (*env)->GetLongArrayElements(env, result, NULL);
    r[0] = (jlong)n; r[1] = (jlong)bytes; r[2] = (jlong)served;
    (*env)->ReleaseLongArrayElements(env, result, r, 0);
    if (rc) throw_status(env, rc);
}
JNIEXPORT void JNICALL FN(logTrim)(JNIEnv* env, jclass k, jlong h, jint first, jint count) {
    CHECK(rafting_log_trim(ENG(h), (uint32_t)first, (uint32_t)count, NULL, NULL));
}
JNIEXPORT jint JNICALL FN(logRecovered)(JNIEnv* env, jclass k, jlong h, jint gid, jobject initOut, jobject runsOut, jint cap) {
    uint32_t n = 0;
    CHECK(rafting_log_recovered(ENG(h), (uint32_t)gid, (rafting_group_init_t*)BUF(initOut), (rafting_i64x2_t*)BUF(runsOut), (uint32_t)cap, &n));
    return (jint)n;
}

/* ONE JVM owning several shards (ContextManager.java:46): engines[r] becomes rank r of one communicator */
JNIEXPORT void JNICALL FN(commInitAll)(JNIEnv* env, jclass k, jlongArray handles) {
    const jsize n = (*env)->GetArrayLength(env, handles);
    jlong* hs = (*env)->GetLongArrayElements(env, handles, NULL);
    rafting_engine_t* es[64];
    for (jsize r = 0; r < n && r < 64; r++) es[r] = ENG(hs[r]);
    int rc = n <= 64 ? rafting_comm_init_all(es, (int)n) : RAFTING_E_CAPACITY;
    (*env)->ReleaseLongArrayElements(env, handles, hs, JNI_ABORT);
    if (rc) throw_status(env, rc);
}
JNIEXPORT void JNICALL FN(commInit)(JNIEnv* env, jclass k, jlong h, jint rank, jint world, jobject uid) {
    CHECK(rafting_comm_init(ENG(h), (int)rank, (int)world, BUF(uid), uid ? (size_t)(*env)->GetDirectBufferCapacity(env, uid) : 0));
}
JNIEXPORT void JNICALL FN(allgatherCommitFrom)(JNIEnv* env, jclass k, jlong h, jlong devSrc, jobject hostOut) {
    CHECK(rafting_allgather_commit_from(ENG(h), (const int64_t*)(intptr_t)devSrc, (int64_t*)BUF(hostOut), NULL));
}

/* the stable-storage journal: RaftFactory.restoreContext's StableLock (RaftFactory.java:18-36) becomes one journal per shard */
JNIEXPORT jlong JNICALL FN(journalOpen)(JNIEnv* env, jclass k, jstring dir, jint maxGroups) {
    const char* d = (*env)->GetStringUTFChars(env, dir, NULL);
    rafting_journal_t* j = NULL;
    int rc = rafting_journal_open(d, (uint32_t)maxGroups, &j);
    (*env)->ReleaseStringUTFChars(env, dir, d);
    if (rc) { jclass c = (*env)->FindClass(env, "java/io/IOException"); if (c) (*env)->ThrowNew(env, c, rafting_durable_last_error()); return 0; }
    return (jlong)(intptr_t)j;
}
JNIEXPORT void JNICALL FN(journalClose)(JNIEnv* env, jclass k, jlong j) { rafting_journal_close((rafting_journal_t*)(intptr_t)j); }
JNIEXPORT jlong JNICALL FN(journalCommitStep)(JNIEnv* env, jclass k, jlong j, jobject gids, jint n, jboolean compact, jobject roleWord, jobject currentTerm) {
    uint64_t recs = 0;
    int rc = rafting_journal_commit_step((rafting_journal_t*)(intptr_t)j, (const uint32_t*)BUF(gids), (uint32_t)n, compact ? 1 : 0,
                                         (const uint32_t*)BUF(roleWord), (const int64_t*)BUF(currentTerm), &recs);
    if (rc) { jclass c = (*env)->FindClass(env, "java/io/IOException"); if (c) (*env)->ThrowNew(env, c, rafting_durable_last_error()); }
    return (jlong)recs;
}
JNIEXPORT void JNICALL FN(journalMilestone)(JNIEnv* env, jclass k, jlong j, jint gid, jlong index, jlong term) {
    if (rafting_journal_milestone((rafting_journal_t*)(intptr_t)j, (uint32_t)gid, index, term)) {
        jclass c = (*env)->FindClass(env, "java/io/IOException"); if (c) (*env)->ThrowNew(env, c, rafting_durable_last_error());
    }
}
JNIEXPORT void JNICALL FN(journalRestore)(JNIEnv* env, jclass k, jlong j, jint gid, jobject stableOut) {
    rafting_journal_restore((rafting_journal_t*)(intptr_t)j, (uint32_t)gid, (rafting_stable_t*)BUF(stableOut));
}
JNIEXPORT void JNICALL FN(journalCheckpoint)(JNIEnv* env, jclass k, jlong j) {
    if (rafting_journal_checkpoint((rafting_journal_t*)(intptr_t)j)) {
        jclass c = (*env)->FindClass(env, "java/io/IOException"); if (c) (*env)->ThrowNew(env, c, rafting_durable_last_error());
    }
}

/* transport framing (include/rafting_ingest.h): cut a receive buffer into frames without one object per frame */
JNIEXPORT jint JNICALL FN(frameScan)(JNIEnv* env, jclass k, jobject buf, jlong len, jobject framesOut, jint cap, jobject consumedAndFlags) {
    uint32_t n = 0; size_t used = 0; int transparent = 0;
    int rc = rafting_frame_scan((const uint8_t*)BUF(buf), (size_t)len, (rafting_frame_t*)BUF(framesOut), (uint32_t)cap, &n, &used, &transparent);
    int64_t* o = (int64_t*)BUF(consumedAndFlags);
    if (o) { o[0] = (int64_t)used; o[1] = transparent; o[2] = rc; }
    return (jint)n;
}
/* contextId -> gid registry + the reply bodies of a scanned buffer (RaftResponse, Kryo) without one object per frame */
JNIEXPORT jlong JNICALL FN(ctxmapCreate)(JNIEnv* env, jclass k) {
    rafting_ctxmap_t* m = NULL;
    CHECK(rafting_ctxmap_create(&m));
    return (jlong)(intptr_t)m;
}
JNIEXPORT void JNICALL FN(ctxmapPut)(JNIEnv* env, jclass k, jlong m, jstring contextId, jint gid) {
    const char* c = (*env)->GetStringUTFChars(env, contextId, NULL);
    int rc = c ? rafting_ctxmap_put((rafting_ctxmap_t*)(intptr_t)m, c, (uint32_t)strlen(c), (uint32_t)gid) : RAFTING_E_NOMEM;
    if (c) (*env)->ReleaseStringUTFChars(env, contextId, c);
    if (rc) throw_status(env, rc);
}
JNIEXPORT void JNICALL FN(ctxmapDestroy)(JNIEnv* env, jclass k, jlong m) { rafting_ctxmap_destroy((rafting_ctxmap_t*)(intptr_t)m); }
JNIEXPORT jint JNICALL FN(acksDecode)(JNIEnv* env, jclass k, jobject buf, jobject frames, jint n, jlong m, jobject ackRecsOut) {
    uint32_t got = 0;
    CHECK(rafting_ack_frames_decode((const uint8_t*)BUF(buf), (const rafting_frame_t*)BUF(frames), (uint32_t)n,
                                    (const rafting_ctxmap_t*)(intptr_t)m, (rafting_ack_rec_t*)BUF(ackRecsOut), &got));
    return (jint)got;
}
/* engine-to-engine traffic: the pump's dispatch loop in C (one request / reply batch per peer and step, include/rafting_ingest.h) */
JNIEXPORT jlong JNICALL FN(dispatchCreate)(JNIEnv* env, jclass k, jint nGroups, jint followers, jint localSlot) {
    rafting_dispatch_t* d = NULL;
    CHECK(rafting_dispatch_create((uint32_t)nGroups, (uint32_t)followers, (uint32_t)localSlot, &d));
    return (jlong)(intptr_t)d;
}
JNIEXPORT void JNICALL FN(dispatchDestroy)(JNIEnv* env, jclass k, jlong d) { rafting_dispatch_destroy((rafting_dispatch_t*)(intptr_t)d); }
JNIEXPORT jint JNICALL FN(outboxToRequests)(JNIEnv* env, jclass k, jlong d, jobject outStruct, jint rows, jobject recsOut, jint cap) {
    uint32_t n = 0, unknown = 0;
    CHECK(rafting_outbox_to_requests((rafting_dispatch_t*)(intptr_t)d, (const rafting_outbox_t*)BUF(outStruct), (uint32_t)rows,
                                     (rafting_req_rec_t*)BUF(recsOut), (uint32_t)cap, &n, &unknown));
    return (jint)n;
}
/* the same over a waited-for compact outbox of a step begun with `flags`; tagsOut gets the pending entry's tag per record */
JNIEXPORT jint JNICALL FN(coutboxToRequests)(JNIEnv* env, jclass k, jlong d, jobject coutStruct, jint rows, jint flags, jobject recsOut,
                                             jobject tagsOut, jint cap) {
    uint32_t n = 0, unknown = 0;
    CHECK(rafting_coutbox_to_requests((rafting_dispatch_t*)(intptr_t)d, (const rafting_coutbox_t*)BUF(coutStruct), (uint32_t)rows,
                                      (uint32_t)flags, (rafting_req_rec_t*)BUF(recsOut), (uint8_t*)BUF(tagsOut), (uint32_t)cap, &n, &unknown));
    return (jint)n;
}
JNIEXPORT jint JNICALL FN(requestToInbox)(JNIEnv* env, jclass k, jobject rec, jobject entryTerms, jint row, jlong nowMs, jboolean hostResult,
                                          jobject inStruct, jint nGroups, jint entCap, jint entCount) {
    uint32_t cnt = (uint32_t)entCount;
    CHECK(rafting_request_to_inbox((const rafting_req_rec_t*)BUF(rec), (const int64_t*)BUF(entryTerms), (uint32_t)row, nowMs,
                                   hostResult ? 1 : 0, (const rafting_inbox_t*)BUF(inStruct), (uint32_t)nGroups, (uint32_t)entCap, &cnt));
    return (jint)cnt;                                       /* the pool's new fill level */
}
JNIEXPORT jint JNICALL FN(outboxToReplies)(JNIEnv* env, jclass k, jobject outStruct, jint nGroups, jint localSlot, jobject placed,
                                           jobject placedRow, jint n, jobject repliesOut) {
    uint32_t got = 0;
    CHECK(rafting_outbox_to_replies((const rafting_outbox_t*)BUF(outStruct), (uint32_t)nGroups, (uint32_t)localSlot,
                                    (const rafting_req_rec_t*)BUF(placed), (const uint8_t*)BUF(placedRow), (uint32_t)n,
                                    (rafting_batch_rec_t*)BUF(repliesOut), &got));
    return (jint)got;
}
/* the same two ends for the compact host path: a record into the step's request list (its counts grow in the struct), and
   the replies of a waited-for compact outbox */
JNIEXPORT void JNICALL FN(requestToCreq)(JNIEnv* env, jclass k, jobject rec, jobject entryTerms, jint row, jlong nowMs, jboolean hostResult,
                                         jobject cinStruct, jint nGroups, jobject creqsStruct, jint reqCap, jint escCap, jint entCap) {
    CHECK(rafting_request_to_creq((const rafting_req_rec_t*)BUF(rec), (const int64_t*)BUF(entryTerms), (uint32_t)row, nowMs, hostResult ? 1 : 0,
                                  (const rafting_cinbox_t*)BUF(cinStruct), (uint32_t)nGroups, (rafting_creqs_t*)BUF(creqsStruct),
                                  (uint32_t)reqCap, (uint32_t)escCap, (uint32_t)entCap));
}
JNIEXPORT void JNICALL FN(requestToCreqEx)(JNIEnv* env, jclass k, jobject rec, jobject entryTerms, jint row, jlong nowMs, jboolean hostResult,
                                           jobject cinStruct, jint nGroups, jobject creqsStruct, jint reqCap, jint escCap, jint entCap, jint flags) {
    CHECK(rafting_request_to_creq_ex((const rafting_req_rec_t*)BUF(rec), (const int64_t*)BUF(entryTerms), (uint32_t)row, nowMs, hostResult ? 1 : 0,
                                     (const rafting_cinbox_t*)BUF(cinStruct), (uint32_t)nGroups, (rafting_creqs_t*)BUF(creqsStruct),
                                     (uint32_t)reqCap, (uint32_t)escCap, (uint32_t)entCap, (uint32_t)flags));
}
JNIEXPORT jint JNICALL FN(coutboxToReplies)(JNIEnv* env, jclass k, jobject coutStruct, jint nGroups, jint localSlot, jobject placed,
                                            jobject placedRow, jint n, jobject repliesOut) {
    uint32_t got = 0;
    CHECK(rafting_coutbox_to_replies((const rafting_coutbox_t*)BUF(coutStruct), (uint32_t)nGroups, (uint32_t)localSlot,
                                     (const rafting_req_rec_t*)BUF(placed), (const uint8_t*)BUF(placedRow), (uint32_t)n,
                                     (rafting_batch_rec_t*)BUF(repliesOut), &got));
    return (jint)got;
}
/* commit records of a step -> (gid, first, last) ranges for RaftMachine.apply; `applied` is the pump's long[G] in a direct buffer */
JNIEXPORT jint JNICALL FN(applyRanges)(JNIEnv* env, jclass k, jobject outStruct, jobject gids, jint n, jobject applied, jint nGroups,
                                       jobject rangesOut, jint cap) {
    uint32_t got = 0;
    CHECK(rafting_outbox_apply_ranges((const rafting_outbox_t*)BUF(outStruct), (const uint32_t*)BUF(gids), (uint32_t)n, (int64_t*)BUF(applied),
                                      (uint32_t)nGroups, (rafting_apply_rec_t*)BUF(rangesOut), (uint32_t)cap, &got));
    return (jint)got;
}
/* the pending-invocation table + replies -> compact wire words (what NettyNode.getInvocationIfPresent + the AE-Echo closure do per ack) */
JNIEXPORT jlong JNICALL FN(pendingCreate)(JNIEnv* env, jclass k, jint capacityHint) {
    rafting_pending_t* p = NULL;
    CHECK(rafting_pending_create((uint32_t)capacityHint, &p));
    return (jlong)(intptr_t)p;
}
JNIEXPORT void JNICALL FN(pendingDestroy)(JNIEnv* env, jclass k, jlong p) { rafting_pending_destroy((rafting_pending_t*)(intptr_t)p); }
JNIEXPORT void JNICALL FN(pendingPut)(JNIEnv* env, jclass k, jlong p, jint peer, jint sequence, jint evKind, jint gid, jint lane, jint tag,
                                      jint incarnation, jlong term, jlong epochAtSend, jlong lastAtSend) {
    CHECK(rafting_pending_put((rafting_pending_t*)(intptr_t)p, (uint32_t)peer, sequence, (uint32_t)evKind, (uint32_t)gid, (uint32_t)lane,
                              (uint32_t)tag, (uint32_t)incarnation, term, epochAtSend, lastAtSend));
}
/* timed-out / cancelled invocations -> the same row; counters as in acksToCinbox */
JNIEXPORT void JNICALL FN(failuresToCinbox)(JNIEnv* env, jclass k, jlong p, jint peer, jobject sequences, jint n, jint outcome, jlong nowMs, jint row,
                                            jobject cinStruct, jint nGroups, jint followers, jobject esc, jint escCap, jobject deferredOut,
                                            jobject counters) {
    int64_t* c = (int64_t*)BUF(counters);
    uint32_t nEsc = c ? (uint32_t)c[0] : 0, nDef = 0, nUnknown = 0;
    int rc = rafting_failures_to_cinbox((rafting_pending_t*)(intptr_t)p, (uint32_t)peer, (const int32_t*)BUF(sequences), (uint32_t)n,
                                        (uint32_t)outcome, nowMs, (uint32_t)row, (const rafting_cinbox_t*)BUF(cinStruct), (uint32_t)nGroups,
                                        (uint32_t)followers, (rafting_cesc_in_t*)BUF(esc), (uint32_t)escCap, &nEsc, (uint32_t*)BUF(deferredOut),
                                        &nDef, &nUnknown);
    if (c) { c[0] = nEsc; c[1] = nDef; c[2] = nUnknown; }
    if (rc) throw_status(env, rc);
}
JNIEXPORT void JNICALL FN(failuresToCinboxEx)(JNIEnv* env, jclass k, jlong p, jint peer, jobject sequences, jint n, jint outcome, jlong nowMs,
                                              jint row, jobject cinStruct, jint nGroups, jint followers, jobject esc, jint escCap,
                                              jobject deferredOut, jobject counters, jint flags) {
    int64_t* c = (int64_t*)BUF(counters);
    uint32_t nEsc = c ? (uint32_t)c[0] : 0, nDef = 0, nUnknown = 0;
    int rc = rafting_failures_to_cinbox_ex((rafting_pending_t*)(intptr_t)p, (uint32_t)peer, (const int32_t*)BUF(sequences), (uint32_t)n,
                                           (uint32_t)outcome, nowMs, (uint32_t)row, (const rafting_cinbox_t*)BUF(cinStruct), (uint32_t)nGroups,
                                           (uint32_t)followers, (rafting_cesc_in_t*)BUF(esc), (uint32_t)escCap, &nEsc, (uint32_t*)BUF(deferredOut),
                                           &nDef, &nUnknown, (uint32_t)flags);
    if (c) { c[0] = nEsc; c[1] = nDef; c[2] = nUnknown; }
    if (rc) throw_status(env, rc);
}
JNIEXPORT jboolean JNICALL FN(pendingRemove)(JNIEnv* env, jclass k, jlong p, jint peer, jint sequence) {
    return rafting_pending_remove((rafting_pending_t*)(intptr_t)p, (uint32_t)peer, sequence) == RAFTING_OK;
}
/* counters: long[3] in a direct buffer = { escape records used (in/out), deferred acks, unknown sequences } */
JNIEXPORT void JNICALL FN(acksToCinbox)(JNIEnv* env, jclass k, jlong p, jint peer, jobject acks, jint n, jlong nowMs, jint row, jobject cinStruct,
                                        jint nGroups, jint followers, jobject esc, jint escCap, jobject deferredOut, jobject counters) {
    int64_t* c = (int64_t*)BUF(counters);
    uint32_t nEsc = c ? (uint32_t)c[0] : 0, nDef = 0, nUnknown = 0;
    int rc = rafting_acks_to_cinbox((rafting_pending_t*)(intptr_t)p, (uint32_t)peer, (const rafting_ack_rec_t*)BUF(acks), (uint32_t)n, nowMs,
                                    (uint32_t)row, (const rafting_cinbox_t*)BUF(cinStruct), (uint32_t)nGroups, (uint32_t)followers,
                                    (rafting_cesc_in_t*)BUF(esc), (uint32_t)escCap, &nEsc, (uint32_t*)BUF(deferredOut), &nDef, &nUnknown);
    if (c) { c[0] = nEsc; c[1] = nDef; c[2] = nUnknown; }
    if (rc) throw_status(env, rc);
}
JNIEXPORT void JNICALL FN(acksToCinboxEx)(JNIEnv* env, jclass k, jlong p, jint peer, jobject acks, jint n, jlong nowMs, jint row, jobject cinStruct,
                                          jint nGroups, jint followers, jobject esc, jint escCap, jobject deferredOut, jobject counters, jint flags) {
    int64_t* c = (int64_t*)BUF(counters);
    uint32_t nEsc = c ? (uint32_t)c[0] : 0, nDef = 0, nUnknown = 0;
    int rc = rafting_acks_to_cinbox_ex((rafting_pending_t*)(intptr_t)p, (uint32_t)peer, (const rafting_ack_rec_t*)BUF(acks), (uint32_t)n, nowMs,
                                       (uint32_t)row, (const rafting_cinbox_t*)BUF(cinStruct), (uint32_t)nGroups, (uint32_t)followers,
                                       (rafting_cesc_in_t*)BUF(esc), (uint32_t)escCap, &nEsc, (uint32_t*)BUF(deferredOut), &nDef, &nUnknown,
                                       (uint32_t)flags);
    if (c) { c[0] = nEsc; c[1] = nDef; c[2] = nUnknown; }
    if (rc) throw_status(env, rc);
}
/* the inbox builder: per-group FIFOs of requests / replies / submits -> the rows of one dense step */
JNIEXPORT jlong JNICALL FN(builderCreate)(JNIEnv* env, jclass k, jint nGroups, jint followers) {
    rafting_builder_t* b = NULL;
    CHECK(rafting_builder_create((uint32_t)nGroups, (uint32_t)followers, &b));
    return (jlong)(intptr_t)b;
}
JNIEXPORT void JNICALL FN(builderDestroy)(JNIEnv* env, jclass k, jlong b) { rafting_builder_destroy((rafting_builder_t*)(intptr_t)b); }
JNIEXPORT void JNICALL FN(builderPushSubmit)(JNIEnv* env, jclass k, jlong b, jint gid, jint count, jint unavailableMask) {
    CHECK(rafting_builder_push_submit((rafting_builder_t*)(intptr_t)b, (uint32_t)gid, (uint32_t)count, (uint32_t)unavailableMask));
}
JNIEXPORT void JNICALL FN(builderPushRequest)(JNIEnv* env, jclass k, jlong b, jobject rec, jobject entryTerms) {
    CHECK(rafting_builder_push_request((rafting_builder_t*)(intptr_t)b, (const rafting_req_rec_t*)BUF(rec), (const int64_t*)BUF(entryTerms)));
}
JNIEXPORT void JNICALL FN(builderPushReply)(JNIEnv* env, jclass k, jlong b, jobject rec) {
    CHECK(rafting_builder_push_reply((rafting_builder_t*)(intptr_t)b, (const rafting_batch_rec_t*)BUF(rec)));
}
JNIEXPORT void JNICALL FN(builderClearGroup)(JNIEnv* env, jclass k, jlong b, jint gid) {
    CHECK(rafting_builder_clear_group((rafting_builder_t*)(intptr_t)b, (uint32_t)gid));
}
/* returns the number of ops placed; counters: long[2] = { entry terms used, items still queued } */
JNIEXPORT jint JNICALL FN(builderBuild)(JNIEnv* env, jclass k, jlong b, jlong nowMs, jobject inStruct, jint entCap, jobject placedOut, jobject placedRowOut,
                                        jint placedCap, jobject counters) {
    uint32_t ents = 0, n = 0;
    CHECK(rafting_builder_build((rafting_builder_t*)(intptr_t)b, nowMs, (const rafting_inbox_t*)BUF(inStruct), (uint32_t)entCap, &ents,
                                (rafting_req_rec_t*)BUF(placedOut), (uint8_t*)BUF(placedRowOut), (uint32_t)placedCap, &n));
    int64_t* c = (int64_t*)BUF(counters);
    if (c) { c[0] = ents; c[1] = rafting_builder_pending((const rafting_builder_t*)(intptr_t)b); }
    return (jint)n;
}
#endif /* RAFTING_HAVE_JNI */
