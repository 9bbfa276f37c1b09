/*
 * rafting_ingest.h — transport-side framing for the engine's pump thread (SURVEY.md §8(f)-2).  HOST code, no CUDA.
 *
 * What it replaces in the reference: EventCodec.FrameDecoder / FrameEncoder
 * (src/main/java/io/lubricant/consensus/raft/transport/EventCodec.java:169-201,222-334) — the byte framing every Raft
 * RPC travels in — and the scope parsing of NettyNode.parseContextId (transport/NettyNode.java:92-107), so that a receive
 * buffer filled by the transport can be cut into frames and routed to group ids without creating one Java object per frame.
 *
 * Wire format, exactly as FrameEncoder writes it (all integers big-endian, Netty ByteBuf.writeInt):
 *     SOH(0x01) TYPE [SEQUENCE i32]  STX(0x02) HEAD_LEN i32  HEAD utf-8  BODY_LEN i32  BODY  ETX(0x03) [EOT(0x04)]
 *   TYPE      ENQ 0x05 PingEvent (RPC request) | ACK 0x06 PongEvent (RPC reply) | SYN 0x16 ShakeHandEvent |
 *             MW 0x95 WaitSnapEvent | PM 0x9E TransSnapEvent          (EventCodec.java:32-41)
 *   SEQUENCE  present for ENQ / ACK only (EventCodec.java:239-244)
 *   HEAD      ENQ / ACK: the scope "<RaftService method name>:<contextId>" (NettyNode.java:55-75); others: the message
 *   BODY      Kryo bytes (Serialization.writeObject -> kryo.writeClassAndObject, support/serial/Serialization.java:96-110).
 *             Request bodies (an Object[] of the RPC arguments, NettyNode.java:55-75) stay OPAQUE here: the pump hands
 *             AppendEntries bodies to rafting_log_append.  REPLY bodies — one RaftResponse(term, success),
 *             RaftResponse.java:10-17 — are decoded / encoded by rafting_reply_body_* below (parity UNPINNED, see there)
 *   limits    HEAD_LEN <= 128, BODY_LEN <= 64 MiB (EventCodec.java:25-26); a violation, or a byte other than
 *             SOH/EOT at a frame start, STX after the type, ETX after the body, is the decoder's DecoderException:
 *             RAFTING_E_INVAL, the channel is to be closed (EventCodec.java:326-330)
 *   EOT       at a frame start switches the channel to transparent mode (snapshot stream): scanning stops there
 *
 * One extension, used only between two engines: TYPE SUB 0x1A carries a BATCH — one frame per peer and step instead of
 * one frame per group (Leader.java:216 sends one RPC per follower and group).  Its BODY is an array of fixed 40-byte
 * little-endian records (rafting_batch_rec_t); rafting_batch_to_inbox writes reply records straight into the SoA inbox
 * columns of a leased step.  A peer that does not know the type rejects the frame like any unknown type.  The same frame
 * type with HEAD "Q" carries REQUEST records (rafting_req_rec_t, 64 bytes: AppendEntries / InstallSnapshot plans and vote
 * broadcasts); rafting_outbox_to_requests / rafting_request_to_inbox / rafting_outbox_to_replies are the pump's dispatch loop
 * in C, checked step by step against the Python pump of tests/cluster_sim.py.
 *
 * Threading: every object of this header (context registry, pending table, builder, dispatcher) belongs to ONE pump thread —
 * the one that owns the engine shard (INTEGRATION.md §2); none of them locks.  The stateless functions (frame scan / encode,
 * reply bodies, record <-> column conversions) may be called from any thread on disjoint buffers.  Status codes are
 * rafting_b200.h's; no function throws across the ABI.
 */
#ifndef RAFTING_INGEST_H
#define RAFTING_INGEST_H

#include <stddef.h>
#include <stdint.h>

#include "rafting_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

enum { RAFTING_FRAME_ENQ = 0x05, RAFTING_FRAME_ACK = 0x06, RAFTING_FRAME_SYN = 0x16, RAFTING_FRAME_MW = 0x95,
       RAFTING_FRAME_PM = 0x9E, RAFTING_FRAME_BATCH = 0x1A };
#define RAFTING_FRAME_MAX_HEAD 128u           /* EventCodec.java:25 */
#define RAFTING_FRAME_MAX_BODY (1u << 26)     /* EventCodec.java:26 */

typedef struct rafting_frame {
    uint8_t  type;
    uint8_t  has_sequence;
    uint8_t  ending;          /* an EOT follows the frame's ETX (Event.Ending) — consumed with the frame               */
    uint8_t  _pad;
    int32_t  sequence;
    uint32_t head_off, head_len;   /* offsets into the scanned buffer                                                  */
    uint32_t body_off, body_len;
} rafting_frame_t;

/* Cuts buf[0..len) into complete frames (at most cap).  *consumed = bytes of complete frames (the caller keeps the rest
 * for the next call, exactly like ByteToMessageDecoder's cumulation); *transparent = 1 when an EOT was met at a frame
 * start (the bytes after it belong to the snapshot stream).  Returns 0, or RAFTING_E_INVAL on malformed input with the
 * frames before the error reported. */
int rafting_frame_scan(const uint8_t* buf, size_t len, rafting_frame_t* out, uint32_t cap, uint32_t* n,
                       size_t* consumed, int* transparent);

/* Byte-for-byte what FrameEncoder writes.  Returns the frame's size, or 0 when cap is too small / the limits are exceeded. */
size_t rafting_frame_encode(uint8_t* dst, size_t cap, uint8_t type, int has_sequence, int32_t sequence,
                            const char* head, uint32_t head_len, const void* body, uint32_t body_len, int ending);

/* scope "<method>:<contextId>" -> RAFTING_OP_AE_REQUEST / _PREVOTE_REQ / _VOTE_REQ / _IS_REQUEST and the offset of the
 * context id inside head; RAFTING_E_INVAL for an unknown method ("unknown context", NettyNode.java:106) */
int rafting_scope_parse(const char* head, uint32_t head_len, uint32_t* op_kind, uint32_t* ctx_off);

/* context id -> gid registry (ContextManager keeps the same map by name, ContextManager.java:57-106) */
typedef struct rafting_ctxmap rafting_ctxmap_t;
int rafting_ctxmap_create (rafting_ctxmap_t** out);
int rafting_ctxmap_destroy(rafting_ctxmap_t* m);
int rafting_ctxmap_put    (rafting_ctxmap_t* m, const char* ctx, uint32_t len, uint32_t gid);
int rafting_ctxmap_get    (const rafting_ctxmap_t* m, const char* ctx, uint32_t len, uint32_t* gid);   /* -1 if unknown */

/* ---- reply bodies: the Kryo bytes of one RaftResponse ----------------------------------------------------------------------
 * The body of every ACK frame is kryo.writeClassAndObject(RaftResponse) with the reference's Kryo configuration: kryo 4.0.2
 * (pom.xml:22-26; a dependency, NOT in the reference tree), `new Kryo()` with only the instantiator strategy changed
 * (Serialization.java:21-26) — so: registration not required, references on, FieldSerializer with variable-length integers.
 * Kryo 4.0.2's published format for that object is restated here (PARITY UNPINNED: the build runs no JVM and the
 * reference's SerializationTest only round-trips, it holds no golden bytes; oracle/java/KryoGen.java prints the vectors
 * tests/test_ingest_cpu.py would pin against, for a box that has a JDK and the kryo jar):
 *     01                          class by NAME        (DefaultClassResolver.writeName: varint NAME + 2)
 *     00                          nameId 0             (first class of this object graph)
 *     "io.lubricant.consensus.raft.RaftRespons" 'e'|0x80      Output.writeString, ASCII form (1 < length < 64): last byte flagged
 *     01                          reference marker NOT_NULL   (Kryo.writeReferenceOrNull, first occurrence)
 *     success  1 byte 00 / 01     FieldSerializer, fields in name order: "success" < "term"
 *     term     1..9 bytes         Output.writeLong(value, optimizePositive = false): zig-zag, then 7 bits per byte, low first,
 *                                 bit 7 = "more"; the ninth byte carries 8 bits
 * 45 .. 53 bytes.  The decoder accepts exactly this shape and nothing else (anything else -> RAFTING_E_INVAL: the pump falls
 * back to the Java decoder for that frame). */
#define RAFTING_REPLY_BODY_MAX 53u
size_t rafting_reply_body_encode(uint8_t* dst, size_t cap, int64_t term, int success);          /* bytes written, 0 = no room */
int    rafting_reply_body_decode(const uint8_t* body, size_t len, int64_t* term, int* success);

/* One ACK frame of a scanned buffer -> what a lane event needs: the group (scope's context id through the registry), the reply
 * kind (appendEntries -> RAFTING_EV_AE_ACK, installSnapshot -> _IS_ACK, preVote -> _PV_REPLY, requestVote -> _RV_REPLY), the
 * frame's sequence (the key of the caller's pending-invocation table, NettyNode.getInvocationIfPresent, NettyNode.java:88-90)
 * and the decoded RaftResponse.  RAFTING_E_INVAL: not an ACK frame, unknown scope / context, or a body of another shape. */
int rafting_ack_frame_decode(const uint8_t* buf, const rafting_frame_t* fr, const rafting_ctxmap_t* map, uint32_t* gid,
                             uint32_t* ev_kind, int32_t* sequence, int64_t* term, int* success);

/* The same for a whole scanned buffer: one record per ACK frame that decodes (frame = its index in `frames`), the others —
 * requests, handshakes, replies with another body — are skipped and stay with the caller.  out has room for n records. */
typedef struct rafting_ack_rec {
    uint32_t gid;
    uint8_t  kind;            /* RAFTING_EV_*                                                                            */
    uint8_t  success;
    uint16_t _pad;
    int32_t  sequence;
    uint32_t frame;
    int64_t  term;
} rafting_ack_rec_t;        /* 24 bytes */
int rafting_ack_frames_decode(const uint8_t* buf, const rafting_frame_t* frames, uint32_t n, const rafting_ctxmap_t* map,
                              rafting_ack_rec_t* out, uint32_t* n_out);

/* ---- engine-to-engine batch records (TYPE 0x1A) ---- */
typedef struct rafting_batch_rec {
    uint32_t gid;             /* both ends open a context under the same gid (rafting_group_open takes the gid)         */
    uint8_t  kind;            /* RAFTING_EV_* : reply to an RPC of that kind                                            */
    uint8_t  lane;            /* follower lane of the RECEIVER the reply belongs to                                     */
    uint8_t  flags;           /* bits 0..1 outcome (RAFTING_OUT_*), bit 2 success                                       */
    uint8_t  row;             /* row of the receiver's step the event goes to (assigned by the receiver's pump)         */
    uint32_t incarnation;     /* echo of plan_meta / ballot_meta bits 32..63                                            */
    uint32_t _pad;
    int64_t  term;            /* RaftResponse.term()                                                                    */
    int64_t  epoch_at_send;   /* echo of plan_epoch                                                                     */
    int64_t  last_at_send;    /* echo of plan_lc.x                                                                      */
} rafting_batch_rec_t;      /* 40 bytes */

/* Writes n reply records into the lane-event columns of a (leased, host) inbox of `rows` x `n_groups` x F: ev_meta, ev_tn =
 * (term, now_ms), ev_el = (epoch, last).  Dense steps only (position == gid).  A slot that is already occupied, a gid /
 * lane / row out of range -> RAFTING_E_INVAL with *n_done records written (the caller defers the rest to the next step:
 * one event per (row, group, lane)). */
int rafting_batch_to_inbox(const rafting_batch_rec_t* recs, uint32_t n, int64_t now_ms, const rafting_inbox_t* in,
                           uint32_t n_groups, uint32_t F, uint32_t* n_done);

/* ---- engine-to-engine REQUEST records (TYPE 0x1A with HEAD "Q"; reply batches use HEAD "R") -----------------------------
 * What Leader.replicateLog / Follower.prepareElection / Candidate.startElection send — one RPC per follower and group
 * (Leader.java:170-216, Follower.java:241-256, Candidate.java:94-110) — as fixed records, one frame per peer and step.
 * rafting_outbox_to_requests is the pump's dispatch loop in C (INTEGRATION.md §4): it walks a host outbox in the serial
 * order of the step (row, then group, then lane) and emits one record per AE / IS plan and per lane of a vote broadcast.
 * An AppendEntries plan does not carry its term (a role object's term is fixed for its lifetime, RaftMember.java:16-26):
 * the dispatcher remembers (incarnation -> current_term) per group from the end-of-step columns it has seen. */
typedef struct rafting_req_rec {
    uint32_t gid;
    uint8_t  kind;            /* RAFTING_OP_AE_REQUEST / _PREVOTE_REQ / _VOTE_REQ / _IS_REQUEST                          */
    uint8_t  src_slot;        /* the sending node (the op's `peer` on the receiving side)                                */
    uint8_t  dst_slot;        /* the node the record goes to: slot of the sender's follower lane                        */
    uint8_t  row;             /* row of the sender's step                                                                */
    uint32_t incarnation;     /* of the sending role object; the reply echoes it                                         */
    uint32_t count;           /* AE: number of entries (their terms / payloads travel beside the record)                */
    int64_t  term;            /* term argument of the RPC                                                                */
    int64_t  a, b;            /* AE: prevLogIndex, prevLogTerm | votes: lastLogIndex, lastLogTerm | IS: lastIncluded*   */
    int64_t  commit;          /* AE: leaderCommit                                                                        */
    int64_t  epoch, last;     /* AE / IS: (epochAtSend, lastIndexAtSend) — the closure of the reply callback            */
} rafting_req_rec_t;        /* 64 bytes */

typedef struct rafting_dispatch rafting_dispatch_t;
int rafting_dispatch_create(uint32_t n_groups, uint32_t F, uint32_t local_slot, rafting_dispatch_t** out);
int rafting_dispatch_destroy(rafting_dispatch_t* d);
/* Dense host outbox of `rows` rows -> records (at most cap; RAFTING_E_CAPACITY beyond).  *n_unknown counts AE / IS plans
 * whose role object's term the dispatcher has never seen (skipped). */
int rafting_outbox_to_requests(rafting_dispatch_t* d, const rafting_outbox_t* ob, uint32_t rows, rafting_req_rec_t* out,
                               uint32_t cap, uint32_t* n_out, uint32_t* n_unknown);
/* Receiving side: one record -> the op slot (row, gid) of a dense host inbox (op_meta / op_nr / op_ab / op_cd / op_e); an AE
 * record's entry terms are appended to ent_terms at *ent_count.  host_result: RaftContext.installSnapshot's answer for an IS
 * request (RaftRoutine.java:408-445), ignored otherwise.  RAFTING_E_INVAL: slot taken, gid / row out of range, no room. */
int rafting_request_to_inbox(const rafting_req_rec_t* r, const int64_t* entry_terms, uint32_t row, int64_t now_ms, int host_result,
                             const rafting_inbox_t* in, uint32_t n_groups, uint32_t ent_cap, uint32_t* ent_count);

/* After the step: the replies to the requests that were placed.  placed[i] went to row placed_row[i]; a request whose
 * rep_meta is not valid (the handler threw: no reply leaves, the sender's Async times out — EventLoop semantics) is skipped.
 * Emits reply records for rafting_batch_to_inbox on the SENDER's side: lane = this node's follower lane there, the echo
 * fields copied from the request, term = RaftResponse.term().  out has room for n records. */
int rafting_outbox_to_replies(const rafting_outbox_t* ob, uint32_t n_groups, uint32_t local_slot, const rafting_req_rec_t* placed,
                              const uint8_t* placed_row, uint32_t n, rafting_batch_rec_t* out, uint32_t* n_out);

/* The same two ends for the compact host path (include/rafting_b200.h, rafting_step_begin_compact_req).
 * rafting_request_to_creq places one record at (row, gid) of a compact step: an AppendEntries that fits the record rules
 * becomes a rafting_creq_t (its time relative to in->row_base[row], which the caller sets before placing), anything else a
 * rafting_cesc_op_t whose entry terms are appended to q->ent_terms.  Both lists stay strictly increasing (placing in slot
 * order appends).  The list arrays are the caller's, with room for req_cap / esc_cap / ent_cap entries; q's counts grow.
 * RAFTING_E_INVAL: slot taken (an op_c word, a record or an op escape), gid / row out of range, no room. */
int rafting_request_to_creq(const rafting_req_rec_t* r, const int64_t* entry_terms, uint32_t row, int64_t now_ms, int host_result,
                            const rafting_cinbox_t* in, uint32_t n_groups, rafting_creqs_t* q, uint32_t req_cap, uint32_t esc_cap,
                            uint32_t ent_cap);
/* rafting_outbox_to_replies over a waited-for compact outbox: the reply of a placed request is its rep_c byte (bit 7) or its
 * RAFTING_CESC_REPLY escape record.  RAFTING_E_CAPACITY when the escape list overflowed (fetch the dense outbox instead). */
int rafting_coutbox_to_replies(const rafting_coutbox_t* co, uint32_t n_groups, uint32_t local_slot, const rafting_req_rec_t* placed,
                               const uint8_t* placed_row, uint32_t n, rafting_batch_rec_t* out, uint32_t* n_out);
/* rafting_outbox_to_requests over a waited-for compact outbox of a step begun with `flags` (RAFTING_COMPACT_ELECTIONS /
 * RAFTING_COMPACT_PREV_TERM, or 0): the same records, in the same order, that rafting_outbox_to_requests emits for the dense
 * outbox the compact one stands for, with the same incarnation -> term memory in d.  Plans come from their plan_c words (kind
 * 7 under RAFTING_COMPACT_PREV_TERM) or their RAFTING_CESC_PLAN records, ballots from their lanes' words (under
 * RAFTING_COMPACT_ELECTIONS) or their RAFTING_CESC_BALLOT records; escape records are matched by slot, whatever their order.
 * tags[i] is the tag the pump puts into the pending entry of out[i] (rafting_pending_put): the plan's tag for an AE / IS, the
 * lane's tag for a compact ballot, RAFTING_CTAG_NONE for an escaped ballot or an untagged plan.  out and tags have room for
 * cap records (RAFTING_E_CAPACITY beyond).  RAFTING_E_CAPACITY too when the escape list overflowed (counts[0] > esc_cap):
 * fetch the dense outbox and use rafting_outbox_to_requests.  RAFTING_E_INVAL: an unknown flag, or an escaped plan word
 * without its record. */
int rafting_coutbox_to_requests(rafting_dispatch_t* d, const rafting_coutbox_t* co, uint32_t rows, uint32_t flags,
                                rafting_req_rec_t* out, uint8_t* tags, uint32_t cap, uint32_t* n_out, uint32_t* n_unknown);

/* ---- replies -> compact wire words (the compact host path of include/rafting_b200.h) -------------------------------------
 * The pending-invocation table of the pump: what NettyNode keeps per connection as (scope, sequence) -> Invocation
 * (NettyNode.java:88-90, Async.java) — here (peer, sequence) -> the group, the follower lane, the TAG the plan was sent under
 * (plan_c bits 5..10; the echo pair and the incarnation wait in the engine's in-flight table under that tag), the term the
 * request carried, and the echo pair itself for replies that have to travel in full.
 * rafting_acks_to_cinbox takes the decoded ACK records of one peer (rafting_ack_frames_decode), looks each sequence up and
 * writes the reply into row `row` of a compact inbox under construction: a 32-bit ev_c word when it fits the compact rules
 * (an AE / IS ack, tag 0..31, 0 <= now - row_base[row] <= 65535, RaftResponse.term() == the term sent), else the word
 * RAFTING_CEV_ESCAPED plus one escape record with every field.  A reply whose lane slot in that row is taken is DEFERRED (its
 * index goes to deferred[], its pending entry stays) — one event per (row, group, lane); an unknown sequence (the invocation
 * timed out and was removed) is counted and dropped, as the reference drops it (NettyNode.getInvocationIfPresent == null). */
typedef struct rafting_pending rafting_pending_t;
int rafting_pending_create(uint32_t capacity_hint, rafting_pending_t** out);
int rafting_pending_destroy(rafting_pending_t* p);
int rafting_pending_put(rafting_pending_t* p, uint32_t peer, int32_t sequence, uint32_t ev_kind /* RAFTING_EV_* of the reply */, uint32_t gid,
                        uint32_t lane, uint32_t tag /* 0..31 | 63 */, uint32_t incarnation, int64_t term, int64_t epoch_at_send,
                        int64_t last_at_send);
int rafting_pending_remove(rafting_pending_t* p, uint32_t peer, int32_t sequence);          /* time-out: RAFTING_E_INVAL if absent */
uint32_t rafting_pending_size(const rafting_pending_t* p);
int rafting_acks_to_cinbox(rafting_pending_t* p, uint32_t peer, const rafting_ack_rec_t* acks, uint32_t n, int64_t now_ms, uint32_t row,
                           const rafting_cinbox_t* cin, uint32_t n_groups, uint32_t F, rafting_cesc_in_t* esc, uint32_t esc_cap,
                           uint32_t* n_esc /* in/out */, uint32_t* deferred /* [n] */, uint32_t* n_deferred, uint32_t* n_unknown);

/* Invocations that completed WITHOUT a reply — the Async timed out or was cancelled (Async.java:239-254: outcome ERROR /
 * CANCELED; Leader's callback then runs statFailure) — written the same way: the ev_c word carries the outcome and the tag
 * (success 0), or an escape record when the plan had no tag / the time offset does not fit.  Same deferral rule. */
int rafting_failures_to_cinbox(rafting_pending_t* p, uint32_t peer, const int32_t* sequences, uint32_t n, uint32_t outcome, int64_t now_ms,
                               uint32_t row, const rafting_cinbox_t* cin, uint32_t n_groups, uint32_t F, rafting_cesc_in_t* esc,
                               uint32_t esc_cap, uint32_t* n_esc, uint32_t* deferred, uint32_t* n_deferred, uint32_t* n_unknown);

/* The same three writers for a step begun with RAFTING_COMPACT_ELECTIONS (rafting_step_begin_compact_ex); flags == 0 is exactly
 * the function without _ex.  They accept RAFTING_COMPACT_PREV_TERM and ignore it (an ack to a kind-7 plan is an ordinary AE
 * ack), so that a pump passes one flags word everywhere.  Under RAFTING_COMPACT_ELECTIONS:
 *   rafting_request_to_creq_ex  a PreVote / RequestVote with src_slot < 32, 0 <= now - row_base[row] <= 65535 and
 *                               0 <= term - lastLogTerm < 2^32 becomes a vote record (no entries, d_commit 0)
 *   rafting_acks_to_cinbox_ex   a vote reply whose pending entry has a tag (the ballot lane's, put with term = the ballot
 *                               term) and whose term lies 0..7 below the ballot term becomes a vote word
 *   rafting_failures_to_cinbox_ex   a timed-out / cancelled vote RPC with a tag becomes a vote word (c = 0)
 * and every escaped word carries the tag of its pending entry (RAFTING_CEV_ESCAPED | tag << 8), which unpack frees. */
int rafting_request_to_creq_ex(const rafting_req_rec_t* r, const int64_t* entry_terms, uint32_t row, int64_t now_ms, int host_result,
                               const rafting_cinbox_t* in, uint32_t n_groups, rafting_creqs_t* q, uint32_t req_cap, uint32_t esc_cap,
                               uint32_t ent_cap, uint32_t flags);
int rafting_acks_to_cinbox_ex(rafting_pending_t* p, uint32_t peer, const rafting_ack_rec_t* acks, uint32_t n, int64_t now_ms, uint32_t row,
                              const rafting_cinbox_t* cin, uint32_t n_groups, uint32_t F, rafting_cesc_in_t* esc, uint32_t esc_cap,
                              uint32_t* n_esc, uint32_t* deferred, uint32_t* n_deferred, uint32_t* n_unknown, uint32_t flags);
int rafting_failures_to_cinbox_ex(rafting_pending_t* p, uint32_t peer, const int32_t* sequences, uint32_t n, uint32_t outcome,
                                  int64_t now_ms, uint32_t row, const rafting_cinbox_t* cin, uint32_t n_groups, uint32_t F,
                                  rafting_cesc_in_t* esc, uint32_t esc_cap, uint32_t* n_esc, uint32_t* deferred, uint32_t* n_deferred,
                                  uint32_t* n_unknown, uint32_t flags);

/* ---- the inbox builder: what the event loops' queues become (dense / leased path) -------------------------------------------
 * The reference queues work per context on its event loop (EventLoop.java:87-101): replies hop back with execute(urgent),
 * inbound requests and RaftStub.submit are queued behind them.  The builder keeps one FIFO per group — requests (records +
 * entry terms), replies (batch records) and submits (placed at the FRONT: RaftStub.process runs before what is already
 * queued for the tick) — and turns them into the rows of one dense step: row 0 is the sweep row (row_now[0] = now fires the
 * due timers); per group the queue is drained in order, an op taking the op slot of the row AFTER the cursor's row, a lane
 * event the slot of its lane in the cursor's row when that slot lies behind the cursor, else in the next row; what does not
 * fit into `rows` rows stays queued for the next step (one op per (row, group), one event per (row, group, lane), the serial
 * order of the step == arrival order).  tests/cluster_sim.py holds the same rule in Python; the two are compared on every
 * step of randomized cluster runs. */
typedef struct rafting_builder rafting_builder_t;
int rafting_builder_create(uint32_t n_groups, uint32_t F, rafting_builder_t** out);
int rafting_builder_destroy(rafting_builder_t* b);
int rafting_builder_push_submit (rafting_builder_t* b, uint32_t gid, uint32_t count, uint32_t unavailable_mask);
int rafting_builder_push_request(rafting_builder_t* b, const rafting_req_rec_t* r, const int64_t* entry_terms);
int rafting_builder_push_reply  (rafting_builder_t* b, const rafting_batch_rec_t* r);
int rafting_builder_clear_group (rafting_builder_t* b, uint32_t gid);
uint32_t rafting_builder_pending(const rafting_builder_t* b);
/* in: a dense host inbox with row_now, all op_* and ev_* columns and ent_terms[ent_cap]; the builder zeroes and fills it.
 * placed / placed_row / is_submit: what went in, in (group, row) order — requests for rafting_outbox_to_replies, submits
 * (kind RAFTING_OP_SUBMIT, count) so that the caller can store the payloads of accepted commands. */
int rafting_builder_build(rafting_builder_t* b, int64_t now_ms, const rafting_inbox_t* in, uint32_t ent_cap, uint32_t* ent_count,
                          rafting_req_rec_t* placed, uint8_t* placed_row, uint32_t placed_cap, uint32_t* n_placed);

/* ---- commit records -> apply ranges (SURVEY.md §8(f)-4) --------------------------------------------------------------------
 * What RaftRoutine.commitState hands to applyCommand (RaftRoutine.java:224-306): for every group whose role_word carries the
 * commit-dirty bit (bit 31) and whose commit_index is ahead of applied[gid], one record (gid, applied + 1 .. commit_index);
 * applied[gid] is advanced to commit_index.  The caller feeds the ranges to rafting_log_gather and the state machine.
 * gids == NULL: dense columns (position == gid); otherwise RAFTING_INBOX_COMPACT_GROUPS columns indexed by position. */
typedef struct rafting_apply_rec { uint32_t gid; uint32_t _pad; int64_t first, last; } rafting_apply_rec_t;   /* 24 bytes */
int rafting_outbox_apply_ranges(const rafting_outbox_t* ob, const uint32_t* gids, uint32_t n, int64_t* applied, uint32_t n_groups,
                                rafting_apply_rec_t* out, uint32_t cap, uint32_t* n_out);

#ifdef __cplusplus
}
#endif
#endif
