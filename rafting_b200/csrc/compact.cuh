// compact.cuh — the compact host path: an eighth of the dense path's PCIe bytes, losslessly (include/rafting_b200.h,
// "COMPACT host path").  Two kernels bracket the unchanged step kernel:
//
//   unpack_kernel   wire columns (ev_c 4 B / lane slot, op_c 4 B / group row, row_base)  ->  the dense SoA inbox the step kernel
//                   reads; the (epochAtSend, lastIndexAtSend) pair AND the incarnation of every ack come out of the HBM
//                   in-flight table under the tag the reply echoes, and the tag's slot is freed
//   pack_kernel     the dense outbox  ->  plan_c 4 B / lane slot, rep_c 1 B / group row, the per-group columns;
//                   every AE / IS plan gets a free tag of its (group, follower) lane and parks its echo pair and its
//                   incarnation in the table; whatever breaks a compact rule goes, in full, to the escape list
//
// Under RAFTING_COMPACT_ELECTIONS (the EL instantiations) vote RPCs take tags as well: a compact ballot's lanes park
// (ballot term, 0) and the asking role's incarnation, and a vote reply word gets them back.  Under RAFTING_COMPACT_PREV_TERM
// (the PT instantiations of pack_kernel) an AE plan whose prevLogTerm lies 1..8 below the group's term travels as a kind-7
// word instead of an escape record; it takes and parks its tag as a kind-1 plan does, so its ack is an ordinary AE word.
//
// One thread per (group, follower) walks the rows in order in both kernels, so the tag bitmap of a lane is only ever touched
// by its own thread, and the three kernels of a step (unpack, step, pack) are ordered on the engine's stream.  What this
// replaces in the reference is the closure state of the Async callbacks registered by Leader.replicateLog
// (Leader.java:216-237 captures epoch.index() and lastIndex per RPC): here it lives in HBM next to Leadership.State.
//
// Included at the end of engine.cu (same translation unit: it uses rafting_engine, Slot, fail(), CU()).
#pragma once
#include <cub/device/device_scan.cuh>

namespace rafting {

constexpr uint32_t CESC_INLINE = 256;            // escape records that always travel down with the columns (14 KB)
constexpr int CTAGS = 32;                        // in-flight slots per (group, follower): IN_FLIGHT_LIMIT is 20 (Leadership.java:11)

struct InboxW {                                  // writable view of the dense staging columns unpack_kernel fills
    uint64_t* op_meta; i64x2* op_nr; i64x2* op_ab; uint64_t* ev_meta; i64x2* ev_tn; i64x2* ev_el;
    i64x2* op_cd; int64_t* op_e; int64_t* ent_terms;   // steps with a request list only, else null
};
struct CInD {                                    // device view of rafting_cinbox_t
    uint32_t rows, n_esc;
    const int64_t* row_base; const uint32_t* op_c; const uint16_t* op_unavail; const uint32_t* ev_c; const rafting_cesc_in_t* esc;
};
struct COutD {                                   // device view of rafting_coutbox_t
    uint32_t* plan_c; uint8_t* rep_c;
    int64_t* commit_index; int64_t* current_term; uint32_t* role_word; uint32_t* incarnation; uint32_t* err_word;
    i64x2* last_entry; i64x2* epoch; rafting_cesc_out_t* esc; uint32_t esc_cap; uint32_t* counts;
    bool compact_replies;                        // rep_c bits 6 / 7 (steps begun with a request list)
};

// the active list of a step begun with rafting_step_begin_compact_active (device copy): position i stands for gids[i]
struct ActiveD { const uint32_t* gids; uint32_t n; };

// EL: steps begun with RAFTING_COMPACT_ELECTIONS (vote replies as words, escaped words that free their tag)
// AL: steps over an active list.  One thread per (position, follower); the wire and the dense staging are positional, the
//     in-flight table, its tag bitmap and the group tables stay indexed by gid (table stride G * F)
template <bool EL, bool AL>
__global__ void __launch_bounds__(256) unpack_kernel(Tables T, CInD in, InboxW out, const i64x2* __restrict__ table, const uint32_t* __restrict__ tinc, uint32_t* __restrict__ bits, ActiveD act) {
    const uint32_t GF = T.G * T.F;
    const uint32_t NF = AL ? act.n * T.F : GF;                       // lane slots of one row of the step
    const uint32_t t = blockIdx.x * 256u + threadIdx.x;
    if (t >= NF) return;
    const uint32_t i = t / T.F, f = t - i * T.F;                    // position in the step (the gid of a whole-shard step)
    const uint32_t g = AL ? act.gids[i] : i;
    const uint32_t s = AL ? g * T.F + f : t;                        // the lane's in-flight state
    if (in.ev_c) {
        const int64_t term_now = T.g_term[g];
        uint32_t b = bits[s];
        for (uint32_t r = 0; r < in.rows; r++) {
            const size_t idx = (size_t)r * NF + t;
            const uint32_t w = in.ev_c[idx];
            const uint32_t kind = w & 0xfu;
            uint64_t em = 0;
            if (kind == RAFTING_EV_AE_ACK || kind == RAFTING_EV_IS_ACK) {
                const uint32_t tag = (w >> 8) & 0xffu;
                i64x2 el = {0, 0}; uint32_t inc = 0;
                if (tag < (uint32_t)CTAGS) { el = table[(size_t)tag * GF + s]; inc = tinc[(size_t)tag * GF + s]; b &= ~(1u << tag); }
                i64x2 tn; tn.x = ((w >> 7) & 1u) ? term_now : 0; tn.y = in.row_base[r] + (int64_t)(w >> 16);
                em = (uint64_t)(w & 0x7fu) | ((uint64_t)inc << 32);         // kind | outcome | success | incarnation (from the table)
                out.ev_tn[idx] = tn; out.ev_el[idx] = el;
            } else if constexpr (EL) {
                if (kind == RAFTING_EV_PV_REPLY || kind == RAFTING_EV_RV_REPLY) {
                    // (ballot term, 0) and the asking role's incarnation wait under the tag; the reply's term is c below it
                    const uint32_t tag = RAFTING_CEV_VOTE_TAG(w);
                    const int64_t bt = table[(size_t)tag * GF + s].x; const uint32_t inc = tinc[(size_t)tag * GF + s];
                    b &= ~(1u << tag);
                    i64x2 tn; tn.x = ((w >> 4) & 3u) == RAFTING_OUT_OK ? (int64_t)((uint64_t)bt - RAFTING_CEV_VOTE_C(w)) : 0;
                    tn.y = in.row_base[r] + (int64_t)(w >> 16);
                    const i64x2 el = {0, 0};
                    em = (uint64_t)(w & 0x7fu) | ((uint64_t)inc << 32);
                    out.ev_tn[idx] = tn; out.ev_el[idx] = el;
                } else if (kind == RAFTING_CEV_ESCAPED) {
                    const uint32_t tag = (w >> 8) & 0xffu;                  // the escaped event's RPC has completed too
                    if (tag < (uint32_t)CTAGS) b &= ~(1u << tag);
                }
            }
            out.ev_meta[idx] = em;                                          // escaped / empty slots read as "no event" until patched
        }
        bits[s] = b;
    }
    if (f == 0 && (in.op_c || out.op_cd)) {
        for (uint32_t r = 0; r < in.rows; r++) {
            const size_t gi = (size_t)r * (AL ? act.n : T.G) + i;
            const uint32_t c = in.op_c ? in.op_c[gi] : 0u;
            out.op_meta[gi] = (uint64_t)RAFTING_OP_MAKE(c & 0xfu, 0u, (c >> 4) & 0xfffu);
            i64x2 nr; nr.x = in.row_base[r] + (int64_t)(c >> 16); nr.y = 0;
            out.op_nr[gi] = nr;
            if (out.op_ab) { i64x2 ab; ab.x = in.op_unavail ? (int64_t)in.op_unavail[gi] : 0; ab.y = 0; out.op_ab[gi] = ab; }
            if (out.op_cd) { const i64x2 z = {0, 0}; out.op_cd[gi] = z; out.op_e[gi] = 0; }
        }
    }
}

// ---- the request list (rafting_creqs_t): records and op escapes, after unpack_kernel has written the op_c words ----
struct CReqD {                                   // device view of rafting_creqs_t
    uint32_t n_req, n_esc, slots;                // slots = rows * n (n: the step's groups, max_groups or n_active)
    const rafting_creq_t* req; const rafting_cesc_op_t* esc;
    const int64_t* row_base; const uint32_t* op_c;
    uint32_t ent_count, pool_end;                // records' terms start at ent_count; the step's pool ends at pool_end
    uint64_t* counts; uint64_t* offs;            // [n_req] entry count of each record, its exclusive scan
    uint32_t* order;                             // bit 0: req decreases somewhere, bit 1: esc does
};
constexpr uint32_t CREQ_META_ZERO = 0xf800u;     // bits 11..15 of a record's meta
constexpr uint32_t CREQ_META_ZERO_EL = 0xe000u;  // bits 13..15 (under RAFTING_COMPACT_ELECTIONS bits 11..12 name a vote)

// Pass 1, one thread per list position: entry counts for the scan, and whether either list decreases anywhere.  A
// decreasing list can hold the same slot twice at positions that are not adjacent; rather than search for them, every
// op of both lists is then malformed, so that all writers of a slot write the same thing.
__global__ void creq_prepare_kernel(CReqD q) {
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k < q.n_req) {
        q.counts[k] = RAFTING_CREQ_COUNT(q.req[k].meta);
        if (k + 1 < q.n_req && q.req[k + 1].slot < q.req[k].slot) atomicOr(q.order, 1u);
    }
    if (k + 1 < q.n_esc && q.esc[k + 1].slot < q.esc[k].slot) atomicOr(q.order, 2u);
}

template <typename Rec> __device__ __forceinline__ bool list_holds(const Rec* v, uint32_t n, uint32_t slot) {
    uint32_t lo = 0, hi = n;                     // binary search of a non-decreasing list
    while (lo < hi) { const uint32_t m = (lo + hi) >> 1; if (v[m].slot < slot) lo = m + 1; else hi = m; }
    return lo < n && v[lo].slot == slot;
}

__device__ __forceinline__ void put_op(const InboxW& o, size_t gi, uint64_t meta, int64_t now, int64_t draw, int64_t a, int64_t b,
                                       int64_t c, int64_t d, int64_t e) {
    o.op_meta[gi] = meta;
    i64x2 v; v.x = now; v.y = draw; o.op_nr[gi] = v;
    v.x = a; v.y = b; o.op_ab[gi] = v;
    v.x = c; v.y = d; o.op_cd[gi] = v;
    o.op_e[gi] = e;
}

// Pass 2, one thread per record (k < n_req) or op escape (k - n_req): the op in full at its slot.  Every writer of a slot
// that is claimed twice detects it from read-only inputs and writes the same malformed op, so the result never depends on
// the order of the writes.
// EL (RAFTING_COMPACT_ELECTIONS): a record with meta bits 11..12 set is a PreVote / RequestVote
template <bool EL>
__global__ void unpack_requests_kernel(CReqD q, InboxW o, uint32_t n) {
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if ((uint64_t)k >= (uint64_t)q.n_req + q.n_esc) return;
    const bool is_req = k < q.n_req;
    const uint32_t j = is_req ? k : k - q.n_req;
    const uint32_t slot = is_req ? q.req[j].slot : q.esc[j].slot;
    if (slot >= q.slots) return;
    const uint32_t r = slot / n;
    bool bad = q.order[0] != 0 || (q.op_c && (q.op_c[slot] & 0xfu) != RAFTING_OP_NONE);
    if (is_req) {
        if constexpr (EL) {
            const uint32_t m = q.req[j].meta, vk = RAFTING_CREQ_VOTE(m);
            bad = bad || (j > 0 && q.req[j - 1].slot == slot) || (j + 1 < q.n_req && q.req[j + 1].slot == slot) ||
                  list_holds(q.esc, q.n_esc, slot) || (m & CREQ_META_ZERO_EL) != 0 || vk == 3u ||
                  (vk != 0u && (RAFTING_CREQ_COUNT(m) != 0u || q.req[j].d_commit != 0));
            if (!bad && vk != 0u) {
                const rafting_creq_t x = q.req[j];
                put_op(o, slot, (uint64_t)RAFTING_OP_MAKE(vk == RAFTING_CREQ_VOTE_PRE ? RAFTING_OP_PREVOTE_REQ : RAFTING_OP_VOTE_REQ, RAFTING_CREQ_PEER(m), 0u),
                       q.row_base[r] + (int64_t)RAFTING_CREQ_DT(m), 0, x.term, x.prev_index, (int64_t)((uint64_t)x.term - (uint64_t)x.d_prev_term), 0, 0);
                return;
            }
        } else {
            bad = bad || (j > 0 && q.req[j - 1].slot == slot) || (j + 1 < q.n_req && q.req[j + 1].slot == slot) ||
                  list_holds(q.esc, q.n_esc, slot) || (q.req[j].meta & CREQ_META_ZERO) != 0;
        }
    } else {
        bad = bad || (j > 0 && q.esc[j - 1].slot == slot) || (j + 1 < q.n_esc && q.esc[j + 1].slot == slot) ||
              list_holds(q.req, q.n_req, slot);
    }
    if (bad) { put_op(o, slot, RAFTING_COP_MALFORMED, q.row_base[r], 0, 0, 0, 0, 0, 0); return; }
    if (!is_req) {
        const rafting_cesc_op_t x = q.esc[j];
        put_op(o, slot, (uint64_t)(uint32_t)x.op_meta | ((uint64_t)x.ent << 32), x.now_ms, x.draw, x.a, x.b, x.c, x.d, x.e);
        return;
    }
    const rafting_creq_t x = q.req[j];
    const uint32_t count = RAFTING_CREQ_COUNT(x.meta);
    const uint64_t off = (uint64_t)q.ent_count + q.offs[j];
    if (off + count <= q.pool_end)
        for (uint32_t i = 0; i < count; i++) o.ent_terms[off + i] = x.term;
    const uint32_t ent = off < 0xffffffffull ? (uint32_t)off : 0xffffffffu;   // past the pool: the step answers BAD_EVENT
    const int64_t prev = x.prev_index;
    put_op(o, slot, (uint64_t)RAFTING_OP_MAKE(RAFTING_OP_AE_REQUEST, RAFTING_CREQ_PEER(x.meta), count) | ((uint64_t)ent << 32),
           q.row_base[r] + (int64_t)RAFTING_CREQ_DT(x.meta), 0, x.term, prev,
           (int64_t)((uint64_t)x.term - (uint64_t)x.d_prev_term), (int64_t)((uint64_t)prev + (uint64_t)(int64_t)x.d_commit),
           (int64_t)((uint64_t)prev + 1u));
}
// escape records: the event in full, after unpack_kernel has written the slot as empty
__global__ void unpack_escapes_kernel(CInD in, InboxW out, uint32_t slots) {
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= in.n_esc) return;
    const rafting_cesc_in_t e = in.esc[k];
    if (e.slot >= slots) return;
    out.ev_meta[e.slot] = e.ev_meta;
    i64x2 v; v.x = e.term; v.y = e.now_ms; out.ev_tn[e.slot] = v;
    v.x = e.epoch_at_send; v.y = e.last_at_send; out.ev_el[e.slot] = v;
}

__device__ __forceinline__ void put_escape(const COutD& o, uint32_t kind, uint32_t slot, uint64_t meta, int64_t a, int64_t b, int64_t c, int64_t d, int64_t e) {
    const uint32_t k = atomicAdd(o.counts + 0, 1u);
    if (k < o.esc_cap) {
        rafting_cesc_out_t r; r.kind = kind; r.slot = slot; r.meta = meta; r.a = a; r.b = b; r.c = c; r.d = d; r.e = e;
        o.esc[k] = r;
    }
}

// Under RAFTING_COMPACT_ELECTIONS: the plan_c kind the ballot of (row, group) gi travels as, or 0 when it stays an escape
// record.  Every lane thread of the group and its f == 0 thread reach the same answer from the same read-only columns.
__device__ __forceinline__ uint32_t ballot_lane_kind(const OutboxD& in, size_t gi, uint32_t F, int64_t term_end, uint32_t inc_end, i64x2 last_end) {
    if (!in.ballot_meta) return 0;
    const uint64_t bm = in.ballot_meta[gi];
    const uint32_t bk = (uint32_t)bm;                                   // bits 4..31 must be clear as well
    if ((bk != RAFTING_BALLOT_PREVOTE && bk != RAFTING_BALLOT_VOTE) || (uint32_t)(bm >> 32) != inc_end) return 0;
    const bool pre = bk == RAFTING_BALLOT_PREVOTE;
    const i64x2 bl = in.ballot_last[gi];
    if ((uint64_t)in.ballot_term[gi] != (uint64_t)term_end + (pre ? 1u : 0u) || bl.x != last_end.x || bl.y != last_end.y) return 0;
    if (in.plan_meta)
        for (uint32_t f = 0; f < F; f++) if (in.plan_meta[gi * F + f] != 0) return 0;
    return pre ? RAFTING_CPLAN_PREVOTE : RAFTING_CPLAN_VOTE;
}
// the plan_c word of a compact ballot's lane: the lowest free tag of the lane parks (ballot term, 0) and the incarnation
__device__ __forceinline__ uint32_t ballot_lane_word(const OutboxD& in, size_t gi, uint32_t F, int64_t term_end, uint32_t inc_end, i64x2 last_end,
                                                     i64x2* table, uint32_t* tinc, size_t at, uint32_t& b) {
    const uint32_t bk = ballot_lane_kind(in, gi, F, term_end, inc_end, last_end);
    if (!bk) return 0;
    uint32_t tag = RAFTING_CTAG_NONE;
    const uint32_t fr = ~b;
    if (fr) {
        tag = (uint32_t)__ffs((int)fr) - 1u; b |= 1u << tag;
        i64x2 v; v.x = in.ballot_term[gi]; v.y = 0; table[(size_t)tag * at] = v; tinc[(size_t)tag * at] = inc_end;
    }
    return bk | (tag << 5);
}

// PT: steps begun with RAFTING_COMPACT_PREV_TERM (an AE plan that breaks only the prevLogTerm rule becomes a kind-7 word)
// AL: steps over an active list, as for unpack_kernel; the dense outbox's group columns are positional (COMPACT_GROUPS)
template <bool EL, bool PT, bool AL>
__global__ void __launch_bounds__(256) pack_kernel(Tables T, uint32_t rows, OutboxD in, COutD out, i64x2* __restrict__ table, uint32_t* __restrict__ tinc, uint32_t* __restrict__ bits, ActiveD act) {
    const uint32_t GF = T.G * T.F;
    const uint32_t N = AL ? act.n : T.G, NF = AL ? act.n * T.F : GF;
    const uint32_t t = blockIdx.x * 256u + threadIdx.x;
    if (t >= NF) return;
    const uint32_t i = t / T.F, f = t - i * T.F;
    const uint32_t g = AL ? act.gids[i] : i;
    const uint32_t s = AL ? g * T.F + f : t;
    // the group's end-of-step snapshot: what the compact plan fields are relative to
    const int64_t commit_end = in.commit_index[i], term_end = in.current_term[i];
    const uint32_t inc_end = in.incarnation[i];
    const i64x2 last_end = in.last_entry[i], epoch_end = T.g_epoch[g];
    uint32_t b = bits[s];
    if (in.plan_meta) {
        for (uint32_t r = 0; r < rows; r++) {
            const size_t idx = (size_t)r * NF + t;
            const uint64_t pm = in.plan_meta[idx];
            uint32_t pc = 0;
            if constexpr (EL) {
                if (pm == 0) pc = ballot_lane_word(in, (size_t)r * N + i, T.F, term_end, inc_end, last_end, table + s, tinc + s, GF, b);
            }
            if (pm != 0) {
                const uint32_t kind = RAFTING_PLM_KIND(pm), count = RAFTING_PLM_COUNT(pm);
                const i64x2 pp = in.plan_pp[idx], lc = in.plan_lc[idx];
                const int64_t pe = in.plan_epoch[idx];
                uint32_t tag = RAFTING_CTAG_NONE;
                if (kind == RAFTING_PLAN_AE || kind == RAFTING_PLAN_IS) {
                    const uint32_t fr = ~b;
                    if (fr) {
                        tag = (uint32_t)__ffs((int)fr) - 1u; b |= 1u << tag;
                        i64x2 v; v.x = pe; v.y = lc.x; table[(size_t)tag * GF + s] = v; tinc[(size_t)tag * GF + s] = RAFTING_PLM_INC(pm);
                    }
                }
                const uint64_t dcommit = (uint64_t)commit_end - (uint64_t)lc.y;
                uint64_t dprev = 0;
                bool fits = pe == epoch_end.x && RAFTING_PLM_INC(pm) == inc_end && count < 64u;
                [[maybe_unused]] bool older = false;                                // PT: fits kind 7 (then never kind 1)
                [[maybe_unused]] uint64_t gap = 0;                                  // PT: current_term - prevLogTerm
                if (kind == RAFTING_PLAN_AE) {
                    dprev = (uint64_t)last_end.x - (uint64_t)pp.x;
                    if constexpr (PT) {
                        gap = (uint64_t)term_end - (uint64_t)pp.y;
                        older = fits && gap - 1u < 8u && lc.x == (int64_t)((uint64_t)pp.x + count) && dprev < 256u && dcommit < 16u;
                    }
                    fits = fits && pp.y == term_end && lc.x == (int64_t)((uint64_t)pp.x + count) && dprev < 256u && dcommit < 128u;
                } else if (kind == RAFTING_PLAN_IS) {
                    fits = fits && pp.x == epoch_end.x && pp.y == epoch_end.y && lc.x == epoch_end.x && dcommit < 128u;
                } else fits = fits && pp.x == 0 && pp.y == 0 && lc.x == 0 && lc.y == 0;
                pc = kind | ((uint32_t)RAFTING_PLM_HB(pm) << 3) | (tag << 5);
                if (fits) pc |= (count << 11) | ((uint32_t)dprev << 17) | ((kind == RAFTING_PLAN_AE || kind == RAFTING_PLAN_IS) ? ((uint32_t)dcommit << 25) : 0u);
                else if (PT && older)
                    pc |= RAFTING_CPLAN_AE_PREV_TERM | (count << 11) | ((uint32_t)dprev << 17) | ((uint32_t)(gap - 1u) << 25) | ((uint32_t)dcommit << 28);
                else { pc |= 1u << 4; put_escape(out, RAFTING_CESC_PLAN, (uint32_t)idx, pm | ((uint64_t)(tag == RAFTING_CTAG_NONE ? 255u : tag) << 8), pp.x, pp.y, lc.x, lc.y, pe); }
            }
            out.plan_c[idx] = pc;
        }
    } else if constexpr (EL) {
        for (uint32_t r = 0; r < rows; r++)
            out.plan_c[(size_t)r * NF + t] = ballot_lane_word(in, (size_t)r * N + i, T.F, term_end, inc_end, last_end, table + s, tinc + s, GF, b);
    } else {
        for (uint32_t r = 0; r < rows; r++) out.plan_c[(size_t)r * NF + t] = 0;
    }
    bits[s] = b;
    if (f == 0) {
        for (uint32_t r = 0; r < rows; r++) {
            const size_t gi = (size_t)r * N + i;
            const uint32_t rm = in.rep_meta ? in.rep_meta[gi] : 0u;
            uint32_t rc = RAFTING_REP_ERR(rm);
            if (RAFTING_REP_VALID(rm)) {
                atomicAdd(out.counts + 2, 1u);
                const int64_t rt = in.rep_term[gi];
                if (out.compact_replies && rt == term_end) rc |= 0x80u | (RAFTING_REP_SUCCESS(rm) << 6);
                else put_escape(out, RAFTING_CESC_REPLY, (uint32_t)gi, rm, rt, 0, 0, 0, 0);
            }
            out.rep_c[gi] = (uint8_t)rc;
            const uint64_t bm = in.ballot_meta ? in.ballot_meta[gi] : 0ull;
            if constexpr (EL) {
                if (bm != 0) {
                    atomicAdd(out.counts + 1, 1u);
                    if (!ballot_lane_kind(in, gi, T.F, term_end, inc_end, last_end)) {
                        const i64x2 bl = in.ballot_last[gi]; put_escape(out, RAFTING_CESC_BALLOT, (uint32_t)gi, bm, in.ballot_term[gi], bl.x, bl.y, 0, 0);
                    }
                }
            } else {
                if (bm != 0) { atomicAdd(out.counts + 1, 1u); const i64x2 bl = in.ballot_last[gi]; put_escape(out, RAFTING_CESC_BALLOT, (uint32_t)gi, bm, in.ballot_term[gi], bl.x, bl.y, 0, 0); }
            }
        }
        out.commit_index[i] = commit_end; out.current_term[i] = term_end; out.role_word[i] = in.role_word[i];
        out.incarnation[i] = inc_end; out.err_word[i] = in.err_word[i]; out.last_entry[i] = last_end; out.epoch[i] = epoch_end;
    }
}

// the kernel variants of a step: unpack [EL][AL], pack [EL][PT][AL], unpack_requests [EL]
static const decltype(&unpack_kernel<false, false>) UNPACK[2][2] = {
    {unpack_kernel<false, false>, unpack_kernel<false, true>}, {unpack_kernel<true, false>, unpack_kernel<true, true>}};
static const decltype(&pack_kernel<false, false, false>) PACK[2][2][2] = {
    {{pack_kernel<false, false, false>, pack_kernel<false, false, true>}, {pack_kernel<false, true, false>, pack_kernel<false, true, true>}},
    {{pack_kernel<true, false, false>, pack_kernel<true, false, true>}, {pack_kernel<true, true, false>, pack_kernel<true, true, true>}}};
static const decltype(&unpack_requests_kernel<false>) UNPACK_REQUESTS[2] = {unpack_requests_kernel<false>, unpack_requests_kernel<true>};

}  // namespace rafting

struct CompactState {
    rafting::i64x2* table = nullptr;       // [CTAGS][G * F] (epochAtSend, lastIndexAtSend) of the RPC in flight under that tag
    uint32_t* tinc = nullptr;               // [CTAGS][G * F] incarnation of the role object that sent it
    uint32_t* bits = nullptr;               // [G * F] tags in use
};
static void compact_release(rafting_engine* e) { delete e->compact; e->compact = nullptr; }   // the buffers are in dev_allocs
static uint32_t* compact_bits(rafting_engine* e) { return e->compact ? e->compact->bits : nullptr; }
// p is one of the in-flight table's three allocations
static bool compact_owns(const rafting_engine* e, const void* p) {
    return e->compact && (p == e->compact->table || p == e->compact->tinc || p == e->compact->bits);
}
static int compact_state(rafting_engine* e) {
    if (e->compact) return RAFTING_OK;
    CompactState* c = new CompactState();
    const size_t GF = (size_t)e->G * e->F;
    e->alloc_state = true;                  // protocol state: covered by rafting_checkpoint / rafting_restore
    int rc = dalloc(e, &c->table, GF * rafting::CTAGS);
    if (!rc) rc = dalloc(e, &c->tinc, GF * rafting::CTAGS);
    if (!rc) rc = dalloc(e, &c->bits, GF);
    e->alloc_state = false;
    if (rc) { delete c; return rc; }
    e->compact = c;
    return RAFTING_OK;
}

// byte layout of the two wire blocks of a slot (device copy and — for the small items — a pinned landing block)
struct CLayout { size_t row_base, op_c, op_un, ev_c, esc, in_total; size_t plan_c, rep_c, commit, term, role, inc, err, last, epoch, counts, esc_out, out_total; };
static CLayout compact_layout(size_t rows, size_t G, size_t F, size_t n_esc_in, size_t esc_cap) {
    CLayout L; Carve in, out;
    // the optional parts come last, so that the single copy of a block-shaped inbox ends where the launch's data ends
    L.row_base = in.take(rows * 8); L.op_c = in.take(rows * G * 4); L.ev_c = in.take(rows * G * F * 4); L.op_un = in.take(rows * G * 2);
    L.esc = in.take((n_esc_in + 1) * sizeof(rafting_cesc_in_t));
    L.in_total = in.o;
    L.plan_c = out.take(rows * G * F * 4); L.rep_c = out.take(rows * G);
    L.commit = out.take(G * 8); L.term = out.take(G * 8); L.role = out.take(G * 4); L.inc = out.take(G * 4); L.err = out.take(G * 4); L.last = out.take(G * 16); L.epoch = out.take(G * 16);
    L.counts = out.take(16);
    L.esc_out = out.take((esc_cap + 1) * sizeof(rafting_cesc_out_t));
    L.out_total = out.o;
    return L;
}

// Byte offsets of the wire columns inside ONE block per direction, as the engine lays them out on the device.  A caller that
// allocates its pinned inbox / outbox as one block with these offsets gets ONE copy up and ONE copy down per launch instead of
// one per column (the engine recognises the layout from the pointers; any other arrangement still works, column by column).
//   in_off : row_base, op_c, op_unavail, ev_c, esc, total        out_off: plan_c, rep_c, commit_index, current_term, role_word,
//                                                                          incarnation, err_word, last_entry, epoch, counts, esc, total
extern "C" int rafting_compact_layout(uint32_t rows, uint32_t G, uint32_t F, uint32_t n_esc_in, uint32_t esc_cap, uint64_t in_off[6], uint64_t out_off[12]) {
    if (!in_off || !out_off) return fail(RAFTING_E_INVAL, "null argument");
    const CLayout L = compact_layout(rows, G, F, n_esc_in, esc_cap);
    const uint64_t i[6] = {L.row_base, L.op_c, L.op_un, L.ev_c, L.esc, L.in_total};
    const uint64_t o[12] = {L.plan_c, L.rep_c, L.commit, L.term, L.role, L.inc, L.err, L.last, L.epoch, L.counts, L.esc_out, L.out_total};
    for (int k = 0; k < 6; k++) in_off[k] = i[k];
    for (int k = 0; k < 12; k++) out_off[k] = o[k];
    return RAFTING_OK;
}

// the request list's block: records, op escapes, then the entry pool (the device block extends the pool by the records' terms)
struct CRLayout { size_t req, esc, ent, total; };
static CRLayout compact_req_layout(size_t n_req, size_t n_esc, size_t ent_count) {
    CRLayout L; Carve c;
    L.req = c.take(n_req * sizeof(rafting_creq_t)); L.esc = c.take(n_esc * sizeof(rafting_cesc_op_t)); L.ent = c.o;
    L.total = L.ent + ent_count * 8;
    return L;
}
extern "C" int rafting_compact_req_layout(uint32_t n_req, uint32_t n_op_esc, uint32_t ent_count, uint64_t off[4]) {
    if (!off) return fail(RAFTING_E_INVAL, "null argument");
    const CRLayout L = compact_req_layout(n_req, n_op_esc, ent_count);
    off[0] = L.req; off[1] = L.esc; off[2] = L.ent; off[3] = L.total;
    return RAFTING_OK;
}

// One column of a wire block: the caller's memory (absent when null or bytes == 0) and its offset in the engine's layout
struct WireCol { const void* h; size_t at, bytes; };
// The caller's block, or null: a caller that carved its columns from one block with the layout above has every present
// column at its laid-out offset from one base
static uint8_t* wire_block(const WireCol* c, int n) {
    uint8_t* base = nullptr;
    for (int k = 0; k < n; k++) {
        if (!c[k].h || !c[k].bytes) continue;
        uint8_t* b = (uint8_t*)c[k].h - c[k].at;
        if (!base) base = b;
        else if (b != base) return nullptr;
    }
    return base;
}
// Between the caller's columns and the device block dev: ONE copy of the caller's block hb up to the end of its last present
// column, or (hb null) one copy per present column
static int wire_copy(const WireCol* c, int n, uint8_t* hb, uint8_t* dev, cudaMemcpyKind dir, cudaStream_t st) {
    const bool up = dir == cudaMemcpyHostToDevice;
    size_t end = 0;
    for (int k = 0; k < n; k++) {
        if (!c[k].h || !c[k].bytes) continue;
        end = c[k].at + c[k].bytes > end ? c[k].at + c[k].bytes : end;
        if (!hb) CU(cudaMemcpyAsync(up ? dev + c[k].at : (void*)c[k].h, up ? c[k].h : dev + c[k].at, c[k].bytes, dir, st));
    }
    if (hb) CU(cudaMemcpyAsync(up ? (void*)dev : hb, up ? hb : dev, end, dir, st));
    return RAFTING_OK;
}

extern "C" int rafting_step_begin_compact(rafting_engine_t* e, uint32_t slot, const rafting_cinbox_t* in, const rafting_coutbox_t* out) {
    return rafting_step_begin_compact_req(e, slot, in, nullptr, out);
}

extern "C" int rafting_step_begin_compact_req(rafting_engine_t* e, uint32_t slot, const rafting_cinbox_t* in, const rafting_creqs_t* reqs,
                                              const rafting_coutbox_t* out) {
    return rafting_step_begin_compact_ex(e, slot, in, reqs, out, 0u);
}

// the device-chosen tail of a step begun with rafting_step_begin_compact_due (timers.cuh)
struct DueTail { uint32_t n_host, cap; uint32_t* tail_out; };

// The list is checked in full before anything is enqueued: a lane's tag bitmap must have exactly one owning thread, and the
// in-flight table is indexed by gid, so a duplicate or an id past max_groups would race on it or index past it.
static int check_active_list(rafting_engine_t* e, uint32_t n_active, const uint32_t* gids) {
    if (!e || !gids) return fail(RAFTING_E_INVAL, "bad argument");
    if (n_active == 0) return fail(RAFTING_E_INVAL, "an active list holds at least one group");
    if (n_active > e->G) return fail(RAFTING_E_CAPACITY, "n_active %u > max_groups %u", n_active, e->G);
    for (uint32_t k = 0; k < n_active; k++) {
        if (gids[k] >= e->G) return fail(RAFTING_E_INVAL, "gids[%u] = %u is not below max_groups", k, gids[k]);
        if (k > 0 && gids[k] <= gids[k - 1]) return fail(RAFTING_E_INVAL, "gids must be strictly increasing (gids[%u] = %u)", k, gids[k]);
    }
    return RAFTING_OK;
}

// One compact step: its arguments, what compact_check found, and the slot's blocks and staging views compact_reserve made
struct CompactStep {
    const rafting_cinbox_t* in; const rafting_creqs_t* reqs; const rafting_coutbox_t* out;
    const uint32_t* gids; const int64_t* sweep; const DueTail* due;
    size_t rows, n, n_listed;                    // n: groups per row of the step; n_listed: entries of gids the host wrote
    bool list, has_reqs, has_sweep, el, pt;
    size_t n_req, n_oesc, ent_esc, pool;         // records, op escapes, entries the host sends, the step's entry pool
    Layout LD; CLayout LC; CRLayout LR;          // dense staging, wire blocks, request block
    DueLayout LT;                                // a due step's tail selection (S.ctail)
    size_t w_counts, w_offs, w_tmp, scan_tmp;    // the request scan's scratch (S.creqw): order word, counts, offsets, CUB's
    size_t sweep_at;                             // offset of the sweep column in the staged copy of [gids | pad] sweep
    rafting_inbox_t din; rafting_outbox_t dout;  // the dense staging views the step kernel works on
};

// Every refusal of a compact step, before anything is enqueued (the slot stays free); fills the step's shape into p
static int compact_check(rafting_engine_t* e, uint32_t slot, uint32_t flags, uint32_t n_active, CompactStep& p) {
    const rafting_cinbox_t* in = p.in; const rafting_creqs_t* reqs = p.reqs; const rafting_coutbox_t* out = p.out; const DueTail* due = p.due;
    if (!e || !in || !out || slot >= RAFTING_HOST_SLOTS || (due && (!p.sweep || !due->tail_out || (due->n_host && !p.gids))))
        return fail(RAFTING_E_INVAL, "bad argument");
    if (p.sweep) for (uint32_t r = 0; r < in->rows && r < e->cfg.max_rows; r++) p.has_sweep |= p.sweep[r] != 0;
    if (due) {
        if (due->cap == 0) return fail(RAFTING_E_INVAL, "a due step's tail holds at least one group (cap >= 1)");
        if ((uint64_t)due->n_host + due->cap > e->G)
            return fail(RAFTING_E_CAPACITY, "n_host %u + cap %u > max_groups %u: not enough groups outside the list to fill the tail", due->n_host, due->cap, e->G);
        if (due->n_host) { if (int rc = check_active_list(e, due->n_host, p.gids)) return rc; }
        if (!p.has_sweep) return fail(RAFTING_E_INVAL, "a due step needs a sweep row");
    }
    if (flags & ~(RAFTING_COMPACT_ELECTIONS | RAFTING_COMPACT_PREV_TERM)) return fail(RAFTING_E_INVAL, "unknown compact step flags 0x%x", flags);
    p.el = (flags & RAFTING_COMPACT_ELECTIONS) != 0; p.pt = (flags & RAFTING_COMPACT_PREV_TERM) != 0;
    p.has_reqs = reqs && (reqs->n_req || reqs->n_op_esc);
    if (!in->row_base || (!in->op_c && !in->ev_c && !p.has_reqs && !p.has_sweep))
        return fail(RAFTING_E_INVAL, "compact inbox needs row_base and at least one of op_c / ev_c / a request / a sweep row");
    if (reqs && ((reqs->n_req && !reqs->req) || (reqs->n_op_esc && !reqs->op_esc) || (reqs->ent_count && !reqs->ent_terms)))
        return fail(RAFTING_E_INVAL, "request list: a count without its array");
    if (reqs && (uint64_t)reqs->ent_count + reqs->req_entries > e->cfg.entry_pool_cap)
        return fail(RAFTING_E_CAPACITY, "ent_count + req_entries > entry_pool_cap");
    if (in->n_esc && !in->esc) return fail(RAFTING_E_INVAL, "n_esc without esc");
    if (!out->plan_c || !out->rep_c || !out->commit_index || !out->current_term || !out->role_word || !out->incarnation ||
        !out->err_word || !out->last_entry || !out->epoch || !out->counts || (out->esc_cap && !out->esc))
        return fail(RAFTING_E_INVAL, "compact outbox: every column is required");
    if (e->F > 16) return fail(RAFTING_E_CAPACITY, "the compact path carries a 16-lane unavailable mask: use the dense path for larger clusters");
    if (in->op_unavail && !in->op_c) return fail(RAFTING_E_INVAL, "op_unavail without op_c");
    CU(cudaSetDevice(e->cfg.device));
    int rc = hostpath_init(e); if (rc) return rc;
    if ((rc = compact_state(e))) return rc;
    const Slot& S = hp(e)->slot[slot];
    if (S.leased) return fail(RAFTING_E_BUSY, "slot %u is held by an outstanding lease", slot);
    if (S.inflight) return fail(RAFTING_E_BUSY, "slot %u has a step in flight", slot);
    if (S.gathering) return fail(RAFTING_E_BUSY, "slot %u: the gather of its plans has not been waited for", slot);
    p.list = p.gids != nullptr || due != nullptr;
    const size_t rows = in->rows, n = p.list ? n_active : e->G, F = e->F;
    p.rows = rows; p.n = n; p.n_listed = due ? due->n_host : n;
    if (rows == 0 || rows > e->cfg.max_rows) return fail(RAFTING_E_CAPACITY, "rows %zu beyond max_rows %u", rows, e->cfg.max_rows);
    p.n_req = p.has_reqs ? reqs->n_req : 0; p.n_oesc = p.has_reqs ? reqs->n_op_esc : 0;
    if (p.has_reqs && (uint64_t)rows * n * F >= (1ull << 32)) return fail(RAFTING_E_CAPACITY, "rows * groups * followers must stay below 2^32 per step");
    if (p.n_req > rows * n || p.n_oesc > rows * n || p.n_req > 0x7fffffffu)
        return fail(RAFTING_E_INVAL, "a request list longer than rows * n cannot be strictly increasing");
    // A sweep row's op slot belongs to the sweep: the step would drop a request placed there without a trace.  A due step
    // (always with a sweep row) chooses its tail's groups on the device: nothing the host sends can name one of their positions.
    for (size_t k = 0; p.has_sweep && k < p.n_req + p.n_oesc; k++) {
        const uint32_t at = k < p.n_req ? reqs->req[k].slot : reqs->op_esc[k - p.n_req].slot;
        const char* what = k < p.n_req ? "request record" : "op escape";
        const size_t j = k < p.n_req ? k : k - p.n_req;
        if (at < rows * n && p.sweep[at / n] != 0) return fail(RAFTING_E_INVAL, "%s %zu (slot %u) lies on sweep row %zu", what, j, at, (size_t)(at / n));
        if (at < rows * n && due && at % n >= p.n_listed) return fail(RAFTING_E_INVAL, "%s %zu (slot %u) lies at tail position %zu", what, j, at, (size_t)(at % n));
    }
    for (uint32_t k = 0; due && k < in->n_esc; k++) {
        const uint32_t at = in->esc[k].slot;
        if (at < rows * n * F && (at / F) % n >= p.n_listed)
            return fail(RAFTING_E_INVAL, "escape record %u (slot %u) lies at tail position %zu", k, at, (size_t)((at / F) % n));
    }
    p.ent_esc = p.has_reqs ? reqs->ent_count : 0; p.pool = p.has_reqs ? p.ent_esc + reqs->req_entries : 0;
    return RAFTING_OK;
}

// The slot's blocks for the step, and the dense staging views the step kernel works on
static int compact_reserve(rafting_engine_t* e, Slot& S, CompactStep& p) {
    const size_t rows = p.rows, n = p.n, F = e->F;
    // the entry pool lives in the request block; with an active list the group columns are positional
    // (RAFTING_INBOX_COMPACT_GROUPS) and the list itself travels in the gids column
    p.LD = make_layout(rows, n, F, n, p.list ? n : 0, 0);
    p.LC = compact_layout(rows, n, F, p.in->n_esc, p.out->esc_cap);
    p.LR = compact_req_layout(p.n_req, p.n_oesc, p.ent_esc);
    if (p.n_req) CU(cub::DeviceScan::ExclusiveSum(nullptr, p.scan_tmp, (const uint64_t*)nullptr, (uint64_t*)nullptr, (int)p.n_req));
    Carve w; w.take(4); p.w_counts = w.take(p.n_req * 8); p.w_offs = w.take(p.n_req * 8); p.w_tmp = w.o;
    int rc;
    if ((rc = blk_reserve(S.din, p.LD.in_total, false)) || (rc = blk_reserve(S.dout, p.LD.out_total, false)) ||
        (rc = blk_reserve(S.cin, p.LC.in_total, false)) || (rc = blk_reserve(S.cout, p.LC.out_total, false)) ||
        (rc = blk_reserve(S.chout, 256 + (p.due ? (size_t)p.due->cap * 4 : 0), true))) return rc;
    if (p.due && ((rc = due_layout(e->G, p.LT)) || (rc = blk_reserve(S.ctail, p.LT.total, false)))) return rc;
    if (p.has_reqs && ((rc = blk_reserve(S.creq, p.LR.ent + p.pool * 8, false)) || (rc = blk_reserve(S.creqw, p.w_tmp + p.scan_tmp, false)))) return rc;
    rafting_inbox_t& d = p.din = stage_inbox(p.LD, S.din.p);
    if (!p.list) d.gids = nullptr;
    if (!p.has_sweep) d.row_now = nullptr;
    if (!p.in->op_c && !p.has_reqs) { d.op_meta = nullptr; d.op_nr = nullptr; }
    if (!p.in->op_unavail && !p.has_reqs) d.op_ab = nullptr;                // nobody is unavailable
    if (!p.has_reqs) { d.op_cd = nullptr; d.op_e = nullptr; }
    d.ent_terms = p.has_reqs ? (const int64_t*)(S.creq.p + p.LR.ent) : nullptr;
    if (!p.in->ev_c && !p.in->n_esc) { d.ev_meta = nullptr; d.ev_tn = nullptr; d.ev_el = nullptr; }
    d.rows = (uint32_t)rows; d.n_active = p.list ? (uint32_t)n : 0; d.ent_count = (uint32_t)p.pool;
    d.flags = (p.has_reqs ? 0u : RAFTING_INBOX_NO_REQUESTS) | (p.list ? RAFTING_INBOX_COMPACT_GROUPS : 0u);
    p.dout = stage_outbox(p.LD, S.dout.p, nullptr, d.op_meta || d.row_now);
    // the sweep column travels in the copy of the list (whole shard: alone), staged in the slot's pinned block so that the copy
    // is asynchronous whatever memory the caller's column lives in
    p.sweep_at = p.list && p.has_sweep ? (size_t)((const uint8_t*)d.row_now - (const uint8_t*)d.gids) : 0;
    if (p.has_sweep && (rc = blk_reserve(S.chin, p.sweep_at + rows * 8, true))) return rc;
    return RAFTING_OK;
}

// H2D on the slot's copy stream: the wire columns as they are, the request list, the active list and the sweep column
static int compact_upload(rafting_engine_t* e, Slot& S, const CompactStep& p) {
    HostPath* H = hp(e);
    const rafting_cinbox_t* in = p.in; const rafting_creqs_t* q = p.reqs; const CLayout& LC = p.LC;
    const size_t rows = p.rows, n = p.n;
    const WireCol cols[] = {{in->row_base, LC.row_base, rows * 8}, {in->op_c, LC.op_c, rows * n * 4}, {in->ev_c, LC.ev_c, rows * n * e->F * 4},
                            {in->op_unavail, LC.op_un, rows * n * 2}, {in->esc, LC.esc, (size_t)in->n_esc * sizeof(rafting_cesc_in_t)}};
    // only an inbox with both op_c and ev_c counts as a block: its one copy spans every column before the last present one
    if (int rc = wire_copy(cols, 5, in->op_c && in->ev_c ? wire_block(cols, 5) : nullptr, S.cin.p, cudaMemcpyHostToDevice, H->s_h2d)) return rc;
    if (p.has_reqs) {                                                          // the request list: one copy when carved as laid out
        const WireCol rcols[] = {{q->req, p.LR.req, p.n_req * sizeof(rafting_creq_t)}, {q->op_esc, p.LR.esc, p.n_oesc * sizeof(rafting_cesc_op_t)},
                                 {q->ent_terms, p.LR.ent, p.ent_esc * 8}};
        if (int rc = wire_copy(rcols, 3, wire_block(rcols, 3), S.creq.p, cudaMemcpyHostToDevice, H->s_h2d)) return rc;
    }
    if (p.has_sweep) {                                                         // [gids | pad] sweep: one copy
        if (p.list && p.n_listed) memcpy(S.chin.p, p.gids, p.n_listed * 4);
        memcpy(S.chin.p + p.sweep_at, p.sweep, rows * 8);
        CU(cudaMemcpyAsync((uint8_t*)p.din.row_now - p.sweep_at, S.chin.p, p.sweep_at + rows * 8, cudaMemcpyHostToDevice, H->s_h2d));
    } else if (p.list) {
        CU(cudaMemcpyAsync((void*)p.din.gids, p.gids, n * 4, cudaMemcpyHostToDevice, H->s_h2d));
    }
    CU(cudaEventRecord(S.ev_h2d, H->s_h2d));
    return RAFTING_OK;
}

// unpack -> step -> pack on the engine's stream, behind the slot's H2D copies
static int compact_run(rafting_engine_t* e, Slot& S, const CompactStep& p) {
    using namespace rafting;
    const rafting_cinbox_t* in = p.in; const CLayout& LC = p.LC;
    const size_t rows = p.rows, NF = p.n * e->F;
    CInD ci; ci.rows = (uint32_t)rows; ci.n_esc = in->n_esc;
    ci.row_base = (const int64_t*)(S.cin.p + LC.row_base); ci.esc = (const rafting_cesc_in_t*)(S.cin.p + LC.esc);
    ci.op_c = in->op_c ? (const uint32_t*)(S.cin.p + LC.op_c) : nullptr;
    ci.op_unavail = in->op_unavail ? (const uint16_t*)(S.cin.p + LC.op_un) : nullptr;
    ci.ev_c = in->ev_c ? (const uint32_t*)(S.cin.p + LC.ev_c) : nullptr;
    InboxD di; OutboxD dov;
    to_dev_views(&p.din, &p.dout, e->G, (uint32_t*)(S.dout.p + p.LD.flags_off), di, dov);
    ActiveD act; act.gids = di.gids; act.n = (uint32_t)p.n;
    COutD co;
    co.plan_c = (uint32_t*)(S.cout.p + LC.plan_c); co.rep_c = (uint8_t*)(S.cout.p + LC.rep_c);
    co.commit_index = (int64_t*)(S.cout.p + LC.commit); co.current_term = (int64_t*)(S.cout.p + LC.term); co.role_word = (uint32_t*)(S.cout.p + LC.role);
    co.incarnation = (uint32_t*)(S.cout.p + LC.inc); co.err_word = (uint32_t*)(S.cout.p + LC.err); co.last_entry = (i64x2*)(S.cout.p + LC.last);
    co.epoch = (i64x2*)(S.cout.p + LC.epoch); co.counts = (uint32_t*)(S.cout.p + LC.counts);
    co.esc = (rafting_cesc_out_t*)(S.cout.p + LC.esc_out); co.esc_cap = p.out->esc_cap; co.compact_replies = p.reqs != nullptr;
    const uint32_t blocks = (uint32_t)((NF + 255u) / 256u);
    CU(cudaStreamWaitEvent(e->stream, S.ev_h2d, 0));
    CU(cudaMemsetAsync(dov.flags, 0, 16, e->stream));
    CU(cudaMemsetAsync(co.counts, 0, 16, e->stream));
    if (p.due) {                                                               // the tail of the list, and counts[3]
        int64_t until = 0;
        for (size_t r = 0; r < rows; r++) until = p.sweep[r] > until ? p.sweep[r] : until;
        uint32_t* list = (uint32_t*)act.gids;
        if (int rc = due_select(e, p.LT, S.ctail.p, until, list, p.due->n_host, list + p.due->n_host, p.due->cap, true, co.counts + 3, nullptr)) return rc;
    }
    InboxW dw;                                                                // unpack writes what the step kernel reads
    dw.op_meta = (uint64_t*)di.op_meta; dw.op_nr = (i64x2*)di.op_nr; dw.op_ab = (i64x2*)di.op_ab;
    dw.ev_meta = (uint64_t*)di.ev_meta; dw.ev_tn = (i64x2*)di.ev_tn; dw.ev_el = (i64x2*)di.ev_el;
    dw.op_cd = (i64x2*)di.op_cd; dw.op_e = (int64_t*)di.op_e; dw.ent_terms = (int64_t*)di.ent_terms;
    UNPACK[p.el][p.list]<<<blocks, 256, 0, e->stream>>>(e->T, ci, dw, e->compact->table, e->compact->tinc, e->compact->bits, act);
    if (in->ev_c == nullptr && in->n_esc) CU(cudaMemsetAsync((void*)di.ev_meta, 0, rows * NF * 8, e->stream));
    if (in->n_esc) unpack_escapes_kernel<<<(in->n_esc + 255u) / 256u, 256, 0, e->stream>>>(ci, dw, (uint32_t)(rows * NF));
    if (p.has_reqs) {
        CReqD q;
        q.n_req = (uint32_t)p.n_req; q.n_esc = (uint32_t)p.n_oesc; q.slots = (uint32_t)(rows * p.n);
        q.req = (const rafting_creq_t*)(S.creq.p + p.LR.req); q.esc = (const rafting_cesc_op_t*)(S.creq.p + p.LR.esc);
        q.row_base = ci.row_base; q.op_c = ci.op_c;
        q.ent_count = (uint32_t)p.ent_esc; q.pool_end = (uint32_t)p.pool;
        q.order = (uint32_t*)S.creqw.p; q.counts = (uint64_t*)(S.creqw.p + p.w_counts); q.offs = (uint64_t*)(S.creqw.p + p.w_offs);
        const uint32_t most = (uint32_t)(p.n_req > p.n_oesc ? p.n_req : p.n_oesc);
        CU(cudaMemsetAsync(q.order, 0, 4, e->stream));
        creq_prepare_kernel<<<(most + 255u) / 256u, 256, 0, e->stream>>>(q);
        if (p.n_req) { size_t tb = p.scan_tmp; CU(cub::DeviceScan::ExclusiveSum(S.creqw.p + p.w_tmp, tb, q.counts, q.offs, (int)p.n_req, e->stream)); }
        UNPACK_REQUESTS[p.el]<<<(uint32_t)((p.n_req + p.n_oesc + 255u) / 256u), 256, 0, e->stream>>>(q, dw, (uint32_t)p.n);
    }
    CU(cudaGetLastError());
    if (int rc = launch_step(e, di, dov, e->stream)) return rc;
    PACK[p.el][p.pt][p.list]<<<blocks, 256, 0, e->stream>>>(e->T, (uint32_t)rows, dov, co, e->compact->table, e->compact->tinc, e->compact->bits, act);
    CU(cudaGetLastError());
    CU(cudaEventRecord(S.ev_kernel, e->stream));
    return RAFTING_OK;
}

// One compact step in `slot`: over the whole shard (gids == nullptr, n = G), or over the n groups gids[0 .. n) that the caller
// has checked (strictly increasing, each < G).  Every wire column and every dense staging column holds n groups per row.
// sweep (host, [rows], may be null): the step's row_now column (rafting_step_begin_compact_sweep).
// due (rafting_step_begin_compact_due): gids holds due->n_host entries and n_active = n_host + cap; the device writes the
// rest of the list before unpack_kernel reads it.
static int compact_begin(rafting_engine_t* e, uint32_t slot, const rafting_cinbox_t* in, const rafting_creqs_t* reqs,
                         const rafting_coutbox_t* out, uint32_t flags, uint32_t n_active, const uint32_t* gids,
                         const int64_t* sweep = nullptr, const DueTail* due = nullptr) {
    CompactStep p = {in, reqs, out, gids, sweep, due};
    int rc = compact_check(e, slot, flags, n_active, p);
    if (rc || (rc = compact_reserve(e, hp(e)->slot[slot], p))) return rc;   // refused: nothing is enqueued, the slot stays free
    HostPath* H = hp(e); Slot& S = H->slot[slot];
    if ((rc = compact_upload(e, S, p)) || (rc = compact_run(e, S, p))) { cudaStreamSynchronize(H->s_h2d); return rc; }
    // ---- D2H: every wire column + the counters; the escape list only when the counters say it holds something ----
    // the first escape records always travel with the columns (a steady-state launch produces a handful): fetching them
    // on demand at wait time would have to drain the D2H stream, i.e. wait for the copies of every LATER launch as well
    CU(cudaStreamWaitEvent(H->s_d2h, S.ev_kernel, 0));
    const CLayout& LC = p.LC; const size_t rows = p.rows, n = p.n;
    const uint32_t esc_inline = out->esc_cap < rafting::CESC_INLINE ? out->esc_cap : rafting::CESC_INLINE;
    WireCol cols[] = {{out->plan_c, LC.plan_c, rows * n * e->F * 4}, {out->rep_c, LC.rep_c, rows * n}, {out->commit_index, LC.commit, n * 8},
                      {out->current_term, LC.term, n * 8}, {out->role_word, LC.role, n * 4}, {out->incarnation, LC.inc, n * 4},
                      {out->err_word, LC.err, n * 4}, {out->last_entry, LC.last, n * 16}, {out->epoch, LC.epoch, n * 16},
                      {out->counts, LC.counts, 16}, {out->esc, LC.esc_out, (size_t)esc_inline * sizeof(rafting_cesc_out_t)}};
    WireCol& counts = cols[9];
    uint8_t* hb = wire_block(cols, 11);
    if (!hb) counts.h = S.chout.p;                                            // column by column: into the slot's pinned block
    if ((rc = wire_copy(cols, 11, hb, S.cout.p, cudaMemcpyDeviceToHost, H->s_d2h))) return rc;
    if (due) CU(cudaMemcpyAsync(S.chout.p + 256, p.din.gids + due->n_host, (size_t)due->cap * 4, cudaMemcpyDeviceToHost, H->s_d2h));
    CU(cudaEventRecord(S.ev_done, H->s_d2h));
    S.compact_step = true; S.c_host = *out; S.c_counts_pinned = (uint32_t*)counts.h; S.c_esc_dev = S.cout.p + LC.esc_out;
    S.c_tail_user = due ? due->tail_out : nullptr; S.c_tail_n = due ? due->cap : 0;
    S.dev_out = p.dout; S.rows_ = rows; S.n_ = n; S.c_gids = p.list ? p.din.gids : nullptr;
    S.inflight = true;
    return RAFTING_OK;
}

extern "C" int rafting_step_begin_compact_ex(rafting_engine_t* e, uint32_t slot, const rafting_cinbox_t* in, const rafting_creqs_t* reqs,
                                             const rafting_coutbox_t* out, uint32_t flags) {
    return compact_begin(e, slot, in, reqs, out, flags, 0, nullptr);
}

extern "C" int rafting_step_begin_compact_active(rafting_engine_t* e, uint32_t slot, uint32_t n_active, const uint32_t* gids,
                                                 const rafting_cinbox_t* in, const rafting_creqs_t* reqs, const rafting_coutbox_t* out,
                                                 uint32_t flags) {
    if (int rc = check_active_list(e, n_active, gids)) return rc;
    return compact_begin(e, slot, in, reqs, out, flags, n_active, gids);
}

// The dense step with row_now = sweep, over the whole shard (gids == NULL) or an active list
extern "C" int rafting_step_begin_compact_sweep(rafting_engine_t* e, uint32_t slot, uint32_t n_active, const uint32_t* gids, const int64_t* sweep,
                                                const rafting_cinbox_t* in, const rafting_creqs_t* reqs, const rafting_coutbox_t* out,
                                                uint32_t flags) {
    if (gids) { if (int rc = check_active_list(e, n_active, gids)) return rc; }
    return compact_begin(e, slot, in, reqs, out, flags, n_active, gids, sweep);
}

// A sweep step over gids[0 .. n_host) followed by cap gids chosen on the device: the groups outside gids that the sweep
// fires, lowest first, then groups that are not due (fillers)
extern "C" int rafting_step_begin_compact_due(rafting_engine_t* e, uint32_t slot, uint32_t n_host, const uint32_t* gids, uint32_t cap,
                                              const int64_t* sweep, const rafting_cinbox_t* in, const rafting_creqs_t* reqs,
                                              const rafting_coutbox_t* out, uint32_t* tail_out, uint32_t flags) {
    const DueTail due = {n_host, cap, tail_out};
    return compact_begin(e, slot, in, reqs, out, flags, n_host + cap, gids, sweep, &due);
}

extern "C" int rafting_step_wait_compact(rafting_engine_t* e, uint32_t slot) {
    if (!e || slot >= RAFTING_HOST_SLOTS) return fail(RAFTING_E_INVAL, "bad argument");
    CU(cudaSetDevice(e->cfg.device));
    HostPath* H = hp(e); Slot& S = H->slot[slot];
    if (!S.inflight) return RAFTING_OK;
    if (!S.compact_step) return fail(RAFTING_E_INVAL, "slot %u holds a dense step (use rafting_step_wait_slot)", slot);
    CU(cudaEventSynchronize(S.ev_done));
    S.inflight = false;
    if (S.c_counts_pinned != S.c_host.counts) for (int k = 0; k < 4; k++) S.c_host.counts[k] = S.c_counts_pinned[k];
    if (S.c_tail_user) { memcpy(S.c_tail_user, S.chout.p + 256, (size_t)S.c_tail_n * 4); S.c_tail_user = nullptr; }
    const uint32_t n = S.c_counts_pinned[0] < S.c_host.esc_cap ? S.c_counts_pinned[0] : S.c_host.esc_cap;
    if (n > CESC_INLINE) {                                                    // rare: more than the records that travelled with the columns
        CU(cudaMemcpyAsync(S.c_host.esc + CESC_INLINE, (const rafting_cesc_out_t*)S.c_esc_dev + CESC_INLINE,
                           (size_t)(n - CESC_INLINE) * sizeof(rafting_cesc_out_t), cudaMemcpyDeviceToHost, H->s_d2h));
        CU(cudaStreamSynchronize(H->s_d2h));
    }
    return RAFTING_OK;
}

extern "C" int rafting_step_fetch_dense(rafting_engine_t* e, uint32_t slot, const rafting_outbox_t* out) {
    if (!e || !out || slot >= RAFTING_HOST_SLOTS) return fail(RAFTING_E_INVAL, "bad argument");
    CU(cudaSetDevice(e->cfg.device));
    HostPath* H = hp(e); Slot& S = H->slot[slot];
    if (!S.compact_step || S.inflight) return fail(RAFTING_E_INVAL, "slot %u: no finished compact step to fetch", slot);
    for (int k = 0; k < N_OUT; k++) {
        const ColDesc& c = OUT_COLS[k];
        void* h = out_ptr(out, c); void* d = out_ptr(&S.dev_out, c);
        if (!h || !d) continue;
        CU(cudaMemcpyAsync(h, d, col_bytes(c, S.rows_, S.n_, e->F, S.n_, 0, 0), cudaMemcpyDeviceToHost, H->s_d2h));
    }
    CU(cudaStreamSynchronize(H->s_d2h));
    return RAFTING_OK;
}
