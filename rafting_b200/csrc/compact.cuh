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

__global__ void __launch_bounds__(256) unpack_kernel(Tables T, CInD in, InboxW out, const i64x2* __restrict__ table, const uint32_t* __restrict__ tinc, uint32_t* __restrict__ bits) {
    const uint32_t GF = T.G * T.F;
    const uint32_t t = blockIdx.x * 256u + threadIdx.x;
    if (t >= GF) return;
    const uint32_t g = t / T.F, f = t - g * T.F;
    if (in.ev_c) {
        const int64_t term_now = T.g_term[g];
        uint32_t b = bits[t];
        for (uint32_t r = 0; r < in.rows; r++) {
            const size_t idx = (size_t)r * GF + t;
            const uint32_t w = in.ev_c[idx];
            const uint32_t kind = w & 0xfu;
            uint64_t em = 0;
            if (kind == RAFTING_EV_AE_ACK || kind == RAFTING_EV_IS_ACK) {
                const uint32_t tag = (w >> 8) & 0xffu;
                i64x2 el = {0, 0}; uint32_t inc = 0;
                if (tag < (uint32_t)CTAGS) { el = table[(size_t)tag * GF + t]; inc = tinc[(size_t)tag * GF + t]; b &= ~(1u << tag); }
                i64x2 tn; tn.x = ((w >> 7) & 1u) ? term_now : 0; tn.y = in.row_base[r] + (int64_t)(w >> 16);
                em = (uint64_t)(w & 0x7fu) | ((uint64_t)inc << 32);         // kind | outcome | success | incarnation (from the table)
                out.ev_tn[idx] = tn; out.ev_el[idx] = el;
            }
            out.ev_meta[idx] = em;                                          // escaped / empty slots read as "no event" until patched
        }
        bits[t] = b;
    }
    if (f == 0 && (in.op_c || out.op_cd)) {
        for (uint32_t r = 0; r < in.rows; r++) {
            const size_t gi = (size_t)r * T.G + g;
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
    uint32_t n_req, n_esc, slots;                // slots = rows * G
    const rafting_creq_t* req; const rafting_cesc_op_t* esc;
    const int64_t* row_base; const uint32_t* op_c;
    uint32_t ent_count, pool_end;                // records' terms start at ent_count; the step's pool ends at pool_end
    uint64_t* counts; uint64_t* offs;            // [n_req] entry count of each record, its exclusive scan
    uint32_t* order;                             // bit 0: req decreases somewhere, bit 1: esc does
};
constexpr uint32_t CREQ_META_ZERO = 0xf800u;     // bits 11..15 of a record's meta

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
__global__ void unpack_requests_kernel(CReqD q, InboxW o, uint32_t G) {
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if ((uint64_t)k >= (uint64_t)q.n_req + q.n_esc) return;
    const bool is_req = k < q.n_req;
    const uint32_t j = is_req ? k : k - q.n_req;
    const uint32_t slot = is_req ? q.req[j].slot : q.esc[j].slot;
    if (slot >= q.slots) return;
    const uint32_t r = slot / G;
    bool bad = q.order[0] != 0 || (q.op_c && (q.op_c[slot] & 0xfu) != RAFTING_OP_NONE);
    if (is_req) {
        bad = bad || (j > 0 && q.req[j - 1].slot == slot) || (j + 1 < q.n_req && q.req[j + 1].slot == slot) ||
              list_holds(q.esc, q.n_esc, slot) || (q.req[j].meta & CREQ_META_ZERO) != 0;
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

__global__ void __launch_bounds__(256) pack_kernel(Tables T, uint32_t rows, OutboxD in, COutD out, i64x2* __restrict__ table, uint32_t* __restrict__ tinc, uint32_t* __restrict__ bits) {
    const uint32_t GF = T.G * T.F;
    const uint32_t t = blockIdx.x * 256u + threadIdx.x;
    if (t >= GF) return;
    const uint32_t g = t / T.F, f = t - g * T.F;
    // the group's end-of-step snapshot: what the compact plan fields are relative to
    const int64_t commit_end = in.commit_index[g], term_end = in.current_term[g];
    const uint32_t inc_end = in.incarnation[g];
    const i64x2 last_end = in.last_entry[g], epoch_end = T.g_epoch[g];
    uint32_t b = bits[t];
    if (in.plan_meta) {
        for (uint32_t r = 0; r < rows; r++) {
            const size_t idx = (size_t)r * GF + t;
            const uint64_t pm = in.plan_meta[idx];
            uint32_t pc = 0;
            if (pm != 0) {
                const uint32_t kind = RAFTING_PLM_KIND(pm), count = RAFTING_PLM_COUNT(pm);
                const i64x2 pp = in.plan_pp[idx], lc = in.plan_lc[idx];
                const int64_t pe = in.plan_epoch[idx];
                uint32_t tag = RAFTING_CTAG_NONE;
                if (kind == RAFTING_PLAN_AE || kind == RAFTING_PLAN_IS) {
                    const uint32_t fr = ~b;
                    if (fr) {
                        tag = (uint32_t)__ffs((int)fr) - 1u; b |= 1u << tag;
                        i64x2 v; v.x = pe; v.y = lc.x; table[(size_t)tag * GF + t] = v; tinc[(size_t)tag * GF + t] = RAFTING_PLM_INC(pm);
                    }
                }
                const uint64_t dcommit = (uint64_t)commit_end - (uint64_t)lc.y;
                uint64_t dprev = 0;
                bool fits = pe == epoch_end.x && RAFTING_PLM_INC(pm) == inc_end && count < 64u;
                if (kind == RAFTING_PLAN_AE) {
                    dprev = (uint64_t)last_end.x - (uint64_t)pp.x;
                    fits = fits && pp.y == term_end && lc.x == (int64_t)((uint64_t)pp.x + count) && dprev < 256u && dcommit < 128u;
                } else if (kind == RAFTING_PLAN_IS) {
                    fits = fits && pp.x == epoch_end.x && pp.y == epoch_end.y && lc.x == epoch_end.x && dcommit < 128u;
                } else fits = fits && pp.x == 0 && pp.y == 0 && lc.x == 0 && lc.y == 0;
                pc = kind | ((uint32_t)RAFTING_PLM_HB(pm) << 3) | (tag << 5);
                if (fits) pc |= (count << 11) | ((uint32_t)dprev << 17) | ((kind == RAFTING_PLAN_AE || kind == RAFTING_PLAN_IS) ? ((uint32_t)dcommit << 25) : 0u);
                else { pc |= 1u << 4; put_escape(out, RAFTING_CESC_PLAN, (uint32_t)idx, pm | ((uint64_t)(tag == RAFTING_CTAG_NONE ? 255u : tag) << 8), pp.x, pp.y, lc.x, lc.y, pe); }
            }
            out.plan_c[idx] = pc;
        }
    } else {
        for (uint32_t r = 0; r < rows; r++) out.plan_c[(size_t)r * GF + t] = 0;
    }
    bits[t] = b;
    if (f == 0) {
        for (uint32_t r = 0; r < rows; r++) {
            const size_t gi = (size_t)r * T.G + g;
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
            if (bm != 0) { atomicAdd(out.counts + 1, 1u); const i64x2 bl = in.ballot_last[gi]; put_escape(out, RAFTING_CESC_BALLOT, (uint32_t)gi, bm, in.ballot_term[gi], bl.x, bl.y, 0, 0); }
        }
        out.commit_index[g] = commit_end; out.current_term[g] = term_end; out.role_word[g] = in.role_word[g];
        out.incarnation[g] = inc_end; out.err_word[g] = in.err_word[g]; out.last_entry[g] = last_end; out.epoch[g] = epoch_end;
    }
}

}  // namespace rafting

struct CompactState {
    rafting::i64x2* table = nullptr;       // [CTAGS][G * F] (epochAtSend, lastIndexAtSend) of the RPC in flight under that tag
    uint32_t* tinc = nullptr;               // [CTAGS][G * F] incarnation of the role object that sent it
    uint32_t* bits = nullptr;               // [G * F] tags in use
};
static void compact_release(rafting_engine* e) { delete e->compact; e->compact = nullptr; }   // the buffers are in dev_allocs
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
struct CLayout { size_t row_base, op_c, op_un, ev_c, esc, in_total; size_t plan_c, rep_c, commit, term, role, inc, err, last, epoch, counts, esc_out, out_total, out_dense; };
static CLayout compact_layout(size_t rows, size_t G, size_t F, size_t n_esc_in, size_t esc_cap) {
    CLayout L; size_t o = 0;
    auto take = [&](size_t bytes) { const size_t at = o; o += (bytes + 255) & ~(size_t)255; return at; };
    // the optional parts come last, so that the single copy of a block-shaped inbox ends where the launch's data ends
    L.row_base = take(rows * 8); L.op_c = take(rows * G * 4); L.ev_c = take(rows * G * F * 4); L.op_un = take(rows * G * 2);
    L.esc = take((n_esc_in + 1) * sizeof(rafting_cesc_in_t));
    L.in_total = o; o = 0;
    L.plan_c = take(rows * G * F * 4); L.rep_c = take(rows * G);
    L.commit = take(G * 8); L.term = take(G * 8); L.role = take(G * 4); L.inc = take(G * 4); L.err = take(G * 4); L.last = take(G * 16); L.epoch = take(G * 16);
    L.counts = take(16);
    L.out_dense = o;                                                          // everything before the escape list travels down every step
    L.esc_out = take((esc_cap + 1) * sizeof(rafting_cesc_out_t));
    L.out_total = o;
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
    CRLayout L; size_t o = 0;
    auto take = [&](size_t bytes) { const size_t at = o; o += (bytes + 255) & ~(size_t)255; return at; };
    L.req = take(n_req * sizeof(rafting_creq_t)); L.esc = take(n_esc * sizeof(rafting_cesc_op_t)); L.ent = o; o += ent_count * 8;
    L.total = o;
    return L;
}
extern "C" int rafting_compact_req_layout(uint32_t n_req, uint32_t n_op_esc, uint32_t ent_count, uint64_t off[4]) {
    if (!off) return fail(RAFTING_E_INVAL, "null argument");
    const CRLayout L = compact_req_layout(n_req, n_op_esc, ent_count);
    off[0] = L.req; off[1] = L.esc; off[2] = L.ent; off[3] = L.total;
    return RAFTING_OK;
}

extern "C" int rafting_step_begin_compact(rafting_engine_t* e, uint32_t slot, const rafting_cinbox_t* in, const rafting_coutbox_t* out) {
    return rafting_step_begin_compact_req(e, slot, in, nullptr, out);
}

extern "C" int rafting_step_begin_compact_req(rafting_engine_t* e, uint32_t slot, const rafting_cinbox_t* in, const rafting_creqs_t* reqs,
                                              const rafting_coutbox_t* out) {
    using namespace rafting;
    if (!e || !in || !out || slot >= RAFTING_HOST_SLOTS) return fail(RAFTING_E_INVAL, "bad argument");
    const bool has_reqs = reqs && (reqs->n_req || reqs->n_op_esc);
    if (!in->row_base || (!in->op_c && !in->ev_c && !has_reqs))
        return fail(RAFTING_E_INVAL, "compact inbox needs row_base and at least one of op_c / ev_c / a request");
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
    HostPath* H = hp(e); Slot& S = H->slot[slot];
    if (S.leased) return fail(RAFTING_E_BUSY, "slot %u is held by an outstanding lease", slot);
    if (S.inflight) return fail(RAFTING_E_BUSY, "slot %u has a step in flight", slot);
    const size_t rows = in->rows, G = e->G, F = e->F;
    if (rows == 0 || rows > e->cfg.max_rows) return fail(RAFTING_E_CAPACITY, "rows %zu beyond max_rows %u", rows, e->cfg.max_rows);
    const size_t n_req = has_reqs ? reqs->n_req : 0, n_oesc = has_reqs ? reqs->n_op_esc : 0;
    if (has_reqs && (uint64_t)rows * G * F >= (1ull << 32)) return fail(RAFTING_E_CAPACITY, "rows * groups * followers must stay below 2^32 per step");
    if (n_req > rows * G || n_oesc > rows * G || n_req > 0x7fffffffu)
        return fail(RAFTING_E_INVAL, "a request list longer than rows * G cannot be strictly increasing");
    const size_t ent_esc = has_reqs ? reqs->ent_count : 0, pool = has_reqs ? ent_esc + reqs->req_entries : 0;
    const Layout LD = make_layout(rows, G, F, G, 0, 0);                        // dense staging the step kernel works on (the
                                                                               // entry pool lives in the request block)
    const CLayout LC = compact_layout(rows, G, F, in->n_esc, out->esc_cap);
    const CRLayout LR = compact_req_layout(n_req, n_oesc, ent_esc);
    size_t scan_tmp = 0;
    if (n_req) CU(cub::DeviceScan::ExclusiveSum(nullptr, scan_tmp, (const uint64_t*)nullptr, (uint64_t*)nullptr, (int)n_req));
    const size_t w_counts = 256, w_offs = w_counts + ((n_req * 8 + 255) & ~(size_t)255), w_tmp = w_offs + ((n_req * 8 + 255) & ~(size_t)255);
    if ((rc = blk_reserve(S.din, LD.in_total, false)) || (rc = blk_reserve(S.dout, LD.out_total, false)) ||
        (rc = blk_reserve(S.cin, LC.in_total, false)) || (rc = blk_reserve(S.cout, LC.out_total, false)) ||
        (rc = blk_reserve(S.chout, 256, true))) return rc;
    if (has_reqs && ((rc = blk_reserve(S.creq, LR.ent + pool * 8, false)) || (rc = blk_reserve(S.creqw, w_tmp + scan_tmp, false)))) return rc;
    // ---- H2D: the wire columns as they are ----
    CInD ci; ci.rows = (uint32_t)rows; ci.n_esc = in->n_esc;
    ci.row_base = (const int64_t*)(S.cin.p + LC.row_base); ci.op_c = nullptr; ci.op_unavail = nullptr; ci.ev_c = nullptr;
    ci.esc = (const rafting_cesc_in_t*)(S.cin.p + LC.esc);
    {
        const uint8_t* hb = (const uint8_t*)in->row_base - LC.row_base;      // where the block would start on the host
        const bool one_block = (!in->op_c || (const uint8_t*)in->op_c == hb + LC.op_c) && (!in->op_unavail || (const uint8_t*)in->op_unavail == hb + LC.op_un) &&
                               (!in->ev_c || (const uint8_t*)in->ev_c == hb + LC.ev_c) && (!in->n_esc || (const uint8_t*)in->esc == hb + LC.esc) &&
                               in->op_c && in->ev_c;
        if (one_block) {
            const size_t span = in->n_esc ? LC.esc + (size_t)in->n_esc * sizeof(rafting_cesc_in_t)
                                : (in->op_unavail ? LC.op_un + rows * G * 2 : LC.ev_c + rows * G * F * 4);
            CU(cudaMemcpyAsync(S.cin.p, hb, span, cudaMemcpyHostToDevice, H->s_h2d));
            ci.op_c = (const uint32_t*)(S.cin.p + LC.op_c); ci.ev_c = (const uint32_t*)(S.cin.p + LC.ev_c);
            if (in->op_unavail) ci.op_unavail = (const uint16_t*)(S.cin.p + LC.op_un);
        } else {
            CU(cudaMemcpyAsync(S.cin.p + LC.row_base, in->row_base, rows * 8, cudaMemcpyHostToDevice, H->s_h2d));
            if (in->op_c) { CU(cudaMemcpyAsync(S.cin.p + LC.op_c, in->op_c, rows * G * 4, cudaMemcpyHostToDevice, H->s_h2d)); ci.op_c = (const uint32_t*)(S.cin.p + LC.op_c); }
            if (in->op_c && in->op_unavail) { CU(cudaMemcpyAsync(S.cin.p + LC.op_un, in->op_unavail, rows * G * 2, cudaMemcpyHostToDevice, H->s_h2d)); ci.op_unavail = (const uint16_t*)(S.cin.p + LC.op_un); }
            if (in->ev_c) { CU(cudaMemcpyAsync(S.cin.p + LC.ev_c, in->ev_c, rows * G * F * 4, cudaMemcpyHostToDevice, H->s_h2d)); ci.ev_c = (const uint32_t*)(S.cin.p + LC.ev_c); }
            if (in->n_esc) CU(cudaMemcpyAsync(S.cin.p + LC.esc, in->esc, (size_t)in->n_esc * sizeof(rafting_cesc_in_t), cudaMemcpyHostToDevice, H->s_h2d));
        }
    }
    if (has_reqs) {                                                            // the request list: one copy when carved as laid out
        const uint8_t* hb = n_req ? (const uint8_t*)reqs->req - LR.req : (const uint8_t*)reqs->op_esc - LR.esc;
        const bool one_block = (!n_req || (const uint8_t*)reqs->req == hb + LR.req) && (!n_oesc || (const uint8_t*)reqs->op_esc == hb + LR.esc) &&
                               (!ent_esc || (const uint8_t*)reqs->ent_terms == hb + LR.ent);
        if (one_block) CU(cudaMemcpyAsync(S.creq.p, hb, LR.total, cudaMemcpyHostToDevice, H->s_h2d));
        else {
            if (n_req) CU(cudaMemcpyAsync(S.creq.p + LR.req, reqs->req, n_req * sizeof(rafting_creq_t), cudaMemcpyHostToDevice, H->s_h2d));
            if (n_oesc) CU(cudaMemcpyAsync(S.creq.p + LR.esc, reqs->op_esc, n_oesc * sizeof(rafting_cesc_op_t), cudaMemcpyHostToDevice, H->s_h2d));
            if (ent_esc) CU(cudaMemcpyAsync(S.creq.p + LR.ent, reqs->ent_terms, ent_esc * 8, cudaMemcpyHostToDevice, H->s_h2d));
        }
    }
    CU(cudaEventRecord(S.ev_h2d, H->s_h2d));
    // ---- unpack -> step -> pack on the engine's stream ----
    InboxD di; memset(&di, 0, sizeof(di));
    di.rows = (uint32_t)rows; di.n = (uint32_t)G; di.flags = has_reqs ? 0u : RAFTING_INBOX_NO_REQUESTS;
    if (in->op_c || has_reqs) {
        di.op_meta = (const uint64_t*)(S.din.p + LD.in_off[2]); di.op_nr = (const i64x2*)(S.din.p + LD.in_off[3]);
        if (in->op_unavail || has_reqs) di.op_ab = (const i64x2*)(S.din.p + LD.in_off[4]);   // else nobody is unavailable
    }
    if (has_reqs) {
        di.op_cd = (const i64x2*)(S.din.p + LD.in_off[5]); di.op_e = (const int64_t*)(S.din.p + LD.in_off[6]);
        di.ent_terms = (const int64_t*)(S.creq.p + LR.ent); di.ent_count = (uint32_t)pool;
    }
    if (in->ev_c || in->n_esc) {
        di.ev_meta = (const uint64_t*)(S.din.p + LD.in_off[8]); di.ev_tn = (const i64x2*)(S.din.p + LD.in_off[9]); di.ev_el = (const i64x2*)(S.din.p + LD.in_off[10]);
    }
    OutboxD dov; memset(&dov, 0, sizeof(dov));
    dov.rep_meta = (uint32_t*)(S.dout.p + LD.out_off[0]); dov.rep_term = (int64_t*)(S.dout.p + LD.out_off[1]);
    dov.plan_meta = (uint64_t*)(S.dout.p + LD.out_off[2]); dov.plan_pp = (i64x2*)(S.dout.p + LD.out_off[3]);
    dov.plan_lc = (i64x2*)(S.dout.p + LD.out_off[4]); dov.plan_epoch = (int64_t*)(S.dout.p + LD.out_off[5]);
    dov.ballot_meta = (uint64_t*)(S.dout.p + LD.out_off[6]); dov.ballot_term = (int64_t*)(S.dout.p + LD.out_off[7]);
    dov.ballot_last = (i64x2*)(S.dout.p + LD.out_off[8]); dov.commit_index = (int64_t*)(S.dout.p + LD.out_off[9]);
    dov.current_term = (int64_t*)(S.dout.p + LD.out_off[10]); dov.role_word = (uint32_t*)(S.dout.p + LD.out_off[11]);
    dov.incarnation = (uint32_t*)(S.dout.p + LD.out_off[12]); dov.err_word = (uint32_t*)(S.dout.p + LD.out_off[13]);
    dov.last_entry = (i64x2*)(S.dout.p + LD.out_off[14]);
    dov.flags = (uint32_t*)(S.dout.p + LD.flags_off);
    if (!in->op_c && !has_reqs) { dov.rep_meta = nullptr; dov.rep_term = nullptr; dov.plan_meta = nullptr; dov.plan_pp = nullptr; dov.plan_lc = nullptr; dov.plan_epoch = nullptr; }
    COutD co;
    co.plan_c = (uint32_t*)(S.cout.p + LC.plan_c); co.rep_c = (uint8_t*)(S.cout.p + LC.rep_c);
    co.commit_index = (int64_t*)(S.cout.p + LC.commit); co.current_term = (int64_t*)(S.cout.p + LC.term); co.role_word = (uint32_t*)(S.cout.p + LC.role);
    co.incarnation = (uint32_t*)(S.cout.p + LC.inc); co.err_word = (uint32_t*)(S.cout.p + LC.err); co.last_entry = (i64x2*)(S.cout.p + LC.last);
    co.epoch = (i64x2*)(S.cout.p + LC.epoch); co.counts = (uint32_t*)(S.cout.p + LC.counts);
    co.esc = (rafting_cesc_out_t*)(S.cout.p + LC.esc_out); co.esc_cap = out->esc_cap; co.compact_replies = reqs != nullptr;
    const uint32_t GF = (uint32_t)(G * F), blocks = (GF + 255u) / 256u;
    CU(cudaStreamWaitEvent(e->stream, S.ev_h2d, 0));
    CU(cudaMemsetAsync(dov.flags, 0, 16, e->stream));
    CU(cudaMemsetAsync(co.counts, 0, 16, e->stream));
    InboxW dw;                                                                 // unpack writes what the step kernel reads
    dw.op_meta = (uint64_t*)di.op_meta; dw.op_nr = (i64x2*)di.op_nr; dw.op_ab = (i64x2*)di.op_ab;
    dw.ev_meta = (uint64_t*)di.ev_meta; dw.ev_tn = (i64x2*)di.ev_tn; dw.ev_el = (i64x2*)di.ev_el;
    dw.op_cd = (i64x2*)di.op_cd; dw.op_e = (int64_t*)di.op_e; dw.ent_terms = (int64_t*)di.ent_terms;
    unpack_kernel<<<blocks, 256, 0, e->stream>>>(e->T, ci, dw, e->compact->table, e->compact->tinc, e->compact->bits);
    if (in->ev_c == nullptr && in->n_esc) CU(cudaMemsetAsync((void*)di.ev_meta, 0, rows * G * F * 8, e->stream));
    if (in->n_esc) unpack_escapes_kernel<<<(in->n_esc + 255u) / 256u, 256, 0, e->stream>>>(ci, dw, (uint32_t)(rows * G * F));
    if (has_reqs) {
        CReqD q;
        q.n_req = (uint32_t)n_req; q.n_esc = (uint32_t)n_oesc; q.slots = (uint32_t)(rows * G);
        q.req = (const rafting_creq_t*)(S.creq.p + LR.req); q.esc = (const rafting_cesc_op_t*)(S.creq.p + LR.esc);
        q.row_base = ci.row_base; q.op_c = ci.op_c;
        q.ent_count = (uint32_t)ent_esc; q.pool_end = (uint32_t)pool;
        q.order = (uint32_t*)S.creqw.p; q.counts = (uint64_t*)(S.creqw.p + w_counts); q.offs = (uint64_t*)(S.creqw.p + w_offs);
        const uint32_t most = (uint32_t)(n_req > n_oesc ? n_req : n_oesc);
        CU(cudaMemsetAsync(q.order, 0, 4, e->stream));
        creq_prepare_kernel<<<(most + 255u) / 256u, 256, 0, e->stream>>>(q);
        if (n_req) { size_t tb = scan_tmp; CU(cub::DeviceScan::ExclusiveSum(S.creqw.p + w_tmp, tb, q.counts, q.offs, (int)n_req, e->stream)); }
        unpack_requests_kernel<<<(uint32_t)((n_req + n_oesc + 255u) / 256u), 256, 0, e->stream>>>(q, dw, (uint32_t)G);
    }
    CU(cudaGetLastError());
    rc = launch_step(e, di, dov, e->stream);
    if (rc) { cudaStreamSynchronize(H->s_h2d); return rc; }
    pack_kernel<<<blocks, 256, 0, e->stream>>>(e->T, (uint32_t)rows, dov, co, e->compact->table, e->compact->tinc, e->compact->bits);
    CU(cudaGetLastError());
    CU(cudaEventRecord(S.ev_kernel, e->stream));
    // ---- D2H: every wire column + the counters; the escape list only when the counters say it holds something ----
    CU(cudaStreamWaitEvent(H->s_d2h, S.ev_kernel, 0));
    const uint32_t esc_inline = out->esc_cap < CESC_INLINE ? out->esc_cap : CESC_INLINE;
    uint32_t* counts_land = (uint32_t*)S.chout.p;
    {
        uint8_t* hb = (uint8_t*)out->plan_c - LC.plan_c;
        const bool one_block = (uint8_t*)out->rep_c == hb + LC.rep_c && (uint8_t*)out->commit_index == hb + LC.commit && (uint8_t*)out->current_term == hb + LC.term &&
                               (uint8_t*)out->role_word == hb + LC.role && (uint8_t*)out->incarnation == hb + LC.inc && (uint8_t*)out->err_word == hb + LC.err &&
                               (uint8_t*)out->last_entry == hb + LC.last && (uint8_t*)out->epoch == hb + LC.epoch && (uint8_t*)out->counts == hb + LC.counts &&
                               (!out->esc_cap || (uint8_t*)out->esc == hb + LC.esc_out);
        if (one_block) {
            // columns, counters and the first escape records: one copy (the counters land in the caller's block directly)
            CU(cudaMemcpyAsync(hb, S.cout.p, LC.esc_out + (size_t)esc_inline * sizeof(rafting_cesc_out_t), cudaMemcpyDeviceToHost, H->s_d2h));
            counts_land = out->counts;
        } else {
            CU(cudaMemcpyAsync(out->plan_c, co.plan_c, rows * G * F * 4, cudaMemcpyDeviceToHost, H->s_d2h));
            CU(cudaMemcpyAsync(out->rep_c, co.rep_c, rows * G, cudaMemcpyDeviceToHost, H->s_d2h));
            CU(cudaMemcpyAsync(out->commit_index, co.commit_index, G * 8, cudaMemcpyDeviceToHost, H->s_d2h));
            CU(cudaMemcpyAsync(out->current_term, co.current_term, G * 8, cudaMemcpyDeviceToHost, H->s_d2h));
            CU(cudaMemcpyAsync(out->role_word, co.role_word, G * 4, cudaMemcpyDeviceToHost, H->s_d2h));
            CU(cudaMemcpyAsync(out->incarnation, co.incarnation, G * 4, cudaMemcpyDeviceToHost, H->s_d2h));
            CU(cudaMemcpyAsync(out->err_word, co.err_word, G * 4, cudaMemcpyDeviceToHost, H->s_d2h));
            CU(cudaMemcpyAsync(out->last_entry, co.last_entry, G * 16, cudaMemcpyDeviceToHost, H->s_d2h));
            CU(cudaMemcpyAsync(out->epoch, co.epoch, G * 16, cudaMemcpyDeviceToHost, H->s_d2h));
            CU(cudaMemcpyAsync(S.chout.p, co.counts, 16, cudaMemcpyDeviceToHost, H->s_d2h));
            // the first escape records always travel with the columns (a steady-state launch produces a handful): fetching them
            // on demand at wait time would have to drain the D2H stream, i.e. wait for the copies of every LATER launch as well
            if (esc_inline) CU(cudaMemcpyAsync(out->esc, co.esc, (size_t)esc_inline * sizeof(rafting_cesc_out_t), cudaMemcpyDeviceToHost, H->s_d2h));
        }
    }
    CU(cudaEventRecord(S.ev_done, H->s_d2h));
    S.compact_step = true; S.c_host = *out; S.c_counts_pinned = counts_land; S.c_esc_dev = co.esc;
    S.dev_out = rafting_outbox_t(); memset(&S.dev_out, 0, sizeof(S.dev_out));
    S.dev_out.rep_meta = dov.rep_meta; S.dev_out.rep_term = dov.rep_term; S.dev_out.plan_meta = dov.plan_meta;
    S.dev_out.plan_pp = (rafting_i64x2_t*)dov.plan_pp; S.dev_out.plan_lc = (rafting_i64x2_t*)dov.plan_lc; S.dev_out.plan_epoch = dov.plan_epoch;
    S.dev_out.ballot_meta = dov.ballot_meta; S.dev_out.ballot_term = dov.ballot_term; S.dev_out.ballot_last = (rafting_i64x2_t*)dov.ballot_last;
    S.dev_out.commit_index = dov.commit_index; S.dev_out.current_term = dov.current_term; S.dev_out.role_word = dov.role_word;
    S.dev_out.incarnation = dov.incarnation; S.dev_out.err_word = dov.err_word; S.dev_out.last_entry = (rafting_i64x2_t*)dov.last_entry;
    S.rows_ = rows; S.n_ = G;
    S.inflight = true;
    return RAFTING_OK;
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
        CU(cudaMemcpyAsync(h, d, col_bytes(c, S.rows_, S.n_, e->F, e->G, 0, 0), cudaMemcpyDeviceToHost, H->s_d2h));
    }
    CU(cudaStreamSynchronize(H->s_d2h));
    return RAFTING_OK;
}
