// ingest.cpp — the reference's wire framing, restated for the pump thread (include/rafting_ingest.h).  Host only (g++).
#include "../../include/rafting_ingest.h"

#include <string.h>

#include <algorithm>
#include <deque>
#include <vector>

namespace {
constexpr uint8_t SOH = 0x01, STX = 0x02, ETX = 0x03, EOT = 0x04;          // EventCodec.java:29-32
inline uint32_t be32(const uint8_t* p) { return ((uint32_t)p[0] << 24) | ((uint32_t)p[1] << 16) | ((uint32_t)p[2] << 8) | p[3]; }
inline void put_be32(uint8_t* p, uint32_t v) { p[0] = (uint8_t)(v >> 24); p[1] = (uint8_t)(v >> 16); p[2] = (uint8_t)(v >> 8); p[3] = (uint8_t)v; }
}  // namespace

// FrameDecoder.decode (EventCodec.java:281-334) as a scan over a contiguous buffer: a frame is reported only when all of
// it is present; the decoder's incremental states collapse into "not enough bytes yet -> stop".
extern "C" int rafting_frame_scan(const uint8_t* buf, size_t len, rafting_frame_t* out, uint32_t cap, uint32_t* n,
                                  size_t* consumed, int* transparent) {
    if (!buf || !out || !n || !consumed) return RAFTING_E_INVAL;
    uint32_t cnt = 0; size_t pos = 0;
    if (transparent) *transparent = 0;
    *n = 0; *consumed = 0;
    while (pos < len && cnt < cap) {
        size_t p = pos;
        const uint8_t first = buf[p++];
        if (first == EOT) { if (transparent) *transparent = 1; pos = p; break; }      // verify(buf, SOH, EOT) :299-301
        if (first != SOH) { *n = cnt; *consumed = pos; return RAFTING_E_INVAL; }
        rafting_frame_t f; memset(&f, 0, sizeof(f));
        if (p >= len) break;
        f.type = buf[p++];                                                             // readType :237-242
        f.has_sequence = (f.type == RAFTING_FRAME_ENQ || f.type == RAFTING_FRAME_ACK) ? 1 : 0;
        if (f.has_sequence) {
            if (len - p < 4) break;
            f.sequence = (int32_t)be32(buf + p); p += 4;                               // readSequence :244-247
        }
        if (len - p < 5) break;
        if (buf[p++] != STX) { *n = cnt; *consumed = pos; return RAFTING_E_INVAL; }     // readHeadLen :249-256
        const uint32_t hl = be32(buf + p); p += 4;
        if ((int32_t)hl < 0 || hl > RAFTING_FRAME_MAX_HEAD) { *n = cnt; *consumed = pos; return RAFTING_E_INVAL; }
        if (len - p < (size_t)hl + 4) break;
        f.head_off = (uint32_t)p; f.head_len = hl; p += hl;
        const uint32_t bl = be32(buf + p); p += 4;                                     // readBodyLen :258-266
        if ((int32_t)bl < 0 || bl > RAFTING_FRAME_MAX_BODY) { *n = cnt; *consumed = pos; return RAFTING_E_INVAL; }
        if (len - p < (size_t)bl + 1) break;
        f.body_off = (uint32_t)p; f.body_len = bl; p += bl;
        if (buf[p++] != ETX) { *n = cnt; *consumed = pos; return RAFTING_E_INVAL; }     // readBody :268-278
        // an Event.Ending frame is followed by EOT (FrameEncoder :193-195): the next "frame start" is the EOT that makes the
        // channel transparent; it is reported with the frame it ends so that the caller sees both at once
        if (p < len && buf[p] == EOT) { f.ending = 1; out[cnt++] = f; pos = p + 1; if (transparent) *transparent = 1; break; }
        out[cnt++] = f; pos = p;
    }
    *n = cnt; *consumed = pos;
    return RAFTING_OK;
}

// FrameEncoder.encode — EventCodec.java:171-201
extern "C" size_t rafting_frame_encode(uint8_t* dst, size_t cap, uint8_t type, int has_sequence, int32_t sequence,
                                       const char* head, uint32_t head_len, const void* body, uint32_t body_len, int ending) {
    if (!dst || head_len > RAFTING_FRAME_MAX_HEAD || body_len > RAFTING_FRAME_MAX_BODY || (head_len && !head) || (body_len && !body)) return 0;
    const size_t need = 2 + (has_sequence ? 4 : 0) + 1 + 4 + head_len + 4 + body_len + 1 + (ending ? 1 : 0);
    if (need > cap) return 0;
    uint8_t* p = dst;
    *p++ = SOH; *p++ = type;
    if (has_sequence) { put_be32(p, (uint32_t)sequence); p += 4; }
    *p++ = STX;
    put_be32(p, head_len); p += 4;
    if (head_len) { memcpy(p, head, head_len); p += head_len; }
    put_be32(p, body_len); p += 4;
    if (body_len) { memcpy(p, body, body_len); p += body_len; }
    *p++ = ETX;
    if (ending) *p++ = EOT;
    return (size_t)(p - dst);
}

// NettyNode.parseContextId / prepareLocalInvocation dispatch — NettyNode.java:92-107,109-158
extern "C" int rafting_scope_parse(const char* head, uint32_t head_len, uint32_t* op_kind, uint32_t* ctx_off) {
    if (!head || !op_kind || !ctx_off) return RAFTING_E_INVAL;
    static const struct { const char* name; uint32_t kind; } M[] = {
        {"appendEntries", RAFTING_OP_AE_REQUEST}, {"preVote", RAFTING_OP_PREVOTE_REQ},
        {"requestVote", RAFTING_OP_VOTE_REQ}, {"installSnapshot", RAFTING_OP_IS_REQUEST}};
    for (const auto& m : M) {
        const size_t k = strlen(m.name);
        // startsWith(method name), then the context id begins one character further (the ':')
        if (head_len >= k && memcmp(head, m.name, k) == 0) {
            if (head_len < k + 1) return RAFTING_E_INVAL;          // substring(k + 1) of a shorter string throws
            *op_kind = m.kind; *ctx_off = (uint32_t)k + 1;
            return RAFTING_OK;
        }
    }
    return RAFTING_E_INVAL;
}

// contextId -> gid: an open-addressing table over the key bytes (FNV-1a), looked up straight from the receive buffer — no
// std::string per frame (a lookup per ACK frame is the hot part of rafting_ack_frames_decode).
struct rafting_ctxmap {
    struct Slot { uint64_t hash = 0; uint32_t off = 0, len = 0, gid = 0; bool used = false; };
    std::vector<Slot> slots;
    std::vector<char> keys;
    size_t count = 0;
    static uint64_t fnv(const char* p, uint32_t n) {
        uint64_t h = 1469598103934665603ull;
        for (uint32_t i = 0; i < n; i++) { h ^= (uint8_t)p[i]; h *= 1099511628211ull; }
        return h;
    }
    const Slot* find(const char* p, uint32_t n, uint64_t h) const {
        if (slots.empty()) return nullptr;
        const size_t mask = slots.size() - 1;
        for (size_t i = h & mask;; i = (i + 1) & mask) {
            const Slot& s = slots[i];
            if (!s.used) return nullptr;
            if (s.hash == h && s.len == n && (n == 0 || memcmp(keys.data() + s.off, p, n) == 0)) return &s;
        }
    }
    void place(const Slot& s) {
        const size_t mask = slots.size() - 1;
        size_t i = s.hash & mask;
        while (slots[i].used) i = (i + 1) & mask;
        slots[i] = s;
    }
    void grow() {
        std::vector<Slot> old;
        old.swap(slots);
        slots.assign(old.empty() ? 64 : old.size() * 2, Slot());
        for (const Slot& s : old) if (s.used) place(s);
    }
    void put(const char* p, uint32_t n, uint32_t gid) {
        const uint64_t h = fnv(p, n);
        if (Slot* s = const_cast<Slot*>(find(p, n, h))) { s->gid = gid; return; }
        if ((count + 1) * 2 > slots.size()) grow();
        Slot s; s.hash = h; s.off = (uint32_t)keys.size(); s.len = n; s.gid = gid; s.used = true;
        keys.insert(keys.end(), p, p + n);
        place(s); count++;
    }
};
extern "C" int rafting_ctxmap_create(rafting_ctxmap_t** out) {
    if (!out) return RAFTING_E_INVAL;
    try { *out = new rafting_ctxmap(); } catch (...) { return RAFTING_E_NOMEM; }
    return RAFTING_OK;
}
extern "C" int rafting_ctxmap_destroy(rafting_ctxmap_t* m) { delete m; return RAFTING_OK; }
extern "C" int rafting_ctxmap_put(rafting_ctxmap_t* m, const char* ctx, uint32_t len, uint32_t gid) {
    if (!m || (!ctx && len)) return RAFTING_E_INVAL;
    try { m->put(ctx ? ctx : "", len, gid); } catch (...) { return RAFTING_E_NOMEM; }
    return RAFTING_OK;
}
extern "C" int rafting_ctxmap_get(const rafting_ctxmap_t* m, const char* ctx, uint32_t len, uint32_t* gid) {
    if (!m || !gid || (!ctx && len)) return RAFTING_E_INVAL;
    const rafting_ctxmap::Slot* s = m->find(ctx ? ctx : "", len, rafting_ctxmap::fnv(ctx ? ctx : "", len));
    if (!s) return RAFTING_E_INVAL;
    *gid = s->gid;
    return RAFTING_OK;
}

// ---- reply bodies: kryo.writeClassAndObject(RaftResponse) of kryo 4.0.2, restated (see the header; parity unpinned) ----
static const char RESPONSE_CLASS[] = "io.lubricant.consensus.raft.RaftResponse";      // RaftResponse.java:1,9
static constexpr size_t RESPONSE_CLASS_LEN = sizeof(RESPONSE_CLASS) - 1;
static_assert(RESPONSE_CLASS_LEN > 1 && RESPONSE_CLASS_LEN < 64, "Output.writeString takes its ASCII form for 1 < length < 64 only");

extern "C" size_t rafting_reply_body_encode(uint8_t* dst, size_t cap, int64_t term, int success) {
    uint8_t tmp[RAFTING_REPLY_BODY_MAX];
    size_t n = 0;
    tmp[n++] = 0x01;                                        // NAME + 2
    tmp[n++] = 0x00;                                        // nameId 0
    memcpy(tmp + n, RESPONSE_CLASS, RESPONSE_CLASS_LEN); n += RESPONSE_CLASS_LEN;
    tmp[n - 1] |= 0x80;                                     // end of an ASCII string
    tmp[n++] = 0x01;                                        // NOT_NULL
    tmp[n++] = success ? 1 : 0;                             // boolean success
    uint64_t z = ((uint64_t)term << 1) ^ (uint64_t)(term >> 63);      // zig-zag (optimizePositive = false)
    for (int k = 0; k < 8 && (z >> 7) != 0; k++) { tmp[n++] = (uint8_t)((z & 0x7F) | 0x80); z >>= 7; }
    tmp[n++] = (uint8_t)z;                                  // the last byte: 7 bits, or all 8 when it is the ninth
    if (!dst || cap < n) return 0;
    memcpy(dst, tmp, n);
    return n;
}

extern "C" int rafting_reply_body_decode(const uint8_t* body, size_t len, int64_t* term, int* success) {
    if (!body || !term || !success) return RAFTING_E_INVAL;
    const size_t fixed = 2 + RESPONSE_CLASS_LEN + 2;
    if (len < fixed + 1 || len > RAFTING_REPLY_BODY_MAX) return RAFTING_E_INVAL;
    if (body[0] != 0x01 || body[1] != 0x00) return RAFTING_E_INVAL;
    if (memcmp(body + 2, RESPONSE_CLASS, RESPONSE_CLASS_LEN - 1) != 0 ||
        body[2 + RESPONSE_CLASS_LEN - 1] != (uint8_t)(RESPONSE_CLASS[RESPONSE_CLASS_LEN - 1] | 0x80)) return RAFTING_E_INVAL;
    size_t p = 2 + RESPONSE_CLASS_LEN;
    if (body[p++] != 0x01) return RAFTING_E_INVAL;          // a back-reference (>= 2) or null (0) cannot open an object graph
    if (body[p] > 1) return RAFTING_E_INVAL;
    const int ok = body[p++];
    uint64_t z = 0; int k = 0;
    for (;; k++) {
        if (p >= len) return RAFTING_E_INVAL;               // ran out inside the varlong
        const uint8_t b = body[p++];
        if (k == 8) { z |= (uint64_t)b << 56; break; }      // ninth byte: 8 bits, never a continuation flag
        z |= (uint64_t)(b & 0x7F) << (7 * k);
        if (!(b & 0x80)) break;
    }
    if (p != len) return RAFTING_E_INVAL;                   // trailing bytes: not this object
    *term = (int64_t)(z >> 1) ^ -(int64_t)(z & 1);
    *success = ok;
    return RAFTING_OK;
}

extern "C" int rafting_ack_frame_decode(const uint8_t* buf, const rafting_frame_t* fr, const rafting_ctxmap_t* map, uint32_t* gid,
                                        uint32_t* ev_kind, int32_t* sequence, int64_t* term, int* success) {
    if (!buf || !fr || !map || !gid || !ev_kind || !sequence || !term || !success) return RAFTING_E_INVAL;
    if (fr->type != RAFTING_FRAME_ACK || !fr->has_sequence) return RAFTING_E_INVAL;
    uint32_t op = 0, off = 0;
    const char* head = (const char*)buf + fr->head_off;
    if (rafting_scope_parse(head, fr->head_len, &op, &off) != RAFTING_OK) return RAFTING_E_INVAL;
    if (rafting_ctxmap_get(map, head + off, fr->head_len - off, gid) != RAFTING_OK) return RAFTING_E_INVAL;
    if (rafting_reply_body_decode(buf + fr->body_off, fr->body_len, term, success) != RAFTING_OK) return RAFTING_E_INVAL;
    *ev_kind = op == RAFTING_OP_AE_REQUEST ? RAFTING_EV_AE_ACK : op == RAFTING_OP_IS_REQUEST ? RAFTING_EV_IS_ACK
             : op == RAFTING_OP_PREVOTE_REQ ? RAFTING_EV_PV_REPLY : RAFTING_EV_RV_REPLY;
    *sequence = fr->sequence;
    return RAFTING_OK;
}

extern "C" int rafting_ack_frames_decode(const uint8_t* buf, const rafting_frame_t* frames, uint32_t n, const rafting_ctxmap_t* map,
                                         rafting_ack_rec_t* out, uint32_t* n_out) {
    if (!buf || (!frames && n) || !map || !out || !n_out) return RAFTING_E_INVAL;
    // The registry lookup is a random access into a table of one slot per hosted context: frames are taken in blocks, the
    // scopes of a block are parsed and their slots prefetched first, then looked up and their bodies decoded.
    constexpr uint32_t BLK = 16;
    uint32_t k = 0;
    for (uint32_t base = 0; base < n; base += BLK) {
        const uint32_t m = n - base < BLK ? n - base : BLK;
        uint32_t op[BLK], off[BLK]; uint64_t h[BLK]; bool ok[BLK];
        for (uint32_t j = 0; j < m; j++) {
            const rafting_frame_t& f = frames[base + j];
            const char* head = (const char*)buf + f.head_off;
            ok[j] = f.type == RAFTING_FRAME_ACK && f.has_sequence && rafting_scope_parse(head, f.head_len, &op[j], &off[j]) == RAFTING_OK;
            if (!ok[j]) continue;
            h[j] = rafting_ctxmap::fnv(head + off[j], f.head_len - off[j]);
            if (!map->slots.empty()) __builtin_prefetch(&map->slots[h[j] & (map->slots.size() - 1)]);
        }
        for (uint32_t j = 0; j < m; j++) {
            if (!ok[j]) continue;
            const rafting_frame_t& f = frames[base + j];
            const char* head = (const char*)buf + f.head_off;
            const rafting_ctxmap::Slot* s = map->find(head + off[j], f.head_len - off[j], h[j]);
            if (!s) continue;
            rafting_ack_rec_t r{};
            int success = 0;
            if (rafting_reply_body_decode(buf + f.body_off, f.body_len, &r.term, &success) != RAFTING_OK) continue;
            r.gid = s->gid;
            r.kind = (uint8_t)(op[j] == RAFTING_OP_AE_REQUEST ? RAFTING_EV_AE_ACK : op[j] == RAFTING_OP_IS_REQUEST ? RAFTING_EV_IS_ACK
                             : op[j] == RAFTING_OP_PREVOTE_REQ ? RAFTING_EV_PV_REPLY : RAFTING_EV_RV_REPLY);
            r.success = (uint8_t)success; r.sequence = f.sequence; r.frame = base + j;
            out[k++] = r;
        }
    }
    *n_out = k;
    return RAFTING_OK;
}

extern "C" int rafting_batch_to_inbox(const rafting_batch_rec_t* recs, uint32_t n, int64_t now_ms, const rafting_inbox_t* in,
                                      uint32_t n_groups, uint32_t F, uint32_t* n_done) {
    if (!recs || !in || !n_done || !in->ev_meta || !in->ev_tn || in->gids) return RAFTING_E_INVAL;
    uint64_t* em = const_cast<uint64_t*>(in->ev_meta);
    rafting_i64x2_t* tn = const_cast<rafting_i64x2_t*>(in->ev_tn);
    rafting_i64x2_t* el = const_cast<rafting_i64x2_t*>(in->ev_el);
    *n_done = 0;
    for (uint32_t k = 0; k < n; k++) {
        const rafting_batch_rec_t& r = recs[k];
        if (r.gid >= n_groups || r.lane >= F || r.row >= in->rows || r.kind == RAFTING_EV_NONE || r.kind > RAFTING_EV_RV_REPLY)
            return RAFTING_E_INVAL;
        const size_t li = ((size_t)r.row * n_groups + r.gid) * F + r.lane;
        if (RAFTING_EVM_KIND(em[li]) != RAFTING_EV_NONE) return RAFTING_E_INVAL;       // one event per (row, group, lane)
        em[li] = RAFTING_EVM_MAKE(r.kind, r.flags & 3u, (r.flags >> 2) & 1u, r.incarnation);
        tn[li].x = r.term; tn[li].y = now_ms;
        if (el) { el[li].x = r.epoch_at_send; el[li].y = r.last_at_send; }
        *n_done = k + 1;
    }
    return RAFTING_OK;
}

// ---- the pump's dispatch loop (INTEGRATION.md §4) in C: outbox -> request records, records -> op slots ----
struct rafting_dispatch {
    uint32_t G, F, slot;
    static constexpr int KEEP = 4;                           // role objects per group whose term is remembered
    std::vector<uint32_t> inc; std::vector<int64_t> term; std::vector<uint8_t> used, next;
    int64_t* find(uint32_t g, uint32_t incarnation) {
        for (int k = 0; k < KEEP; k++) if (used[g * KEEP + k] && inc[g * KEEP + k] == incarnation) return &term[g * KEEP + k];
        return nullptr;
    }
    void learn(uint32_t g, uint32_t incarnation, int64_t t) {
        if (int64_t* p = find(g, incarnation)) { *p = t; return; }
        const uint32_t k = g * KEEP + next[g];
        inc[k] = incarnation; term[k] = t; used[k] = 1; next[g] = (uint8_t)((next[g] + 1) % KEEP);
    }
};
extern "C" int rafting_dispatch_create(uint32_t n_groups, uint32_t F, uint32_t local_slot, rafting_dispatch_t** out) {
    if (!out || !n_groups || !F || local_slot > F) return RAFTING_E_INVAL;
    try {
        auto* d = new rafting_dispatch();
        d->G = n_groups; d->F = F; d->slot = local_slot;
        d->inc.assign((size_t)n_groups * rafting_dispatch::KEEP, 0); d->term.assign((size_t)n_groups * rafting_dispatch::KEEP, 0);
        d->used.assign((size_t)n_groups * rafting_dispatch::KEEP, 0); d->next.assign(n_groups, 0);
        *out = d;
    } catch (...) { return RAFTING_E_NOMEM; }
    return RAFTING_OK;
}
extern "C" int rafting_dispatch_destroy(rafting_dispatch_t* d) { delete d; return RAFTING_OK; }

extern "C" int rafting_outbox_to_requests(rafting_dispatch_t* d, const rafting_outbox_t* ob, uint32_t rows, rafting_req_rec_t* out,
                                          uint32_t cap, uint32_t* n_out, uint32_t* n_unknown) {
    if (!d || !ob || !out || !n_out || !ob->incarnation || !ob->current_term) return RAFTING_E_INVAL;
    if (ob->plan_meta && (!ob->plan_pp || !ob->plan_lc)) return RAFTING_E_INVAL;
    if (ob->ballot_meta && (!ob->ballot_term || !ob->ballot_last)) return RAFTING_E_INVAL;
    const uint32_t G = d->G, F = d->F;
    for (uint32_t g = 0; g < G; g++) d->learn(g, ob->incarnation[g], ob->current_term[g]);
    uint32_t n = 0, unknown = 0;
    auto slot_of = [&](uint32_t lane) { return (uint8_t)(lane < d->slot ? lane : lane + 1); };
    for (uint32_t r = 0; r < rows; r++) {
        if (ob->plan_meta)
            for (uint32_t g = 0; g < G; g++)
                for (uint32_t f = 0; f < F; f++) {
                    const size_t li = ((size_t)r * G + g) * F + f;
                    const uint64_t pm = ob->plan_meta[li];
                    const uint32_t kind = RAFTING_PLM_KIND(pm);
                    if (kind != RAFTING_PLAN_AE && kind != RAFTING_PLAN_IS) continue;
                    const int64_t* t = d->find(g, RAFTING_PLM_INC(pm));
                    if (!t) { unknown++; continue; }
                    if (n >= cap) { *n_out = n; if (n_unknown) *n_unknown = unknown; return RAFTING_E_CAPACITY; }
                    rafting_req_rec_t q{};
                    q.gid = g; q.kind = kind == RAFTING_PLAN_AE ? RAFTING_OP_AE_REQUEST : RAFTING_OP_IS_REQUEST;
                    q.src_slot = (uint8_t)d->slot; q.dst_slot = slot_of(f); q.row = (uint8_t)r;
                    q.incarnation = RAFTING_PLM_INC(pm); q.count = kind == RAFTING_PLAN_AE ? RAFTING_PLM_COUNT(pm) : 0;
                    q.term = *t; q.a = ob->plan_pp[li].x; q.b = ob->plan_pp[li].y;
                    q.last = ob->plan_lc[li].x; q.commit = kind == RAFTING_PLAN_AE ? ob->plan_lc[li].y : 0;
                    q.epoch = ob->plan_epoch ? ob->plan_epoch[li] : 0;
                    out[n++] = q;
                }
        if (ob->ballot_meta)
            for (uint32_t g = 0; g < G; g++) {
                const size_t gi = (size_t)r * G + g;
                const uint64_t bm = ob->ballot_meta[gi];
                const uint32_t kind = (uint32_t)(bm & 0xFu);
                if (kind == RAFTING_BALLOT_NONE) continue;
                for (uint32_t f = 0; f < F; f++) {
                    if (n >= cap) { *n_out = n; if (n_unknown) *n_unknown = unknown; return RAFTING_E_CAPACITY; }
                    rafting_req_rec_t q{};
                    q.gid = g; q.kind = kind == RAFTING_BALLOT_PREVOTE ? RAFTING_OP_PREVOTE_REQ : RAFTING_OP_VOTE_REQ;
                    q.src_slot = (uint8_t)d->slot; q.dst_slot = slot_of(f); q.row = (uint8_t)r;
                    q.incarnation = (uint32_t)(bm >> 32);
                    q.term = ob->ballot_term[gi]; q.a = ob->ballot_last[gi].x; q.b = ob->ballot_last[gi].y;
                    out[n++] = q;
                }
            }
    }
    *n_out = n; if (n_unknown) *n_unknown = unknown;
    return RAFTING_OK;
}

extern "C" int rafting_request_to_inbox(const rafting_req_rec_t* r, const int64_t* entry_terms, uint32_t row, int64_t now_ms,
                                        int host_result, const rafting_inbox_t* in, uint32_t n_groups, uint32_t ent_cap,
                                        uint32_t* ent_count) {
    if (!r || !in || !in->op_meta || !in->op_nr || !in->op_ab || !in->op_cd || in->gids) return RAFTING_E_INVAL;
    if (r->gid >= n_groups || row >= in->rows) return RAFTING_E_INVAL;
    if (r->kind != RAFTING_OP_AE_REQUEST && r->kind != RAFTING_OP_PREVOTE_REQ && r->kind != RAFTING_OP_VOTE_REQ &&
        r->kind != RAFTING_OP_IS_REQUEST) return RAFTING_E_INVAL;
    const size_t gi = (size_t)row * n_groups + r->gid;
    uint64_t* om = const_cast<uint64_t*>(in->op_meta);
    if (RAFTING_OP_KIND(om[gi]) != RAFTING_OP_NONE) return RAFTING_E_INVAL;               // one op per (row, group)
    rafting_i64x2_t* nr = const_cast<rafting_i64x2_t*>(in->op_nr);
    rafting_i64x2_t* ab = const_cast<rafting_i64x2_t*>(in->op_ab);
    rafting_i64x2_t* cd = const_cast<rafting_i64x2_t*>(in->op_cd);
    uint32_t off = 0, count = 0;
    int64_t d = 0, e = 0;
    if (r->kind == RAFTING_OP_AE_REQUEST) {
        count = r->count;
        if (count > 0xFFFFu || !in->op_e) return RAFTING_E_INVAL;               // checked before anything is written
        if (count) {
            if (!ent_count || !in->ent_terms || !entry_terms || (uint64_t)*ent_count + count > ent_cap) return RAFTING_E_INVAL;
            off = *ent_count;
            memcpy(const_cast<int64_t*>(in->ent_terms) + off, entry_terms, (size_t)count * 8);
            *ent_count = off + count;
        } else if (ent_count) off = *ent_count;
        d = r->commit; e = r->a + 1;                                                         // entries[0].index = prevLogIndex + 1
    } else if (r->kind == RAFTING_OP_IS_REQUEST) d = host_result ? 1 : 0;
    om[gi] = (uint64_t)RAFTING_OP_MAKE(r->kind, r->src_slot, count) | ((uint64_t)off << 32);
    nr[gi].x = now_ms; nr[gi].y = 0;
    ab[gi].x = r->term; ab[gi].y = r->a;
    cd[gi].x = r->b; cd[gi].y = d;
    if (in->op_e) const_cast<int64_t*>(in->op_e)[gi] = e;
    return RAFTING_OK;
}

extern "C" int rafting_outbox_to_replies(const rafting_outbox_t* ob, uint32_t n_groups, uint32_t local_slot,
                                         const rafting_req_rec_t* placed, const uint8_t* placed_row, uint32_t n,
                                         rafting_batch_rec_t* out, uint32_t* n_out) {
    if (!ob || !ob->rep_meta || !ob->rep_term || (!placed && n) || (!placed_row && n) || !out || !n_out) return RAFTING_E_INVAL;
    uint32_t k = 0;
    for (uint32_t i = 0; i < n; i++) {
        const rafting_req_rec_t& q = placed[i];
        if (q.gid >= n_groups || q.src_slot == local_slot) return RAFTING_E_INVAL;
        const size_t gi = (size_t)placed_row[i] * n_groups + q.gid;
        const uint32_t m = ob->rep_meta[gi];
        if (!RAFTING_REP_VALID(m)) continue;
        rafting_batch_rec_t r{};
        r.gid = q.gid;
        r.kind = (uint8_t)(q.kind == RAFTING_OP_AE_REQUEST ? RAFTING_EV_AE_ACK : q.kind == RAFTING_OP_IS_REQUEST ? RAFTING_EV_IS_ACK
                         : q.kind == RAFTING_OP_PREVOTE_REQ ? RAFTING_EV_PV_REPLY : RAFTING_EV_RV_REPLY);
        r.lane = (uint8_t)(local_slot < q.src_slot ? local_slot : local_slot - 1);      // this node's lane in the sender's numbering
        r.flags = (uint8_t)(RAFTING_OUT_OK | (RAFTING_REP_SUCCESS(m) << 2));
        r.incarnation = q.incarnation;
        r.term = ob->rep_term[gi];
        r.epoch_at_send = q.epoch; r.last_at_send = q.last;
        out[k++] = r;
    }
    *n_out = k;
    return RAFTING_OK;
}

// ---- the same two ends of the loop for the compact host path (rafting_creqs_t in, rep_c out) ----
namespace {
template <typename Rec> uint32_t lower_slot(const Rec* v, uint32_t n, uint32_t slot) {
    uint32_t lo = 0, hi = n;
    while (lo < hi) { const uint32_t m = (lo + hi) / 2; if (v[m].slot < slot) lo = m + 1; else hi = m; }
    return lo;
}
// inserts x at its place in a strictly increasing list (appending when the pump places in slot order)
template <typename Rec> void insert_at(Rec* v, uint32_t* n, uint32_t at, const Rec& x) {
    if (at < *n) memmove(v + at + 1, v + at, (size_t)(*n - at) * sizeof(Rec));
    v[at] = x; (*n)++;
}
}  // namespace

extern "C" int rafting_request_to_creq(const rafting_req_rec_t* r, const int64_t* entry_terms, uint32_t row, int64_t now_ms,
                                       int host_result, const rafting_cinbox_t* in, uint32_t n_groups, rafting_creqs_t* q,
                                       uint32_t req_cap, uint32_t esc_cap, uint32_t ent_cap) {
    if (!r || !in || !in->row_base || !q || (q->n_req && !q->req) || (q->n_op_esc && !q->op_esc)) return RAFTING_E_INVAL;
    if (r->gid >= n_groups || row >= in->rows) return RAFTING_E_INVAL;
    if (r->kind != RAFTING_OP_AE_REQUEST && r->kind != RAFTING_OP_PREVOTE_REQ && r->kind != RAFTING_OP_VOTE_REQ &&
        r->kind != RAFTING_OP_IS_REQUEST) return RAFTING_E_INVAL;
    const uint32_t slot = row * n_groups + r->gid;
    rafting_creq_t* req = const_cast<rafting_creq_t*>(q->req);
    rafting_cesc_op_t* esc = const_cast<rafting_cesc_op_t*>(q->op_esc);
    const uint32_t at_req = lower_slot(req, q->n_req, slot), at_esc = lower_slot(esc, q->n_op_esc, slot);
    if ((in->op_c && (in->op_c[slot] & 0xfu) != RAFTING_OP_NONE) || (at_req < q->n_req && req[at_req].slot == slot) ||
        (at_esc < q->n_op_esc && esc[at_esc].slot == slot)) return RAFTING_E_INVAL;            // one op per (row, group)
    const bool ae = r->kind == RAFTING_OP_AE_REQUEST;
    const uint32_t count = ae ? r->count : 0;
    if (count > 0xFFFFu || (count && !entry_terms)) return RAFTING_E_INVAL;
    const int64_t dt = now_ms - in->row_base[row];
    const uint64_t dterm = (uint64_t)r->term - (uint64_t)r->b;
    const int64_t dcommit = (int64_t)((uint64_t)r->commit - (uint64_t)r->a);
    bool fits = ae && count <= 63 && r->src_slot < 32 && dt >= 0 && dt <= 0xFFFF && dterm < (1ull << 32) &&
                dcommit >= INT32_MIN && dcommit <= INT32_MAX;
    for (uint32_t i = 0; fits && i < count; i++) fits = entry_terms[i] == r->term;
    if (fits) {
        if (q->n_req >= req_cap) return RAFTING_E_INVAL;
        rafting_creq_t x;
        x.slot = slot; x.meta = RAFTING_CREQ_MAKE(r->src_slot, count, (uint32_t)dt); x.term = r->term; x.prev_index = r->a;
        x.d_prev_term = (uint32_t)dterm; x.d_commit = (int32_t)dcommit;
        insert_at(req, &q->n_req, at_req, x);
        q->req_entries += count;
        return RAFTING_OK;
    }
    // in full, as rafting_request_to_inbox writes the dense op slot
    if (q->n_op_esc >= esc_cap || (count && (!q->ent_terms || (uint64_t)q->ent_count + count > ent_cap))) return RAFTING_E_INVAL;
    rafting_cesc_op_t x;
    memset(&x, 0, sizeof(x));
    x.slot = slot; x.ent = q->ent_count; x.op_meta = RAFTING_OP_MAKE(r->kind, r->src_slot, count);
    x.now_ms = now_ms; x.a = r->term; x.b = r->a; x.c = r->b;
    if (ae) { x.d = r->commit; x.e = r->a + 1; }
    else if (r->kind == RAFTING_OP_IS_REQUEST) x.d = host_result ? 1 : 0;
    if (count) { memcpy(const_cast<int64_t*>(q->ent_terms) + q->ent_count, entry_terms, (size_t)count * 8); q->ent_count += count; }
    insert_at(esc, &q->n_op_esc, at_esc, x);
    return RAFTING_OK;
}

extern "C" int rafting_coutbox_to_replies(const rafting_coutbox_t* co, uint32_t n_groups, uint32_t local_slot,
                                          const rafting_req_rec_t* placed, const uint8_t* placed_row, uint32_t n,
                                          rafting_batch_rec_t* out, uint32_t* n_out) {
    if (!co || !co->rep_c || !co->current_term || !co->counts || (!placed && n) || (!placed_row && n) || !out || !n_out) return RAFTING_E_INVAL;
    if (co->counts[0] > co->esc_cap) return RAFTING_E_CAPACITY;               // the escape list overflowed: use the dense outbox
    if (co->counts[0] && !co->esc) return RAFTING_E_INVAL;
    std::vector<std::pair<uint32_t, uint32_t>> esc;                          // (slot, index) of the reply escapes, sorted
    for (uint32_t k = 0; k < co->counts[0]; k++)
        if (co->esc[k].kind == RAFTING_CESC_REPLY) esc.push_back({co->esc[k].slot, k});
    std::sort(esc.begin(), esc.end());
    uint32_t k = 0;
    for (uint32_t i = 0; i < n; i++) {
        const rafting_req_rec_t& q = placed[i];
        if (q.gid >= n_groups || q.src_slot == local_slot) return RAFTING_E_INVAL;
        const uint32_t gi = (uint32_t)placed_row[i] * n_groups + q.gid;
        const uint8_t rc = co->rep_c[gi];
        int64_t term; uint32_t success;
        if (rc & 0x80u) { term = co->current_term[q.gid]; success = (rc >> 6) & 1u; }
        else {
            const auto it = std::lower_bound(esc.begin(), esc.end(), std::make_pair(gi, 0u));
            if (it == esc.end() || it->first != gi) continue;                 // no valid reply: the handler threw
            const rafting_cesc_out_t& e = co->esc[it->second];
            term = e.a; success = RAFTING_REP_SUCCESS(e.meta);
        }
        rafting_batch_rec_t r{};
        r.gid = q.gid;
        r.kind = (uint8_t)(q.kind == RAFTING_OP_AE_REQUEST ? RAFTING_EV_AE_ACK : q.kind == RAFTING_OP_IS_REQUEST ? RAFTING_EV_IS_ACK
                         : q.kind == RAFTING_OP_PREVOTE_REQ ? RAFTING_EV_PV_REPLY : RAFTING_EV_RV_REPLY);
        r.lane = (uint8_t)(local_slot < q.src_slot ? local_slot : local_slot - 1);
        r.flags = (uint8_t)(RAFTING_OUT_OK | (success << 2));
        r.incarnation = q.incarnation;
        r.term = term;
        r.epoch_at_send = q.epoch; r.last_at_send = q.last;
        out[k++] = r;
    }
    *n_out = k;
    return RAFTING_OK;
}

// commit records -> apply ranges: the scan RaftRoutine.commitState does per context, for the whole shard (RaftRoutine.java:224-306)
extern "C" int rafting_outbox_apply_ranges(const rafting_outbox_t* ob, const uint32_t* gids, uint32_t n, int64_t* applied,
                                           uint32_t n_groups, rafting_apply_rec_t* out, uint32_t cap, uint32_t* n_out) {
    if (!ob || !ob->role_word || !ob->commit_index || !applied || !out || !n_out) return RAFTING_E_INVAL;
    uint32_t k = 0;
    for (uint32_t i = 0; i < n; i++) {
        if (!(ob->role_word[i] & (1u << 31))) continue;                       // commit-dirty: commitIndex moved in this step
        const uint32_t gid = gids ? gids[i] : i;
        if (gid >= n_groups) { *n_out = k; return RAFTING_E_INVAL; }
        const int64_t c = ob->commit_index[i];
        if (c <= applied[gid]) continue;                                      // a snapshot already moved the machine past it
        if (k >= cap) { *n_out = k; return RAFTING_E_CAPACITY; }
        out[k].gid = gid; out[k]._pad = 0; out[k].first = applied[gid] + 1; out[k].last = c;
        applied[gid] = c;
        k++;
    }
    *n_out = k;
    return RAFTING_OK;
}

// ---- the pending-invocation table and replies -> compact wire words ----
struct rafting_pending {
    struct E { uint64_t key; uint32_t gid; uint8_t lane, tag, used, kind; uint32_t inc; int64_t term, epoch, last; };
    std::vector<E> t;
    size_t count = 0;
    static uint64_t mix(uint64_t x) { x ^= x >> 33; x *= 0xff51afd7ed558ccdull; x ^= x >> 33; x *= 0xc4ceb9fe1a85ec53ull; return x ^ (x >> 33); }
    static uint64_t key_of(uint32_t peer, int32_t seq) { return ((uint64_t)peer << 32) | (uint32_t)seq; }
    E* find(uint64_t key) {
        if (t.empty()) return nullptr;
        const size_t mask = t.size() - 1;
        for (size_t i = mix(key) & mask;; i = (i + 1) & mask) {
            if (!t[i].used) return nullptr;
            if (t[i].key == key) return &t[i];
        }
    }
    void place(const E& e) {
        const size_t mask = t.size() - 1;
        size_t i = mix(e.key) & mask;
        while (t[i].used) i = (i + 1) & mask;
        t[i] = e;
    }
    void grow(size_t want) {
        size_t cap = 64;
        while (cap < want * 2) cap <<= 1;
        if (cap <= t.size()) return;
        std::vector<E> old; old.swap(t);
        t.assign(cap, E{});
        for (const E& e : old) if (e.used) place(e);
    }
    void erase(E* e) {                                        // linear probing, backward-shift deletion (no tombstones)
        const size_t mask = t.size() - 1;
        size_t i = (size_t)(e - t.data());
        t[i].used = 0;
        for (size_t j = (i + 1) & mask; t[j].used; j = (j + 1) & mask) {
            const size_t home = mix(t[j].key) & mask;
            const bool between = i <= j ? (home > i && home <= j) : (home > i || home <= j);   // home cyclically in (i, j]: stays
            if (between) continue;
            t[i] = t[j]; t[j].used = 0; i = j;
        }
        count--;
    }
};
extern "C" int rafting_pending_create(uint32_t capacity_hint, rafting_pending_t** out) {
    if (!out) return RAFTING_E_INVAL;
    try { auto* p = new rafting_pending(); p->grow(capacity_hint ? capacity_hint : 32); *out = p; } catch (...) { return RAFTING_E_NOMEM; }
    return RAFTING_OK;
}
extern "C" int rafting_pending_destroy(rafting_pending_t* p) { delete p; return RAFTING_OK; }
extern "C" uint32_t rafting_pending_size(const rafting_pending_t* p) { return p ? (uint32_t)p->count : 0; }
extern "C" int rafting_pending_put(rafting_pending_t* p, uint32_t peer, int32_t sequence, uint32_t ev_kind, uint32_t gid, uint32_t lane,
                                   uint32_t tag, uint32_t incarnation, int64_t term, int64_t epoch_at_send, int64_t last_at_send) {
    if (!p || lane > 255 || (tag > 31 && tag != RAFTING_CTAG_NONE) || ev_kind == RAFTING_EV_NONE || ev_kind > RAFTING_EV_RV_REPLY)
        return RAFTING_E_INVAL;
    const uint64_t key = rafting_pending::key_of(peer, sequence);
    try {
        rafting_pending::E* e = p->find(key);
        if (!e) {
            if ((p->count + 1) * 2 > p->t.size()) p->grow(p->count + 1);
            rafting_pending::E n{}; n.key = key; n.used = 1;
            p->place(n); p->count++;
            e = p->find(key);
        }
        e->gid = gid; e->lane = (uint8_t)lane; e->tag = (uint8_t)tag; e->kind = (uint8_t)ev_kind; e->inc = incarnation; e->term = term;
        e->epoch = epoch_at_send; e->last = last_at_send;
    } catch (...) { return RAFTING_E_NOMEM; }
    return RAFTING_OK;
}
extern "C" int rafting_pending_remove(rafting_pending_t* p, uint32_t peer, int32_t sequence) {
    if (!p) return RAFTING_E_INVAL;
    rafting_pending::E* e = p->find(rafting_pending::key_of(peer, sequence));
    if (!e) return RAFTING_E_INVAL;
    p->erase(e);
    return RAFTING_OK;
}

extern "C" int rafting_acks_to_cinbox(rafting_pending_t* p, uint32_t peer, const rafting_ack_rec_t* acks, uint32_t n, int64_t now_ms,
                                      uint32_t row, const rafting_cinbox_t* cin, uint32_t n_groups, uint32_t F, rafting_cesc_in_t* esc,
                                      uint32_t esc_cap, uint32_t* n_esc, uint32_t* deferred, uint32_t* n_deferred, uint32_t* n_unknown) {
    if (!p || (!acks && n) || !cin || !cin->ev_c || !cin->row_base || !n_esc || !n_deferred || (!deferred && n) || row >= cin->rows)
        return RAFTING_E_INVAL;
    uint32_t* ev = const_cast<uint32_t*>(cin->ev_c);
    const int64_t dt = now_ms - cin->row_base[row];
    uint32_t unknown = 0, nd = 0;
    constexpr uint32_t AHEAD = 12;                                           // the table is a random access per reply: prefetch ahead
    const size_t tmask = p->t.empty() ? 0 : p->t.size() - 1;
    for (uint32_t i = 0; i < n; i++) {
        if (i + AHEAD < n && !p->t.empty())
            __builtin_prefetch(&p->t[rafting_pending::mix(rafting_pending::key_of(peer, acks[i + AHEAD].sequence)) & tmask]);
        const rafting_ack_rec_t& a = acks[i];
        rafting_pending::E* e = p->find(rafting_pending::key_of(peer, a.sequence));
        if (!e || e->gid != a.gid || e->kind != a.kind) { unknown++; continue; }   // timed out earlier, or a sequence of another scope
        if (e->gid >= n_groups || e->lane >= F) return RAFTING_E_INVAL;
        const size_t li = ((size_t)row * n_groups + e->gid) * F + e->lane;
        if (ev[li] != 0) { deferred[nd++] = i; continue; }                    // one event per (row, group, lane)
        const bool is_ack = a.kind == RAFTING_EV_AE_ACK || a.kind == RAFTING_EV_IS_ACK;
        const bool fits = is_ack && e->tag < 32 && dt >= 0 && dt <= 0xFFFF && a.term == e->term;
        if (fits) {
            ev[li] = RAFTING_CEV_MAKE(a.kind, RAFTING_OUT_OK, a.success ? 1 : 0, 1, e->tag, (uint32_t)dt);
        } else {
            if (!esc || *n_esc >= esc_cap) { *n_deferred = nd; if (n_unknown) *n_unknown = unknown; return RAFTING_E_CAPACITY; }
            rafting_cesc_in_t& x = esc[(*n_esc)++];
            memset(&x, 0, sizeof(x));
            x.slot = (uint32_t)li;
            x.ev_meta = RAFTING_EVM_MAKE(a.kind, RAFTING_OUT_OK, a.success ? 1 : 0, e->inc);
            x.term = a.term; x.now_ms = now_ms; x.epoch_at_send = e->epoch; x.last_at_send = e->last;
            ev[li] = RAFTING_CEV_ESCAPED;
        }
        p->erase(e);
    }
    *n_deferred = nd;
    if (n_unknown) *n_unknown = unknown;
    return RAFTING_OK;
}

extern "C" int rafting_failures_to_cinbox(rafting_pending_t* p, uint32_t peer, const int32_t* sequences, uint32_t n, uint32_t outcome,
                                          int64_t now_ms, uint32_t row, const rafting_cinbox_t* cin, uint32_t n_groups, uint32_t F,
                                          rafting_cesc_in_t* esc, uint32_t esc_cap, uint32_t* n_esc, uint32_t* deferred,
                                          uint32_t* n_deferred, uint32_t* n_unknown) {
    if (!p || (!sequences && n) || !cin || !cin->ev_c || !cin->row_base || !n_esc || !n_deferred || (!deferred && n) || row >= cin->rows ||
        (outcome != RAFTING_OUT_ERROR && outcome != RAFTING_OUT_CANCELED)) return RAFTING_E_INVAL;
    uint32_t* ev = const_cast<uint32_t*>(cin->ev_c);
    const int64_t dt = now_ms - cin->row_base[row];
    uint32_t unknown = 0, nd = 0;
    for (uint32_t i = 0; i < n; i++) {
        rafting_pending::E* e = p->find(rafting_pending::key_of(peer, sequences[i]));
        if (!e) { unknown++; continue; }
        if (e->gid >= n_groups || e->lane >= F) return RAFTING_E_INVAL;
        const size_t li = ((size_t)row * n_groups + e->gid) * F + e->lane;
        if (ev[li] != 0) { deferred[nd++] = i; continue; }
        const bool is_ack = e->kind == RAFTING_EV_AE_ACK || e->kind == RAFTING_EV_IS_ACK;
        if (is_ack && e->tag < 32 && dt >= 0 && dt <= 0xFFFF) {
            ev[li] = RAFTING_CEV_MAKE(e->kind, outcome, 0, 0, e->tag, (uint32_t)dt);
        } else {
            if (!esc || *n_esc >= esc_cap) { *n_deferred = nd; if (n_unknown) *n_unknown = unknown; return RAFTING_E_CAPACITY; }
            rafting_cesc_in_t& x = esc[(*n_esc)++];
            memset(&x, 0, sizeof(x));
            x.slot = (uint32_t)li;
            x.ev_meta = RAFTING_EVM_MAKE(e->kind, outcome, 0, e->inc);
            x.term = 0; x.now_ms = now_ms; x.epoch_at_send = e->epoch; x.last_at_send = e->last;
            ev[li] = RAFTING_CEV_ESCAPED;
        }
        p->erase(e);
    }
    *n_deferred = nd;
    if (n_unknown) *n_unknown = unknown;
    return RAFTING_OK;
}

// ---- the inbox builder: per-group FIFOs -> the rows of one dense step (the placement rule of tests/cluster_sim.py) ----
struct rafting_builder {
    struct Item { uint8_t is_event; rafting_req_rec_t req; rafting_batch_rec_t rep; std::vector<int64_t> terms; };
    uint32_t G, F;
    std::vector<std::deque<Item>> q;
    size_t pending = 0;
};
extern "C" int rafting_builder_create(uint32_t n_groups, uint32_t F, rafting_builder_t** out) {
    if (!out || !n_groups || !F || F > 255) return RAFTING_E_INVAL;
    try { auto* b = new rafting_builder(); b->G = n_groups; b->F = F; b->q.resize(n_groups); *out = b; } catch (...) { return RAFTING_E_NOMEM; }
    return RAFTING_OK;
}
extern "C" int rafting_builder_destroy(rafting_builder_t* b) { delete b; return RAFTING_OK; }
extern "C" uint32_t rafting_builder_pending(const rafting_builder_t* b) { return b ? (uint32_t)b->pending : 0; }
extern "C" int rafting_builder_clear_group(rafting_builder_t* b, uint32_t gid) {
    if (!b || gid >= b->G) return RAFTING_E_INVAL;
    b->pending -= b->q[gid].size(); b->q[gid].clear();
    return RAFTING_OK;
}
extern "C" int rafting_builder_push_submit(rafting_builder_t* b, uint32_t gid, uint32_t count, uint32_t unavailable_mask) {
    if (!b || gid >= b->G || count == 0 || count > 0xFFFFu) return RAFTING_E_INVAL;
    try {
        rafting_builder::Item it{}; it.is_event = 0;
        it.req.gid = gid; it.req.kind = RAFTING_OP_SUBMIT; it.req.count = count; it.req.a = (int64_t)unavailable_mask;
        b->q[gid].push_front(std::move(it)); b->pending++;
    } catch (...) { return RAFTING_E_NOMEM; }
    return RAFTING_OK;
}
extern "C" int rafting_builder_push_request(rafting_builder_t* b, const rafting_req_rec_t* r, const int64_t* entry_terms) {
    if (!b || !r || r->gid >= b->G) return RAFTING_E_INVAL;
    if (r->kind != RAFTING_OP_AE_REQUEST && r->kind != RAFTING_OP_PREVOTE_REQ && r->kind != RAFTING_OP_VOTE_REQ) return RAFTING_E_INVAL;
    if (r->kind == RAFTING_OP_AE_REQUEST && (r->count > 0xFFFFu || (r->count && !entry_terms))) return RAFTING_E_INVAL;
    try {
        rafting_builder::Item it{}; it.is_event = 0; it.req = *r;
        if (r->kind == RAFTING_OP_AE_REQUEST && r->count) it.terms.assign(entry_terms, entry_terms + r->count);
        b->q[r->gid].push_back(std::move(it)); b->pending++;
    } catch (...) { return RAFTING_E_NOMEM; }
    return RAFTING_OK;
}
extern "C" int rafting_builder_push_reply(rafting_builder_t* b, const rafting_batch_rec_t* r) {
    if (!b || !r || r->gid >= b->G || r->lane >= b->F || r->kind == RAFTING_EV_NONE || r->kind > RAFTING_EV_RV_REPLY) return RAFTING_E_INVAL;
    try {
        rafting_builder::Item it{}; it.is_event = 1; it.rep = *r;
        b->q[r->gid].push_back(std::move(it)); b->pending++;
    } catch (...) { return RAFTING_E_NOMEM; }
    return RAFTING_OK;
}

extern "C" int rafting_builder_build(rafting_builder_t* b, int64_t now_ms, const rafting_inbox_t* in, uint32_t ent_cap, uint32_t* ent_count,
                                     rafting_req_rec_t* placed, uint8_t* placed_row, uint32_t placed_cap, uint32_t* n_placed) {
    if (!b || !in || !in->row_now || !in->op_meta || !in->op_nr || !in->op_ab || !in->op_cd || !in->op_e || !in->ev_meta || !in->ev_tn ||
        !in->ev_el || in->gids || !ent_count || !n_placed || (!placed && placed_cap) || (!placed_row && placed_cap) || in->rows < 2 ||
        (ent_cap && !in->ent_terms)) return RAFTING_E_INVAL;
    const uint32_t G = b->G, F = b->F, rows = in->rows;
    const size_t ng = (size_t)rows * G, nl = ng * F;
    uint64_t* om = const_cast<uint64_t*>(in->op_meta);
    rafting_i64x2_t* nr = const_cast<rafting_i64x2_t*>(in->op_nr);
    rafting_i64x2_t* ab = const_cast<rafting_i64x2_t*>(in->op_ab);
    rafting_i64x2_t* cd = const_cast<rafting_i64x2_t*>(in->op_cd);
    int64_t* oe = const_cast<int64_t*>(in->op_e);
    uint64_t* em = const_cast<uint64_t*>(in->ev_meta);
    rafting_i64x2_t* tn = const_cast<rafting_i64x2_t*>(in->ev_tn);
    rafting_i64x2_t* el = const_cast<rafting_i64x2_t*>(in->ev_el);
    memset(om, 0, ng * 8); memset(nr, 0, ng * 16); memset(ab, 0, ng * 16); memset(cd, 0, ng * 16); memset(oe, 0, ng * 8);
    memset(em, 0, nl * 8); memset(tn, 0, nl * 16); memset(el, 0, nl * 16);
    int64_t* rn = const_cast<int64_t*>(in->row_now);
    memset(rn, 0, (size_t)rows * 8);
    rn[0] = now_ms;                                                         // the sweep row: every due election / keepAlive timer
    uint32_t ents = 0, np = 0;
    for (uint32_t g = 0; g < G; g++) {
        auto& q = b->q[g];
        uint32_t cursor = 0;                                                // position r * (F + 1) + (0 = op | 1 + lane)
        while (!q.empty()) {
            rafting_builder::Item& it = q.front();
            uint32_t r, pos;
            if (!it.is_event) { r = cursor / (F + 1) + 1; pos = r * (F + 1); }
            else {
                r = cursor / (F + 1); pos = r * (F + 1) + 1 + it.rep.lane;
                if (pos <= cursor) { r += 1; pos += F + 1; }
            }
            if (r >= rows) break;                                           // stays queued for the next step
            if (!it.is_event && np >= placed_cap) break;                    // the caller's list of placed ops is full: next step
            const size_t gi = (size_t)r * G + g;
            if (!it.is_event) {
                const rafting_req_rec_t& x = it.req;
                uint32_t off = 0, count = 0;
                int64_t a = 0, bb = 0, c = 0, d = 0, e = 0;
                if (x.kind == RAFTING_OP_SUBMIT) { count = x.count; a = x.a; }
                else {
                    a = x.term; bb = x.a; c = x.b;
                    if (x.kind == RAFTING_OP_AE_REQUEST) {
                        count = x.count; off = ents;
                        if ((uint64_t)ents + count > ent_cap) break;       // no room for the entry terms in this step: next step
                        if (count) memcpy(const_cast<int64_t*>(in->ent_terms) + ents, it.terms.data(), (size_t)count * 8);
                        ents += count;
                        d = x.commit; e = x.a + 1;
                    }
                }
                placed[np] = x; placed_row[np] = (uint8_t)r;
                np++;
                om[gi] = (uint64_t)RAFTING_OP_MAKE(x.kind, x.kind == RAFTING_OP_SUBMIT ? 0 : x.src_slot, count) | ((uint64_t)off << 32);
                nr[gi].x = now_ms; nr[gi].y = 0; ab[gi].x = a; ab[gi].y = bb; cd[gi].x = c; cd[gi].y = d; oe[gi] = e;
            } else {
                const rafting_batch_rec_t& x = it.rep;
                const size_t li = gi * F + x.lane;
                em[li] = RAFTING_EVM_MAKE(x.kind, x.flags & 3u, (x.flags >> 2) & 1u, x.incarnation);
                tn[li].x = x.term; tn[li].y = now_ms;
                if (x.kind == RAFTING_EV_AE_ACK || x.kind == RAFTING_EV_IS_ACK) { el[li].x = x.epoch_at_send; el[li].y = x.last_at_send; }
            }
            cursor = pos;
            q.pop_front(); b->pending--;
        }
    }
    *ent_count = ents; *n_placed = np;
    return RAFTING_OK;
}
