// seglog.cuh — HBM-resident segmented entry buffer with asynchronous pinned-host spill.
//
// SURVEY.md §8(f)-1 / north_star: on the hot path the RocksDB-backed RaftLog
// (M/command/storage/RocksLog.java:82-242, one RocksDB per context, key = 8-byte BE index,
// value = 8-byte BE term || Kryo(cmd), flushWal(true) on every write) is replaced by an in-memory
// store: entry payloads live in a ring of fixed-size SEGMENTS in HBM; a segment that must be recycled
// is first copied to pinned host memory on a side stream (the cold tier).  The index->term map the
// protocol needs stays in the run-length tables of the step kernel; this file only moves payload bytes.
//
//   RocksLog.newEntry / append  (put)          -> rafting_log_append  (batch: one H2D + one index kernel)
//   RocksLog.get / batch        (multiGet)     -> rafting_log_read    (one group), rafting_log_gather
//                                                 (many (gid, first, count) ranges = the AE plans of a step)
//   RocksLog.truncate / flush   (deleteRange)  -> visibility of a record is decided by the group's stored key range
//                                                 [g_lo, g_hi] in the tables, and a re-appended index overwrites
//                                                 its ring slot; rafting_log_trim reclaims what a flush left behind
//
// Record layout inside a segment: 24-byte header {gid u32, len u32, index i64, term i64} + payload padded
// to 8 bytes.  Records never straddle segments.  A logical byte offset (segment number * seg_bytes + offset)
// names a record forever; the HBM arena holds the newest `nseg` segments, older ones are read from the
// host copy.  Per group a device ring of K slots maps index -> logical offset for the gather kernel.
//
// Included at the end of engine.cu (same translation unit: it uses rafting_engine, fail(), CU()).
#pragma once
#include <errno.h>
#include <fcntl.h>
#include <sys/stat.h>
#include <unistd.h>

namespace rafting {

struct alignas(16) SegHdr { uint32_t gid, len; int64_t index, term; uint64_t seq; };
static_assert(sizeof(SegHdr) == 32, "segment record header");

struct HostLoc { uint64_t off; uint32_t len; int64_t term; uint64_t file_off; };      // len == 0xffffffff: absent; file_off: payload offset in the durable file (~0 = none)
constexpr uint64_t NO_FILE = ~0ull, NO_ARENA = ~0ull;                                  // off == NO_ARENA: recovered from the file, never resident
struct GroupIdx { int64_t base = 0; std::vector<HostLoc> v; int64_t epoch_index = 0, epoch_term = 0; };     // host index of one group: v[i] <-> index base + i
// What a group's host index has dropped while the device ring may still name it: indices below `index` (rafting_log_trim, the
// index window moving up) and records appended before `seq` (the window restarting elsewhere).  The ring serves neither.
struct Floor { int64_t index; uint64_t seq; };

struct SegLog {
    uint32_t seg_bytes = 0, nseg = 0, K = 0;
    uint8_t* arena = nullptr;                 // [nseg * seg_bytes] in HBM
    uint64_t head = 0;                        // logical offset of the next record
    uint64_t spilled_upto = 0;                // logical segments < this have a host copy enqueued
    unsigned long long* ring = nullptr;       // [G * K]: 1 + logical offset of the newest record whose index maps to the slot
    std::vector<uint8_t*> cold;               // pinned host copy per logical segment (null until spilled)
    std::vector<cudaEvent_t> cold_ready;      // spill completion per logical segment
    std::vector<GroupIdx> index;              // authoritative (lengths, terms, cold tier); the device ring is a cache of it
    uint8_t* stage = nullptr; size_t stage_cap = 0;       // pinned staging of one append batch
    void* d_req = nullptr; size_t d_req_cap = 0;           // device scratch (append records / gather requests)
    uint8_t* d_blob = nullptr; size_t d_blob_cap = 0;      // staged payload blob of the append in flight
    uint8_t* d_out = nullptr; size_t d_out_cap = 0;
    cudaStream_t s_spill = nullptr;
    cudaStream_t s_log = nullptr;             // every append / gather / read of the entry buffer runs here: the step kernel's stream
                                              // never waits for payload traffic (only the other way round, for the stored key ranges)
    cudaEvent_t ev_tables = nullptr, ev_log = nullptr;
    // durable tier (rafting_log_store_open): every appended record is also framed into an append-only file; fdatasync is one
    // call per step (rafting_log_sync).  The file doubles as the coldest tier, which is what lets the pinned pool be bounded.
    int wal_fd = -1; uint64_t wal_bytes = 0, wal_synced = 0, wal_syncs = 0; bool wal_failed = false;
    std::vector<uint8_t> wal_buf;
    uint32_t cold_max = 0;                    // pinned cold segments kept at most (0 = unbounded; needs the file tier)
    std::vector<uint64_t> cold_lru;           // spilled segments in spill order
    uint64_t cold_evicted = 0, file_hits = 0;
    uint64_t appended = 0, spilled_bytes = 0, hbm_hits = 0, cold_hits = 0, indexed = 0;
    std::vector<uint32_t> seg_live;           // live (indexed, not overwritten, not trimmed) records per logical segment
    uint64_t trimmed = 0, cold_freed_bytes = 0, spills_skipped = 0;
    cudaEvent_t t0 = nullptr, t1 = nullptr;    // device time of the last gather's kernel
    std::vector<Floor> floor;                 // [G] host copy of d_floor; gids floor_lo..floor_hi changed since the last upload
    Floor* d_floor = nullptr;
    uint32_t floor_lo = UINT32_MAX, floor_hi = 0;
    uint32_t gathers = 0;                     // step and range gathers begun and not waited for: the host index must stay put
    ::StepGather* ticket[RAFTING_GATHER_TICKETS] = {};      // rafting_log_gather_begin, created on first use
    bool ticket_busy[RAFTING_GATHER_TICKETS] = {};
    float last_gather_kernel_ms = 0; uint64_t last_gather_bytes = 0;
};

struct AppendRec { uint32_t gid, len; int64_t index, term; uint64_t loc; uint64_t src; };   // 40 B per appended entry
// 8 lanes per appended record: write the header, copy the payload from the staged blob into the arena and
// publish the record in the group's ring.  Logical offsets only grow, so atomicMax makes "the latest put wins"
// (RocksDB semantics) hold inside a batch and across batches without any ordering between threads.
__global__ void seglog_scatter_kernel(const AppendRec* __restrict__ recs, uint32_t n, uint64_t seq0, const uint8_t* __restrict__ blob,
                                      uint8_t* __restrict__ arena, uint64_t arena_bytes, unsigned long long* ring, uint32_t K) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t en = t >> 3, sub = t & 7;
    if (en >= n) return;
    const AppendRec r = recs[en];
    uint8_t* dst = arena + (r.loc % arena_bytes);
    if (sub == 0) {
        SegHdr h; h.gid = r.gid; h.len = r.len; h.index = r.index; h.term = r.term; h.seq = seq0 + en;
        *(int4*)dst = *(const int4*)&h; *(int4*)(dst + 16) = *((const int4*)&h + 1);
        atomicMax(&ring[(size_t)r.gid * K + ((uint64_t)r.index & (K - 1))], (unsigned long long)(r.loc + 1));
    }
    const uint8_t* src = blob + r.src;
    uint8_t* pay = dst + sizeof(SegHdr);
    if ((r.src & 15) == 0) {
        const uint32_t words = r.len >> 4;
        for (uint32_t i = sub; i < words; i += 8) ((int4*)pay)[i] = ((const int4*)src)[i];
        for (uint32_t i = (words << 4) + sub; i < r.len; i += 8) pay[i] = src[i];
    } else {
        for (uint32_t i = sub; i < r.len; i += 8) pay[i] = src[i];
    }
}

struct GatherReq { uint32_t gid; uint32_t slot; int64_t index; uint64_t out_off; };   // slot: position in the reply list

// The hit test of the entry buffer: the ring slot of (gid, index) names the newest record published there, and it serves
// the entry when that record is still in the HBM arena and is exactly (gid, index).  rec: the record, len: its payload bytes.
__device__ __forceinline__ bool seglog_hit(const unsigned long long* __restrict__ ring, uint32_t K, const uint8_t* __restrict__ arena,
                                           uint64_t arena_bytes, uint64_t oldest_resident, uint32_t gid, int64_t index,
                                           const uint8_t*& rec, uint32_t& len) {
    const unsigned long long loc1 = ring[(size_t)gid * K + ((uint64_t)index & (K - 1))];
    bool hit = loc1 != 0 && loc1 - 1 >= oldest_resident;
    len = 0;
    rec = arena + ((loc1 - 1) % arena_bytes);
    if (hit) {
        const int4 h0 = *(const int4*)rec;                       // gid, len, index
        const long long idx = ((long long)(unsigned)h0.w << 32) | (unsigned)h0.z;
        hit = (uint32_t)h0.x == gid && idx == index;
        len = (uint32_t)h0.y;
    }
    return hit;
}

// One requested entry on 8 lanes: *len_out = its length, or 0xffffffff when the ring does not hold it; on a hit the payload
// goes to out + q.out_off
__device__ __forceinline__ void seglog_gather_entry(const GatherReq& q, uint32_t sub, const unsigned long long* __restrict__ ring,
                                                    uint32_t K, const uint8_t* __restrict__ arena, uint64_t arena_bytes,
                                                    uint64_t oldest_resident, uint32_t* __restrict__ len_out, uint8_t* __restrict__ out) {
    const uint8_t* rec; uint32_t len;
    const bool hit = seglog_hit(ring, K, arena, arena_bytes, oldest_resident, q.gid, q.index, rec, len);
    if (sub == 0) *len_out = hit ? len : 0xffffffffu;
    if (!hit) return;
    const int4* src = (const int4*)(rec + sizeof(SegHdr));       // records and payloads are 16-byte aligned
    int4* dst = (int4*)(out + q.out_off);                        // out_off is 16-byte aligned
    const uint32_t words = (len + 15) >> 4;
    for (uint32_t i = sub; i < words; i += 8) dst[i] = src[i];
}

// 8 lanes per requested entry (4 entries per warp, so four dependent chains ring -> header -> payload are in
// flight per warp), 16-byte vector copies HBM arena -> contiguous send buffer.  lens[e] = 0xffffffff when the
// ring does not point at a resident record of exactly (gid, index); the host then serves it from its index.
__global__ void seglog_gather_kernel(const GatherReq* __restrict__ req, uint32_t n, const unsigned long long* __restrict__ ring,
                                     uint32_t K, const uint8_t* __restrict__ arena, uint64_t arena_bytes,
                                     uint64_t oldest_resident, uint32_t* __restrict__ lens, uint8_t* __restrict__ out) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t en = t >> 3, sub = t & 7;
    if (en >= n) return;
    const GatherReq q = req[en];
    seglog_gather_entry(q, sub, ring, K, arena, arena_bytes, oldest_resident, lens + en, out);
}

// ---- the payloads of a compact step's plans (rafting_log_gather_step_begin) ----
// Four passes on the entry buffer's stream over the step's dense plan columns, which stay resident after its wait:
//   step_plan_count_kernel   one thread per lane slot: the entries an AE plan asks for, and whether it has any
//   (cub scan)               -> each plan's first ref and its plan record
//   step_plan_probe_kernel   one thread per lane slot, over its entries: hit or miss, and the 16-byte-aligned bytes of its hits
//   (cub scan)               -> each plan's first blob offset, first miss and first gather request
//   step_plan_emit_kernel    the refs and plan records, one gather request per hit, the miss list
//   step_gather_copy_kernel  seglog_gather_entry over the requests, whose number only the device knows
struct GAgg { uint64_t a, b, c; };              // pass 1: (refs, plans, 0); pass 2: (device bytes, misses, hits)
struct GAggSum { __device__ __forceinline__ GAgg operator()(const GAgg& x, const GAgg& y) const { return GAgg{x.a + y.a, x.b + y.b, x.c + y.c}; } };

struct StepPlansD {                             // the step's dense plan columns; lane slot t stands for position (t / F) % n
    const uint64_t* plan_meta; const rafting_i64x2_t* plan_pp; const uint32_t* gids; uint32_t n, F, P;
};
struct ProbeD {                                 // what seglog_hit reads, and the host index's floors
    const unsigned long long* ring; uint32_t K; const uint8_t* arena; uint64_t arena_bytes, oldest; const Floor* floor;
};
struct StepOutD {
    rafting_entry_ref_t* refs; uint32_t refs_cap, plans_cap; rafting_plan_ref_t* plans; uint64_t blob_cap;
    GatherReq* req; uint32_t* miss;
};

__device__ __forceinline__ uint32_t plan_entries(uint64_t m) { return (m & 0xfu) == RAFTING_PLAN_AE ? (uint32_t)(m >> 16) & 0xffffu : 0u; }
__device__ __forceinline__ uint32_t plan_gid(const StepPlansD& s, uint32_t t) { const uint32_t i = (t / s.F) % s.n; return s.gids ? s.gids[i] : i; }
// seglog_hit, minus what the host index no longer holds: an entry rafting_log_trim dropped, or one a moved index window
// dropped (seglog_put), may still be named by the ring; the host then serves it, so both paths answer from the host index
__device__ __forceinline__ bool step_probe(const ProbeD& d, uint32_t gid, int64_t index, const uint8_t*& rec, uint32_t& len) {
    if (!seglog_hit(d.ring, d.K, d.arena, d.arena_bytes, d.oldest, gid, index, rec, len)) return false;
    const Floor f = d.floor[gid];
    return index >= f.index && *(const uint64_t*)(rec + 24) >= f.seq;            // SegHdr::seq
}

// t == P writes the identity, so that the scans' element P is the total
__global__ void step_plan_count_kernel(StepPlansD s, GAgg* __restrict__ agg) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t > s.P) return;
    const uint32_t c = t < s.P ? plan_entries(s.plan_meta[t]) : 0u;
    agg[t] = GAgg{c, c ? 1u : 0u, 0};
}

// entries past refs_cap are neither probed nor written: the wait sizes them on the host
__global__ void step_plan_probe_kernel(StepPlansD s, ProbeD d, const GAgg* __restrict__ off1, uint32_t refs_cap, GAgg* __restrict__ agg) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t > s.P) return;
    GAgg v = {0, 0, 0};
    const uint32_t c = t < s.P ? plan_entries(s.plan_meta[t]) : 0u;
    if (c) {
        const uint64_t first = off1[t].a;
        const uint32_t gid = plan_gid(s, t);
        const int64_t x = s.plan_pp[t].x;
        for (uint32_t j = 0; j < c && first + j < refs_cap; j++) {
            const uint8_t* rec; uint32_t len;
            if (step_probe(d, gid, x + 1 + j, rec, len)) { v.a += ((uint64_t)len + 15) & ~15ull; v.c++; }
            else v.b++;
        }
    }
    agg[t] = v;
}

__global__ void step_plan_emit_kernel(StepPlansD s, ProbeD d, const GAgg* __restrict__ off1, const GAgg* __restrict__ off2, StepOutD o) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= s.P) return;
    const uint32_t c = plan_entries(s.plan_meta[t]);
    if (!c) return;
    const GAgg p = off1[t];
    GAgg q = off2[t];
    if (p.b < o.plans_cap) { rafting_plan_ref_t r; r.slot = t; r.first = (uint32_t)p.a; r.count = c; r._pad = 0; o.plans[p.b] = r; }
    const uint32_t gid = plan_gid(s, t);
    const int64_t x = s.plan_pp[t].x;
    for (uint32_t j = 0; j < c && p.a + j < o.refs_cap; j++) {
        const uint64_t k = p.a + j;
        rafting_entry_ref_t r; r.gid = gid; r.index = x + 1 + j;
        const uint8_t* rec; uint32_t len;
        if (step_probe(d, gid, r.index, rec, len)) {
            r.len = len; r.term = *(const int64_t*)(rec + 16); r.blob_off = q.a;                 // SegHdr::term
            GatherReq g; g.gid = gid; g.slot = (uint32_t)k; g.index = r.index; g.out_off = q.a;
            q.a += ((uint64_t)len + 15) & ~15ull;
            if (q.a > o.blob_cap) g.index = 0;        // past the blob: a request the ring never serves (indices start at 1)
            o.req[q.c++] = g;
        } else {
            r.len = 0xffffffffu; r.term = 0; r.blob_off = 0;                                       // the wait fills them in
            o.miss[q.b++] = (uint32_t)k;
        }
        o.refs[k] = r;
    }
}

// total->c requests; a grid-stride loop, so the grid is sized without knowing their number
__global__ void step_gather_copy_kernel(const GatherReq* __restrict__ req, const GAgg* __restrict__ total, const unsigned long long* __restrict__ ring,
                                        uint32_t K, const uint8_t* __restrict__ arena, uint64_t arena_bytes, uint64_t oldest_resident,
                                        uint32_t* __restrict__ lens, uint8_t* __restrict__ out) {
    const uint64_t n = total->c;
    for (uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; (t >> 3) < n; t += (uint64_t)gridDim.x * blockDim.x)
        seglog_gather_entry(req[t >> 3], (uint32_t)(t & 7), ring, K, arena, arena_bytes, oldest_resident, lens + (t >> 3), out);
}

// ---- the payloads of (gid, first, count) ranges (rafting_log_gather_begin), e.g. the apply ranges of a step ----
// The host knows the number of entries, and one range may hold 10^5 of them (a group catching up), so every pass runs one
// thread per entry; the host only writes each range's first ref (an exclusive prefix of the counts).
//   range_probe_kernel       entry k finds its range, then hit or miss, and the 16-byte-aligned bytes of a hit
//   (cub scan)               -> each entry's blob offset (device-served bytes before it), miss ordinal and request ordinal
//   range_emit_kernel        the refs in ref order, one gather request per hit, the miss list
//   step_gather_copy_kernel  as for the step gather
struct GRange { int64_t first; uint32_t gid, ref; };     // first index, group, first ref of one range
struct RangesD { const GRange* r; uint32_t n, N; };       // n ranges, N entries in all
struct RangeOutD { rafting_entry_ref_t* refs; uint64_t blob_cap; GatherReq* req; uint32_t* miss; };

// the last range whose first ref is <= k (k < N): a range without entries shares its first ref with the next one
__device__ __forceinline__ uint32_t range_of(const RangesD& s, uint32_t k) {
    uint32_t lo = 0, hi = s.n;                    // r[lo].ref <= k; every range from hi on starts after k
    while (hi - lo > 1) {
        const uint32_t mid = (lo + hi) >> 1;
        if (s.r[mid].ref <= k) lo = mid; else hi = mid;
    }
    return lo;
}

// k == N writes the identity, so that the scan's element N is the total
__global__ void range_probe_kernel(RangesD s, ProbeD d, GAgg* __restrict__ agg) {
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k > s.N) return;
    GAgg v = {0, 0, 0};
    if (k < s.N) {
        const GRange r = s.r[range_of(s, k)];
        const uint8_t* rec; uint32_t len;
        if (step_probe(d, r.gid, r.first + (k - r.ref), rec, len)) { v.a = ((uint64_t)len + 15) & ~15ull; v.c = 1; }
        else v.b = 1;
    }
    agg[k] = v;
}

// a miss gets the blob offset of the device-served bytes before it; the wait moves what follows a miss the host index holds
__global__ void range_emit_kernel(RangesD s, ProbeD d, const GAgg* __restrict__ off, RangeOutD o) {
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= s.N) return;
    const GRange g = s.r[range_of(s, k)];
    const GAgg q = off[k];
    rafting_entry_ref_t r; r.gid = g.gid; r.index = g.first + (k - g.ref); r.blob_off = q.a;
    const uint8_t* rec; uint32_t len;
    if (step_probe(d, r.gid, r.index, rec, len)) {
        r.len = len; r.term = *(const int64_t*)(rec + 16);                                          // SegHdr::term
        GatherReq w; w.gid = r.gid; w.slot = k; w.index = r.index; w.out_off = q.a;
        if (q.a + (((uint64_t)len + 15) & ~15ull) > o.blob_cap) w.index = 0;   // past the blob: a request the ring never serves
        o.req[q.c] = w;
    } else {
        r.len = 0xffffffffu; r.term = 0;                                                             // the wait fills them in
        o.miss[q.b] = k;
    }
    o.refs[k] = r;
}

}  // namespace rafting

using rafting::SegLog; using rafting::SegHdr; using rafting::HostLoc; using rafting::GatherReq; using rafting::AppendRec;

static void gather_free(StepGather*& g);
static void seglog_release(rafting_engine* e) {
    SegLog* L = e->seglog; if (!L) return;
    if (L->s_log) { cudaStreamSynchronize(L->s_log); cudaStreamDestroy(L->s_log); }
    for (StepGather*& t : L->ticket) gather_free(t);             // a gather not waited for is drained above, then freed
    if (L->s_spill) { cudaStreamSynchronize(L->s_spill); cudaStreamDestroy(L->s_spill); }
    if (L->ev_tables) cudaEventDestroy(L->ev_tables);
    if (L->ev_log) cudaEventDestroy(L->ev_log);
    if (L->wal_fd >= 0) close(L->wal_fd);
    for (auto ev : L->cold_ready) if (ev) cudaEventDestroy(ev);
    for (auto p : L->cold) if (p) cudaFreeHost(p);
    if (L->arena) cudaFree(L->arena);
    if (L->ring) cudaFree(L->ring);
    if (L->stage) cudaFreeHost(L->stage);
    if (L->d_req) cudaFree(L->d_req);
    if (L->d_out) cudaFree(L->d_out);
    if (L->d_blob) cudaFree(L->d_blob);
    if (L->t0) { cudaEventDestroy(L->t0); cudaEventDestroy(L->t1); }
    if (L->d_floor) cudaFree(L->d_floor);
    delete L; e->seglog = nullptr;
}

extern "C" int rafting_log_config(rafting_engine_t* e, uint32_t segment_bytes, uint32_t hbm_segments, uint32_t ring_slots) {
    if (!e) return fail(RAFTING_E_INVAL, "null argument");
    if (e->seglog) return fail(RAFTING_E_INVAL, "entry buffer already configured");
    if (segment_bytes < 4096 || (segment_bytes & 15) || hbm_segments < 2 || ring_slots == 0 || (ring_slots & (ring_slots - 1)))
        return fail(RAFTING_E_INVAL, "segment_bytes >= 4096 and 16-aligned, hbm_segments >= 2, ring_slots a power of two");
    CU(cudaSetDevice(e->cfg.device));
    SegLog* L = new SegLog();
    L->seg_bytes = segment_bytes; L->nseg = hbm_segments; L->K = ring_slots;
    e->seglog = L;
    L->index.resize(e->G);
    L->floor.assign(e->G, rafting::Floor{0, 0});
    const size_t ring = (size_t)e->G * ring_slots;
    CU(cudaMalloc(&L->arena, (size_t)segment_bytes * hbm_segments));
    CU(cudaMalloc(&L->ring, ring * 8));
    CU(cudaMemset(L->ring, 0, ring * 8));                          // 0 = empty slot
    CU(cudaMalloc(&L->d_floor, (size_t)e->G * sizeof(rafting::Floor)));
    CU(cudaMemset(L->d_floor, 0, (size_t)e->G * sizeof(rafting::Floor)));
    CU(cudaStreamCreateWithFlags(&L->s_spill, cudaStreamNonBlocking));
    CU(cudaStreamCreateWithFlags(&L->s_log, cudaStreamNonBlocking));
    CU(cudaEventCreateWithFlags(&L->ev_tables, cudaEventDisableTiming));
    CU(cudaEventCreateWithFlags(&L->ev_log, cudaEventDisableTiming));
    if (!e->ev_seg) CU(cudaEventCreateWithFlags(&e->ev_seg, cudaEventDisableTiming));
    return RAFTING_OK;
}

static inline const HostLoc* seglog_find(const SegLog* L, uint32_t gid, int64_t index) {
    const rafting::GroupIdx& gi = L->index[gid];
    if (index < gi.base || index >= gi.base + (int64_t)gi.v.size()) return nullptr;
    const HostLoc& h = gi.v[(size_t)(index - gi.base)];
    return h.len == 0xffffffffu ? nullptr : &h;
}
constexpr int64_t SEGLOG_INDEX_WINDOW = 1 << 22;      // indices one group's host index spans at most (4 M entries, 128 MB of index)
static inline void seglog_drop(SegLog* L, const HostLoc& h) {
    if (h.len == 0xffffffffu) return;
    if (h.off != rafting::NO_ARENA) L->seg_live[h.off / L->seg_bytes]--;
    L->indexed--;
}
static inline void seglog_floor(SegLog* L, uint32_t gid, int64_t index, uint64_t seq) {
    rafting::Floor& f = L->floor[gid];
    if (index > f.index) f.index = index;
    if (seq > f.seq) f.seq = seq;
    if (gid < L->floor_lo) L->floor_lo = gid;
    if (gid > L->floor_hi) L->floor_hi = gid;
}
// a group's host index starts again from nothing at the record with sequence number seq: every older record of the group is
// excluded by seq, so the index floor goes back to 0 (left where a trim or cut put it, it would keep the ring from serving
// every new index below it)
static inline void seglog_floor_restart(SegLog* L, uint32_t gid, uint64_t seq) {
    L->floor[gid].index = 0;
    seglog_floor(L, gid, 0, seq);
}
// the changed floors go up on the log stream, ahead of every gather enqueued later (a pageable copy: the host may change them
// again as soon as this returns)
static int seglog_floor_flush(SegLog* L) {
    if (L->floor_lo > L->floor_hi) return RAFTING_OK;
    CU(cudaMemcpyAsync(L->d_floor + L->floor_lo, L->floor.data() + L->floor_lo, (size_t)(L->floor_hi - L->floor_lo + 1) * sizeof(rafting::Floor),
                       cudaMemcpyHostToDevice, L->s_log));
    L->floor_lo = UINT32_MAX; L->floor_hi = 0;
    return RAFTING_OK;
}
// seq: the append sequence number the record gets (its SegHdr::seq)
static inline void seglog_put(SegLog* L, uint32_t gid, int64_t index, const HostLoc& hl, uint64_t seq) {
    rafting::GroupIdx& gi = L->index[gid];
    const HostLoc none = {0, 0xffffffffu, 0, rafting::NO_FILE};
    // An empty index that starts below its floor (everything was trimmed, then the group's log starts again lower) is a new
    // window as well.
    const bool below_floor = gi.v.empty() && index < L->floor[gid].index;
    if (gi.v.empty()) gi.base = index;
    // An index far from everything stored (an InstallSnapshot moved the follower's log, RaftRoutine.java:408-445) starts a
    // new window instead of materialising the gap: what lay on the other side of it is no longer reachable by any plan.
    // Below the window that is any index the newest WINDOW indices would not hold: extending down to it and keeping the
    // newest window would cut the very index being put.
    const int64_t end = gi.base + (int64_t)gi.v.size();
    if (below_floor || index < end - SEGLOG_INDEX_WINDOW || index >= end + SEGLOG_INDEX_WINDOW) {
        for (const HostLoc& h : gi.v) seglog_drop(L, h);
        gi.v.clear(); gi.base = index;
        seglog_floor_restart(L, gid, seq);                         // every older record of the group is gone
    }
    if (index < gi.base) { gi.v.insert(gi.v.begin(), (size_t)(gi.base - index), none); gi.base = index; }
    if (index >= gi.base + (int64_t)gi.v.size()) gi.v.resize((size_t)(index - gi.base) + 1, none);
    if (gi.v.size() > (size_t)SEGLOG_INDEX_WINDOW) {                // keep the newest window (index is its newest)
        const size_t cut = gi.v.size() - (size_t)SEGLOG_INDEX_WINDOW;
        for (size_t k = 0; k < cut; k++) seglog_drop(L, gi.v[k]);
        gi.v.erase(gi.v.begin(), gi.v.begin() + (ptrdiff_t)cut); gi.base += (int64_t)cut;
        seglog_floor(L, gid, gi.base, 0);
    }
    HostLoc& slot = gi.v[(size_t)(index - gi.base)];
    if (slot.len == 0xffffffffu) L->indexed++;
    else if (slot.off != rafting::NO_ARENA) L->seg_live[slot.off / L->seg_bytes]--;   // the overwritten record is dead
    if (hl.off != rafting::NO_ARENA) {
        const uint64_t seg = hl.off / L->seg_bytes;
        if (L->seg_live.size() <= seg) L->seg_live.resize(seg + 1, 0);
        L->seg_live[seg]++;
    }
    slot = hl;                                                     // RocksDB put: the latest value wins
}

// make room: every segment about to be overwritten by the span ending at new_head is copied to pinned host first
static int seglog_spill_for(rafting_engine* e, SegLog* L, uint64_t new_head) {
    const uint64_t last_seg = (new_head - 1) / L->seg_bytes;      // highest logical segment that will hold data
    while (last_seg >= L->nseg && L->spilled_upto <= last_seg - L->nseg) {
        const uint64_t s = L->spilled_upto;
        if (L->cold.size() <= s) { L->cold.resize(s + 1, nullptr); L->cold_ready.resize(s + 1, nullptr); }
        if (s < L->seg_live.size() && L->seg_live[s] == 0) {       // nothing live in it (compacted / overwritten): no cold copy
            L->spilled_upto = s + 1; L->spills_skipped++;
            continue;
        }
        CU(cudaHostAlloc((void**)&L->cold[s], L->seg_bytes, cudaHostAllocDefault));
        CU(cudaEventCreateWithFlags(&L->cold_ready[s], cudaEventDisableTiming));
        CU(cudaEventRecord(e->ev_seg, L->s_log));                  // the spill sees every append already enqueued
        CU(cudaStreamWaitEvent(L->s_spill, e->ev_seg, 0));
        CU(cudaMemcpyAsync(L->cold[s], L->arena + (s % L->nseg) * (uint64_t)L->seg_bytes, L->seg_bytes, cudaMemcpyDeviceToHost, L->s_spill));
        CU(cudaEventRecord(L->cold_ready[s], L->s_spill));
        CU(cudaStreamWaitEvent(L->s_log, L->cold_ready[s], 0));    // later appends into that arena slot wait for it
        L->spilled_upto = s + 1; L->spilled_bytes += L->seg_bytes;
        L->cold_lru.push_back(s);
        // bounded pinned pool: the oldest cold copies go once the file tier holds the same bytes durably
        while (L->cold_max && L->wal_fd >= 0 && L->cold_lru.size() > L->cold_max) {
            const uint64_t v = L->cold_lru.front();
            if (L->cold[v]) {
                if ((v + 1) * (uint64_t)L->seg_bytes > L->head) break;
                CU(cudaEventSynchronize(L->cold_ready[v]));
                cudaFreeHost(L->cold[v]); L->cold[v] = nullptr;
                cudaEventDestroy(L->cold_ready[v]); L->cold_ready[v] = nullptr;
                L->cold_evicted++;
            }
            L->cold_lru.erase(L->cold_lru.begin());
        }
    }
    return RAFTING_OK;
}

static int seglog_wal_put(SegLog* L, const rafting_entry_ref_t* refs, uint32_t n, const uint8_t* blob, std::vector<uint64_t>& file_offs);
static int log_append_impl(rafting_engine_t* e, const rafting_entry_ref_t* refs, uint32_t n, const void* blob, size_t blob_bytes) {
    if (!e || !e->seglog) return fail(RAFTING_E_INVAL, "entry buffer not configured (rafting_log_config)");
    if (e->seglog->gathers) return fail(RAFTING_E_BUSY, "a gather has not been waited for (rafting_log_gather_wait / _step_wait)");
    if (n == 0) return RAFTING_OK;
    if (!refs || (!blob && blob_bytes)) return fail(RAFTING_E_INVAL, "null argument");
    SegLog* L = e->seglog;
    CU(cudaSetDevice(e->cfg.device));
    // every ref is checked before anything changes: a bad one must not leave earlier entries of the batch indexed at arena
    // offsets that were never written
    for (uint32_t i = 0; i < n; i++) {
        if (refs[i].gid >= e->G) return fail(RAFTING_E_INVAL, "ref %u: gid out of range", i);
        if (refs[i].index <= 0) return fail(RAFTING_E_INVAL, "ref %u: log indices start at 1", i);
        if (refs[i].blob_off > blob_bytes || (uint64_t)refs[i].len > blob_bytes - refs[i].blob_off) return fail(RAFTING_E_INVAL, "ref %u: payload beyond the blob", i);
        if (sizeof(SegHdr) + (((uint64_t)refs[i].len + 15) & ~15ull) > L->seg_bytes) return fail(RAFTING_E_CAPACITY, "ref %u: record larger than a segment", i);
    }
    if ((uint64_t)L->seg_bytes * (L->nseg - 1) < sizeof(SegHdr) + 16) return fail(RAFTING_E_CAPACITY, "arena too small for a single record");
    // durable tier first (write-ahead): the records are framed into the file buffer; rafting_log_sync makes them durable
    std::vector<uint64_t> file_offs;
    if (L->wal_fd >= 0) { int rc = seglog_wal_put(L, refs, n, (const uint8_t*)blob, file_offs); if (rc) return rc; }
    // the payload blob travels to the device once and stays there while the sub-batches below are scattered
    // (pin it on the host for a truly asynchronous copy)
    CU(cudaStreamSynchronize(L->s_log));                          // previous append done with d_blob / staging
    if (blob_bytes > L->d_blob_cap) {
        if (L->d_blob) cudaFree(L->d_blob);
        L->d_blob_cap = blob_bytes + blob_bytes / 2 + 256;
        CU(cudaMalloc((void**)&L->d_blob, L->d_blob_cap));
    }
    if (blob_bytes) CU(cudaMemcpyAsync(L->d_blob, blob, blob_bytes, cudaMemcpyHostToDevice, L->s_log));
    const uint64_t arena_bytes = (uint64_t)L->seg_bytes * L->nseg;
    uint32_t done = 0;
    while (done < n) {
        // layout pass (arithmetic only): records never straddle a segment; a sub-batch ends before it would reach the arena
        // slot of the segment that holds L->head, whose records before L->head stay resident.  Counted from that segment's
        // start, a sub-batch has the whole arena: every segment it overwrites is spilled first, and its first record always
        // fits, a skipped tail included
        const uint64_t end = (L->head / L->seg_bytes + L->nseg) * L->seg_bytes;
        const size_t need = (size_t)(n - done) * sizeof(AppendRec);
        if (need > L->stage_cap) {
            CU(cudaStreamSynchronize(L->s_log));
            if (L->stage) cudaFreeHost(L->stage);
            L->stage_cap = need + need / 2;
            CU(cudaHostAlloc((void**)&L->stage, L->stage_cap, cudaHostAllocDefault));
        } else if (done) CU(cudaStreamSynchronize(L->s_log));     // the previous sub-batch has left the staging buffer
        AppendRec* recs = (AppendRec*)L->stage;
        uint64_t head = L->head; uint32_t m = 0;
        for (uint32_t i = done; i < n; i++) {
            const uint64_t rec = sizeof(SegHdr) + (((uint64_t)refs[i].len + 15) & ~15ull);
            uint64_t h2 = head;
            if (h2 / L->seg_bytes != (h2 + rec - 1) / L->seg_bytes) h2 = (h2 / L->seg_bytes + 1) * L->seg_bytes;   // skip the tail
            if (h2 + rec > end) break;
            AppendRec& r = recs[m];
            r.gid = refs[i].gid; r.len = refs[i].len; r.index = refs[i].index; r.term = refs[i].term; r.loc = h2; r.src = refs[i].blob_off;
            HostLoc hl; hl.off = h2; hl.len = refs[i].len; hl.term = refs[i].term;
            hl.file_off = file_offs.empty() ? rafting::NO_FILE : file_offs[i];
            seglog_put(L, refs[i].gid, refs[i].index, hl, L->appended + m);
            head = h2 + rec; m++;
        }
        if (m == 0) return fail(RAFTING_E_CAPACITY, "arena too small for a single record");
        int rc = seglog_spill_for(e, L, head); if (rc) return rc;
        const size_t rec_bytes = (size_t)m * sizeof(AppendRec);
        if (rec_bytes > L->d_req_cap) {
            CU(cudaStreamSynchronize(L->s_log));
            if (L->d_req) cudaFree(L->d_req);
            L->d_req_cap = rec_bytes * 2;
            CU(cudaMalloc(&L->d_req, L->d_req_cap));
        }
        CU(cudaMemcpyAsync(L->d_req, recs, rec_bytes, cudaMemcpyHostToDevice, L->s_log));
        rafting::seglog_scatter_kernel<<<(uint32_t)(((uint64_t)m * 8 + 255) / 256), 256, 0, L->s_log>>>(
            (const AppendRec*)L->d_req, m, L->appended, L->d_blob, L->arena, arena_bytes, L->ring, L->K);
        CU(cudaGetLastError());
        L->head = head; L->appended += m; done += m;
    }
    return seglog_floor_flush(L);
}

// no C++ exception may cross the C ABI (a host index that cannot grow is RAFTING_E_NOMEM, not std::terminate)
extern "C" int rafting_log_append(rafting_engine_t* e, const rafting_entry_ref_t* refs, uint32_t n, const void* blob, size_t blob_bytes) {
    try { return log_append_impl(e, refs, n, blob, blob_bytes); }
    catch (const std::bad_alloc&) { return fail(RAFTING_E_NOMEM, "rafting_log_append: out of host memory"); }
    catch (const std::exception& ex) { return fail(RAFTING_E_NOMEM, "rafting_log_append: %s", ex.what()); }
}

// stored key range of a group straight from the tables (RocksLog visibility: epoch / truncate are metadata)
// the tables are written by the step kernels: a read of the stored key ranges is ordered behind every step enqueued so
// far (event on the step stream, waited for by the log stream) — the step stream itself never waits for the entry buffer
static int seglog_after_tables(rafting_engine* e, SegLog* L) {
    CU(cudaEventRecord(L->ev_tables, e->stream));
    CU(cudaStreamWaitEvent(L->s_log, L->ev_tables, 0));
    return RAFTING_OK;
}
static int seglog_range(rafting_engine* e, uint32_t gid, int64_t* lo, int64_t* hi) {
    SegLog* L = e->seglog;
    int rc0 = seglog_after_tables(e, L); if (rc0) return rc0;
    uint64_t meta;
    CU(cudaMemcpyAsync(&meta, e->T.g_meta + gid, 8, cudaMemcpyDeviceToHost, L->s_log));
    CU(cudaMemcpyAsync(lo, e->T.g_lo + gid, 8, cudaMemcpyDeviceToHost, L->s_log));
    CU(cudaMemcpyAsync(hi, e->T.g_hi + gid, 8, cudaMemcpyDeviceToHost, L->s_log));
    CU(cudaStreamSynchronize(L->s_log));
    if ((((uint32_t)meta >> rafting::W_NRUNS_SH) & 0xf) == 0) { *lo = 1; *hi = 0; }
    return RAFTING_OK;
}
// logical offset of the oldest byte the HBM arena still holds (the newest nseg segments)
static inline uint64_t seglog_oldest_resident(const SegLog* L) {
    const uint64_t newest = L->head ? (L->head - 1) / L->seg_bytes : 0;
    return newest + 1 >= L->nseg ? (newest + 1 - L->nseg) * (uint64_t)L->seg_bytes : 0;
}
static inline bool seglog_resident(const SegLog* L, uint64_t off) {
    const uint64_t newest = L->head ? (L->head - 1) / L->seg_bytes : 0;
    return off / L->seg_bytes + L->nseg > newest;
}
static int seglog_fetch(rafting_engine* e, SegLog* L, const HostLoc& hl, void* dst) {
    (void)e;
    const uint64_t arena_bytes = (uint64_t)L->seg_bytes * L->nseg;
    if (hl.off != rafting::NO_ARENA && seglog_resident(L, hl.off)) {                            // still in HBM
        CU(cudaMemcpyAsync(dst, L->arena + (hl.off % arena_bytes) + sizeof(SegHdr), hl.len, cudaMemcpyDeviceToHost, L->s_log));
        L->hbm_hits++;
        return RAFTING_OK;
    }
    const uint64_t seg = hl.off == rafting::NO_ARENA ? ~0ull : hl.off / L->seg_bytes;
    if (seg < L->cold.size() && L->cold[seg]) {                                                 // pinned cold tier
        CU(cudaEventSynchronize(L->cold_ready[seg]));
        memcpy(dst, L->cold[seg] + (hl.off % L->seg_bytes) + sizeof(SegHdr), hl.len);
        L->cold_hits++;
        return RAFTING_OK;
    }
    if (hl.file_off != rafting::NO_FILE && L->wal_fd >= 0) {                                    // durable file tier
        if (hl.file_off + hl.len > L->wal_bytes - L->wal_buf.size()) {                          // still in the write buffer
            const uint64_t flushed = L->wal_bytes - L->wal_buf.size();
            if (hl.file_off >= flushed) { memcpy(dst, L->wal_buf.data() + (hl.file_off - flushed), hl.len); L->file_hits++; return RAFTING_OK; }
            return fail(RAFTING_E_INVAL, "record straddles the file buffer");
        }
        size_t got = 0;
        while (got < hl.len) {
            const ssize_t r = pread(L->wal_fd, (uint8_t*)dst + got, hl.len - got, (off_t)(hl.file_off + got));
            if (r < 0 && errno == EINTR) continue;
            if (r <= 0) return fail(RAFTING_E_CUDA, "pread of the entry file failed: %s", r < 0 ? strerror(errno) : "short file");
            got += (size_t)r;
        }
        L->file_hits++;
        return RAFTING_OK;
    }
    return fail(RAFTING_E_INVAL, "segment %llu neither resident, nor in the pinned pool, nor on file", (unsigned long long)seg);
}

extern "C" int rafting_log_read(rafting_engine_t* e, uint32_t gid, int64_t first_index, uint32_t max_n,
                                rafting_entry_ref_t* refs_out, void* blob_out, size_t blob_cap, uint32_t* n_out) {
    if (!e || !e->seglog) return fail(RAFTING_E_INVAL, "entry buffer not configured (rafting_log_config)");
    if (gid >= e->G || !refs_out || !n_out) return fail(RAFTING_E_INVAL, "bad argument");
    SegLog* L = e->seglog;
    CU(cudaSetDevice(e->cfg.device));
    int64_t lo, hi; int rc = seglog_range(e, gid, &lo, &hi); if (rc) return rc;
    uint32_t n = 0; size_t used = 0;
    for (int64_t idx = first_index; n < max_n; idx++) {
        if (idx < lo || idx > hi) break;                           // RocksLog.get: null outside the stored keys
        const HostLoc* hl = seglog_find(L, gid, idx);
        if (!hl) break;
        if (used + hl->len > blob_cap) break;
        if (hl->len) { rc = seglog_fetch(e, L, *hl, (uint8_t*)blob_out + used); if (rc) return rc; }
        refs_out[n].gid = gid; refs_out[n].len = hl->len; refs_out[n].index = idx; refs_out[n].term = hl->term; refs_out[n].blob_off = used;
        used += ((size_t)hl->len + 15) & ~(size_t)15; n++;
    }
    CU(cudaStreamSynchronize(L->s_log));
    *n_out = n;
    return RAFTING_OK;
}

// Many ranges at once (the AppendEntries plans of a step): entries resident in HBM are gathered by one
// kernel into a contiguous device buffer and copied down once; the rest come from the cold tier.
// refs_out[k].len == 0xffffffff marks an entry that was never appended.
extern "C" int rafting_log_gather(rafting_engine_t* e, uint32_t n_ranges, const uint32_t* gids, const int64_t* firsts,
                                  const uint32_t* counts, rafting_entry_ref_t* refs_out, uint32_t refs_cap,
                                  void* blob_out, size_t blob_cap, uint32_t* n_out, size_t* bytes_out) {
    if (!e || !e->seglog) return fail(RAFTING_E_INVAL, "entry buffer not configured (rafting_log_config)");
    if (!gids || !firsts || !counts || !refs_out || !n_out) return fail(RAFTING_E_INVAL, "null argument");
    SegLog* L = e->seglog;
    CU(cudaSetDevice(e->cfg.device));
    std::vector<GatherReq> req; std::vector<uint32_t> cold;
    uint32_t m = 0; size_t used = 0;
    for (uint32_t r = 0; r < n_ranges; r++) {
        if (gids[r] >= e->G) return fail(RAFTING_E_INVAL, "range %u: gid out of range", r);
        for (uint32_t k = 0; k < counts[r]; k++) {
            if (m >= refs_cap) return fail(RAFTING_E_CAPACITY, "refs_out too small");
            const int64_t idx = firsts[r] + k;
            rafting_entry_ref_t& o = refs_out[m];
            o.gid = gids[r]; o.index = idx; o.term = 0; o.blob_off = used; o.len = 0xffffffffu;
            const HostLoc* hl = seglog_find(L, gids[r], idx);      // lengths / offsets come from the host index
            if (hl) {
                if (used + (((size_t)hl->len + 15) & ~(size_t)15) > blob_cap) return fail(RAFTING_E_CAPACITY, "blob_out too small");
                o.len = hl->len; o.term = hl->term;
                if (hl->off != rafting::NO_ARENA && seglog_resident(L, hl->off)) { GatherReq q; q.gid = gids[r]; q.slot = m; q.index = idx; q.out_off = used; req.push_back(q); }
                else if (hl->len) cold.push_back(m);
                used += ((size_t)hl->len + 15) & ~(size_t)15;
            }
            m++;
        }
    }
    const uint32_t nq = (uint32_t)req.size();
    if (nq) {
        const size_t req_bytes = (size_t)nq * sizeof(GatherReq), len_bytes = (size_t)nq * 4;
        if (req_bytes + len_bytes > L->d_req_cap || used > L->d_out_cap) CU(cudaStreamSynchronize(L->s_log));
        if (req_bytes + len_bytes > L->d_req_cap) {
            if (L->d_req) cudaFree(L->d_req);
            L->d_req_cap = (req_bytes + len_bytes) * 2;
            CU(cudaMalloc(&L->d_req, L->d_req_cap));
        }
        if (used > L->d_out_cap) {
            if (L->d_out) cudaFree(L->d_out);
            L->d_out_cap = used * 2;
            CU(cudaMalloc((void**)&L->d_out, L->d_out_cap));
        }
        uint32_t* d_lens = (uint32_t*)((uint8_t*)L->d_req + req_bytes);
        CU(cudaMemcpyAsync(L->d_req, req.data(), req_bytes, cudaMemcpyHostToDevice, L->s_log));
        if (!L->t0) { CU(cudaEventCreate(&L->t0)); CU(cudaEventCreate(&L->t1)); }
        const uint64_t oldest = seglog_oldest_resident(L);
        CU(cudaEventRecord(L->t0, L->s_log));
        rafting::seglog_gather_kernel<<<(uint32_t)(((uint64_t)nq * 8 + 255) / 256), 256, 0, L->s_log>>>(
            (const GatherReq*)L->d_req, nq, L->ring, L->K, L->arena, (uint64_t)L->seg_bytes * L->nseg, oldest, d_lens, L->d_out);
        CU(cudaGetLastError());
        CU(cudaEventRecord(L->t1, L->s_log));
        std::vector<uint32_t> lens(nq);
        CU(cudaMemcpyAsync(lens.data(), d_lens, len_bytes, cudaMemcpyDeviceToHost, L->s_log));
        CU(cudaMemcpyAsync(blob_out, L->d_out, used, cudaMemcpyDeviceToHost, L->s_log));
        CU(cudaStreamSynchronize(L->s_log));
        CU(cudaEventElapsedTime(&L->last_gather_kernel_ms, L->t0, L->t1));
        L->last_gather_bytes = used;
        // ring misses (the slot now caches a newer index of the same group): direct copy through the host index
        for (uint32_t k = 0; k < nq; k++) {
            if (lens[k] != 0xffffffffu) { L->hbm_hits++; continue; }
            const rafting_entry_ref_t& o = refs_out[req[k].slot];
            const HostLoc* hl = seglog_find(L, o.gid, o.index);
            if (hl && hl->len) { int rc = seglog_fetch(e, L, *hl, (uint8_t*)blob_out + o.blob_off); if (rc) return rc; }
        }
    }
    for (uint32_t k : cold) {                                      // after the bulk copy-down
        const rafting_entry_ref_t& o = refs_out[k];
        int rc = seglog_fetch(e, L, *seglog_find(L, o.gid, o.index), (uint8_t*)blob_out + o.blob_off); if (rc) return rc;
    }
    CU(cudaStreamSynchronize(L->s_log));
    *n_out = m;
    if (bytes_out) *bytes_out = used;
    return RAFTING_OK;
}

// ---- rafting_log_gather_step_begin / _wait: the payloads of the plans of a slot's compact step ----
// Per slot (and per ticket of rafting_log_gather_begin): device scratch of the passes, and a pinned (so mapped) block for the
// totals, the miss list and the outputs the device cannot write directly
struct StepGather {
    Blk dev;                                   // aggregates and scans, CUB's scratch, requests, the copy's lens (a range gather: its ranges first)
    Blk host;                                  // totals (2 x GAgg), miss list [refs_cap], then the staged outputs (a range gather: its ranges last)
    cudaEvent_t ev = nullptr, t0 = nullptr, t1 = nullptr;
    bool timed = false;                        // the kernels ran (the step has plan columns, the ranges have entries)
    bool in_order = false;                     // a range gather: every payload at its place in ref order, host-served ones included
    rafting_entry_ref_t* refs = nullptr; uint32_t refs_cap = 0, plans_cap = 0; uint8_t* blob = nullptr; size_t blob_cap = 0;
    rafting_plan_ref_t* plans = nullptr;
    size_t o_miss = 0, o_refs = 0, o_plans = 0, o_blob = 0;   // offsets in host; the staged outputs only
    bool st_refs = false, st_plans = false, st_blob = false;
};
static void gather_free(StepGather*& g) {
    if (!g) return;
    if (g->ev) { cudaEventSynchronize(g->ev); cudaEventDestroy(g->ev); cudaEventDestroy(g->t0); cudaEventDestroy(g->t1); }
    blk_free(g->dev, false); blk_free(g->host, true);
    delete g; g = nullptr;
}
static void step_gather_release(Slot& s) { gather_free(s.gather); }
static int gather_events(StepGather& g) {
    if (!g.ev) {
        CU(cudaEventCreateWithFlags(&g.ev, cudaEventDisableTiming));
        CU(cudaEventCreate(&g.t0)); CU(cudaEventCreate(&g.t1));
    }
    return RAFTING_OK;
}
// the device address of host memory the device can write (pinned or registered, aligned), else null
static uint8_t* mapped_host(void* p, uintptr_t align) {
    cudaPointerAttributes pa;
    if (p && (uintptr_t)p % align == 0 && cudaPointerGetAttributes(&pa, p) == cudaSuccess && pa.type == cudaMemoryTypeHost && pa.devicePointer)
        return (uint8_t*)pa.devicePointer;
    cudaGetLastError();
    return nullptr;
}

extern "C" int rafting_log_gather_step_begin(rafting_engine_t* e, uint32_t slot, rafting_entry_ref_t* refs_out, uint32_t refs_cap,
                                             void* blob_out, size_t blob_cap, rafting_plan_ref_t* plans_out, uint32_t plans_cap) {
    using namespace rafting;
    if (!e || slot >= RAFTING_HOST_SLOTS || (refs_cap && !refs_out) || (blob_cap && !blob_out) || (plans_cap && !plans_out))
        return fail(RAFTING_E_INVAL, "bad argument");
    if (!e->seglog) return fail(RAFTING_E_INVAL, "entry buffer not configured (rafting_log_config)");
    Slot* S = e->host ? &e->host->slot[slot] : nullptr;
    if (S && S->gathering) return fail(RAFTING_E_BUSY, "slot %u holds a gather that has not been waited for", slot);
    if (!S || !S->compact_step || S->inflight) return fail(RAFTING_E_INVAL, "slot %u: no finished compact step to gather for", slot);
    const uint64_t P = S->dev_out.plan_meta ? (uint64_t)S->rows_ * S->n_ * e->F : 0;   // no op, no sweep row: no plan columns
    if (P >= 0x7fffffffu) return fail(RAFTING_E_CAPACITY, "%llu lane slots: a step gather walks fewer than 2^31", (unsigned long long)P);
    SegLog* L = e->seglog;
    CU(cudaSetDevice(e->cfg.device));
    if (!S->gather) S->gather = new StepGather();
    StepGather& g = *S->gather;
    if (int rc = gather_events(g)) return rc;
    uint8_t* d_refs = mapped_host(refs_out, 8); uint8_t* d_plans = mapped_host(plans_out, 4); uint8_t* d_blob = mapped_host(blob_out, 16);
    g.st_refs = refs_cap && !d_refs; g.st_plans = plans_cap && !d_plans; g.st_blob = blob_cap && !d_blob;
    Carve hc;
    hc.take(2 * sizeof(GAgg));
    g.o_miss = hc.take((size_t)refs_cap * 4);
    g.o_refs = g.st_refs ? hc.take((size_t)refs_cap * sizeof(rafting_entry_ref_t)) : 0;
    g.o_plans = g.st_plans ? hc.take((size_t)plans_cap * sizeof(rafting_plan_ref_t)) : 0;
    g.o_blob = g.st_blob ? hc.take(blob_cap) : 0;
    size_t scan_tmp = 0;
    if (P) CU(cub::DeviceScan::ExclusiveScan(nullptr, scan_tmp, (GAgg*)nullptr, (GAgg*)nullptr, GAggSum(), GAgg{0, 0, 0}, (int)(P + 1)));
    Carve dc;
    const size_t o_agg1 = dc.take((P + 1) * sizeof(GAgg)), o_off1 = dc.take((P + 1) * sizeof(GAgg));
    const size_t o_agg2 = dc.take((P + 1) * sizeof(GAgg)), o_off2 = dc.take((P + 1) * sizeof(GAgg));
    const size_t o_req = dc.take((size_t)refs_cap * sizeof(GatherReq)), o_lens = dc.take((size_t)refs_cap * 4), o_tmp = dc.take(scan_tmp);
    int rc;
    if ((rc = blk_reserve(g.host, hc.o, true)) || (P && (rc = blk_reserve(g.dev, dc.o, false)))) return rc;
    uint8_t* hdev = nullptr;
    CU(cudaHostGetDevicePointer((void**)&hdev, g.host.p, 0));
    if (!d_refs && g.st_refs) d_refs = hdev + g.o_refs;
    if (!d_plans && g.st_plans) d_plans = hdev + g.o_plans;
    if (!d_blob && g.st_blob) d_blob = hdev + g.o_blob;
    if ((rc = seglog_floor_flush(L))) return rc;
    g.timed = P != 0;
    if (P) {
        GAgg* agg1 = (GAgg*)(g.dev.p + o_agg1); GAgg* off1 = (GAgg*)(g.dev.p + o_off1);
        GAgg* agg2 = (GAgg*)(g.dev.p + o_agg2); GAgg* off2 = (GAgg*)(g.dev.p + o_off2);
        StepPlansD sp; sp.plan_meta = S->dev_out.plan_meta; sp.plan_pp = S->dev_out.plan_pp; sp.gids = S->c_gids;
        sp.n = (uint32_t)S->n_; sp.F = e->F; sp.P = (uint32_t)P;
        ProbeD pd; pd.ring = L->ring; pd.K = L->K; pd.arena = L->arena; pd.arena_bytes = (uint64_t)L->seg_bytes * L->nseg;
        pd.oldest = seglog_oldest_resident(L); pd.floor = L->d_floor;
        StepOutD od; od.refs = (rafting_entry_ref_t*)d_refs; od.refs_cap = refs_cap; od.plans = (rafting_plan_ref_t*)d_plans;
        od.plans_cap = plans_cap; od.blob_cap = blob_cap; od.req = (GatherReq*)(g.dev.p + o_req); od.miss = (uint32_t*)(hdev + g.o_miss);
        const uint32_t blocks = (uint32_t)((P + 1 + 255) / 256);
        CU(cudaEventRecord(g.t0, L->s_log));
        step_plan_count_kernel<<<blocks, 256, 0, L->s_log>>>(sp, agg1);
        size_t tb = scan_tmp;
        CU(cub::DeviceScan::ExclusiveScan(g.dev.p + o_tmp, tb, agg1, off1, GAggSum(), GAgg{0, 0, 0}, (int)(P + 1), L->s_log));
        step_plan_probe_kernel<<<blocks, 256, 0, L->s_log>>>(sp, pd, off1, refs_cap, agg2);
        tb = scan_tmp;
        CU(cub::DeviceScan::ExclusiveScan(g.dev.p + o_tmp, tb, agg2, off2, GAggSum(), GAgg{0, 0, 0}, (int)(P + 1), L->s_log));
        step_plan_emit_kernel<<<blocks, 256, 0, L->s_log>>>(sp, pd, off1, off2, od);
        const uint64_t copy_blocks = ((uint64_t)refs_cap * 8 + 255) / 256;
        if (copy_blocks)
            step_gather_copy_kernel<<<(uint32_t)(copy_blocks < 1056 ? copy_blocks : 1056), 256, 0, L->s_log>>>(
                od.req, off2 + P, pd.ring, pd.K, pd.arena, pd.arena_bytes, pd.oldest, (uint32_t*)(g.dev.p + o_lens), d_blob);
        CU(cudaGetLastError());
        CU(cudaEventRecord(g.t1, L->s_log));
        CU(cudaMemcpyAsync(g.host.p, off1 + P, sizeof(GAgg), cudaMemcpyDeviceToHost, L->s_log));
        CU(cudaMemcpyAsync(g.host.p + sizeof(GAgg), off2 + P, sizeof(GAgg), cudaMemcpyDeviceToHost, L->s_log));
    } else {
        memset(g.host.p, 0, 2 * sizeof(GAgg));
    }
    CU(cudaEventRecord(g.ev, L->s_log));
    g.refs = refs_out; g.refs_cap = refs_cap; g.blob = (uint8_t*)blob_out; g.blob_cap = blob_cap; g.plans = plans_out; g.plans_cap = plans_cap;
    S->gathering = true; L->gathers++;
    return RAFTING_OK;
}

// Bytes the refs past refs_cap need (they were neither probed nor written): the plans decoded on the host, lengths from the
// host index.  Only a wait that returns RAFTING_E_CAPACITY gets here.
static int step_gather_overflow(rafting_engine* e, const Slot& S, uint32_t refs_cap, uint64_t* bytes) {
    const size_t P = S.rows_ * S.n_ * e->F;
    std::vector<uint64_t> meta(P); std::vector<rafting_i64x2_t> pp(P); std::vector<uint32_t> gids(S.c_gids ? S.n_ : 0);
    CU(cudaMemcpy(meta.data(), S.dev_out.plan_meta, P * 8, cudaMemcpyDeviceToHost));
    CU(cudaMemcpy(pp.data(), S.dev_out.plan_pp, P * 16, cudaMemcpyDeviceToHost));
    if (S.c_gids) CU(cudaMemcpy(gids.data(), S.c_gids, S.n_ * 4, cudaMemcpyDeviceToHost));
    uint64_t k = 0;
    for (size_t t = 0; t < P; t++) {
        const uint32_t c = RAFTING_PLM_KIND(meta[t]) == RAFTING_PLAN_AE ? RAFTING_PLM_COUNT(meta[t]) : 0;
        const size_t i = (t / e->F) % S.n_;
        const uint32_t gid = S.c_gids ? gids[i] : (uint32_t)i;
        for (uint32_t j = 0; j < c; j++, k++) {
            if (k < refs_cap) continue;
            const HostLoc* hl = seglog_find(e->seglog, gid, pp[t].x + 1 + j);
            if (hl) *bytes += ((uint64_t)hl->len + 15) & ~15ull;
        }
    }
    return RAFTING_OK;
}

// A range gather keeps rafting_log_gather's layout, every payload at its place in ref order, but the device laid its payloads
// out as if no miss had bytes: each ref moves up by the bytes of the host-served entries before it.  Walked from the last ref
// down to the first such entry, so no payload is overwritten before it has moved.
static void gather_make_room(StepGather& g, uint64_t n, const uint32_t* miss, uint64_t n_miss, uint64_t shift) {
    uint64_t m = n_miss;
    for (uint64_t k = n; shift && k-- > 0;) {
        rafting_entry_ref_t& r = g.refs[k];
        if (m && miss[m - 1] == k) {
            m--;
            if (r.len != 0xffffffffu) shift -= ((uint64_t)r.len + 15) & ~15ull;
        } else if (r.len) {
            memmove(g.blob + r.blob_off + shift, g.blob + r.blob_off, r.len);
        }
        r.blob_off += shift;
    }
}

// The host side of both waits, after the device's part: staged outputs copied out, the misses served through the host index,
// the bytes needed, the stats.  t1 = (refs, plans), t2 = (device bytes, misses, hits).  A step gather puts the host-served
// payloads after the device's; a range gather (g.in_order) puts them where rafting_log_gather does.  S: the step gather's slot,
// whose refs past refs_cap are sized on the host.
static int gather_finish(rafting_engine* e, StepGather& g, const rafting::GAgg& t1, const rafting::GAgg& t2, const Slot* S, uint64_t* need_out, bool* fits_out) {
    SegLog* L = e->seglog;
    if (g.st_refs) memcpy(g.refs, g.host.p + g.o_refs, (size_t)(t1.a < g.refs_cap ? t1.a : g.refs_cap) * sizeof(rafting_entry_ref_t));
    if (g.st_plans) memcpy(g.plans, g.host.p + g.o_plans, (size_t)(t1.b < g.plans_cap ? t1.b : g.plans_cap) * sizeof(rafting_plan_ref_t));
    if (g.st_blob) memcpy(g.blob, g.host.p + g.o_blob, (size_t)(t2.a < g.blob_cap ? t2.a : g.blob_cap));
    // the misses: lengths and terms from the host index
    const uint32_t* miss = (const uint32_t*)(g.host.p + g.o_miss);
    uint64_t need = t2.a;
    for (uint64_t m = 0; m < t2.b; m++) {
        rafting_entry_ref_t& r = g.refs[miss[m]];
        if (!g.in_order) r.blob_off = need;
        if (const HostLoc* hl = seglog_find(L, r.gid, r.index)) { r.len = hl->len; r.term = hl->term; need += ((uint64_t)hl->len + 15) & ~15ull; }
    }
    if (S && t1.a > g.refs_cap) { if (int rc = step_gather_overflow(e, *S, g.refs_cap, &need)) return rc; }
    const bool fits = t1.a <= g.refs_cap && t1.b <= g.plans_cap && need <= g.blob_cap;
    if (fits && g.in_order && need > t2.a) gather_make_room(g, t1.a, miss, t2.b, need - t2.a);
    for (uint64_t m = 0; fits && m < t2.b; m++) {
        const rafting_entry_ref_t& r = g.refs[miss[m]];
        if (r.len == 0xffffffffu || r.len == 0) continue;
        if (int rc = seglog_fetch(e, L, *seglog_find(L, r.gid, r.index), g.blob + r.blob_off)) return rc;
    }
    CU(cudaStreamSynchronize(L->s_log));
    if (g.timed) CU(cudaEventElapsedTime(&L->last_gather_kernel_ms, g.t0, g.t1));
    L->last_gather_bytes = need;
    if (fits) L->hbm_hits += t2.c;
    *need_out = need; *fits_out = fits;
    return RAFTING_OK;
}

extern "C" int rafting_log_gather_step_wait(rafting_engine_t* e, uint32_t slot, uint32_t* n_refs, size_t* bytes, uint32_t* n_plans,
                                            uint32_t* host_served) {
    using namespace rafting;
    if (!e || slot >= RAFTING_HOST_SLOTS) return fail(RAFTING_E_INVAL, "bad argument");
    Slot* S = e->host ? &e->host->slot[slot] : nullptr;
    if (!S || !S->gathering) return fail(RAFTING_E_INVAL, "slot %u has no gather in flight", slot);
    CU(cudaSetDevice(e->cfg.device));
    SegLog* L = e->seglog; StepGather& g = *S->gather;
    CU(cudaEventSynchronize(g.ev));
    S->gathering = false; L->gathers--;
    const GAgg t1 = ((const GAgg*)g.host.p)[0], t2 = ((const GAgg*)g.host.p)[1];   // (refs, plans), (device bytes, misses, hits)
    uint64_t need; bool fits;
    if (int rc = gather_finish(e, g, t1, t2, S, &need, &fits)) return rc;
    if (n_refs) *n_refs = (uint32_t)(t1.a < UINT32_MAX ? t1.a : UINT32_MAX);
    if (bytes) *bytes = (size_t)need;
    if (n_plans) *n_plans = (uint32_t)(t1.b < UINT32_MAX ? t1.b : UINT32_MAX);
    if (host_served) *host_served = (uint32_t)t2.b;
    if (!fits)
        return fail(RAFTING_E_CAPACITY, "slot %u: the plans need %llu refs, %llu bytes and %llu plan records (caps %u, %zu, %u)", slot,
                    (unsigned long long)t1.a, (unsigned long long)need, (unsigned long long)t1.b, g.refs_cap, g.blob_cap, g.plans_cap);
    return RAFTING_OK;
}

// ---- rafting_log_gather_begin / _wait: the payloads of (gid, first, count) ranges, rafting_log_gather's result without a
// host lookup per entry and without blocking the caller between the two calls ----
extern "C" int rafting_log_gather_begin(rafting_engine_t* e, uint32_t ticket, uint32_t n_ranges, const uint32_t* gids,
                                        const int64_t* firsts, const uint32_t* counts, rafting_entry_ref_t* refs_out,
                                        uint32_t refs_cap, void* blob_out, size_t blob_cap) {
    using namespace rafting;
    if (!e || ticket >= RAFTING_GATHER_TICKETS || (n_ranges && (!gids || !firsts || !counts)) || (refs_cap && !refs_out) ||
        (blob_cap && !blob_out))
        return fail(RAFTING_E_INVAL, "bad argument");
    if (!e->seglog) return fail(RAFTING_E_INVAL, "entry buffer not configured (rafting_log_config)");
    SegLog* L = e->seglog;
    if (L->ticket_busy[ticket]) return fail(RAFTING_E_BUSY, "ticket %u holds a gather that has not been waited for", ticket);
    uint64_t N = 0;
    for (uint32_t r = 0; r < n_ranges; r++) {
        if (gids[r] >= e->G) return fail(RAFTING_E_INVAL, "range %u: gid out of range", r);
        N += counts[r];
    }
    if (N >= 0x80000000ull) return fail(RAFTING_E_CAPACITY, "%llu entries: a range gather takes fewer than 2^31", (unsigned long long)N);
    if (N > refs_cap) return fail(RAFTING_E_CAPACITY, "the ranges hold %llu entries, refs_out %u", (unsigned long long)N, refs_cap);
    CU(cudaSetDevice(e->cfg.device));
    if (!L->ticket[ticket]) L->ticket[ticket] = new StepGather();
    StepGather& g = *L->ticket[ticket];
    if (int rc = gather_events(g)) return rc;
    g.in_order = true;
    uint8_t* d_refs = mapped_host(refs_out, 8); uint8_t* d_blob = mapped_host(blob_out, 16);
    g.st_refs = N && !d_refs; g.st_plans = false; g.st_blob = blob_cap && !d_blob;
    Carve hc;
    hc.take(2 * sizeof(GAgg));
    g.o_miss = hc.take((size_t)N * 4);
    g.o_refs = g.st_refs ? hc.take((size_t)N * sizeof(rafting_entry_ref_t)) : 0;
    g.o_plans = 0;
    g.o_blob = g.st_blob ? hc.take(blob_cap) : 0;
    const size_t o_ranges_h = hc.take(N ? (size_t)n_ranges * sizeof(GRange) : 0);
    size_t scan_tmp = 0;
    if (N) CU(cub::DeviceScan::ExclusiveScan(nullptr, scan_tmp, (GAgg*)nullptr, (GAgg*)nullptr, GAggSum(), GAgg{0, 0, 0}, (int)(N + 1)));
    Carve dc;
    const size_t o_ranges = dc.take((size_t)n_ranges * sizeof(GRange));
    const size_t o_agg = dc.take((N + 1) * sizeof(GAgg)), o_off = dc.take((N + 1) * sizeof(GAgg));
    const size_t o_req = dc.take(N * sizeof(GatherReq)), o_lens = dc.take(N * 4), o_tmp = dc.take(scan_tmp);
    int rc;
    if ((rc = blk_reserve(g.host, hc.o, true)) || (N && (rc = blk_reserve(g.dev, dc.o, false)))) return rc;
    uint8_t* hdev = nullptr;
    CU(cudaHostGetDevicePointer((void**)&hdev, g.host.p, 0));
    if (!d_refs && g.st_refs) d_refs = hdev + g.o_refs;
    if (!d_blob && g.st_blob) d_blob = hdev + g.o_blob;
    if ((rc = seglog_floor_flush(L))) return rc;
    ((GAgg*)g.host.p)[0] = GAgg{N, 0, 0};
    g.timed = N != 0;
    if (N) {
        // each range's first ref, an exclusive prefix of the counts: the one pass over the ranges, none over their entries
        GRange* hr = (GRange*)(g.host.p + o_ranges_h);
        uint32_t ref = 0;
        for (uint32_t r = 0; r < n_ranges; r++) { hr[r].first = firsts[r]; hr[r].gid = gids[r]; hr[r].ref = ref; ref += counts[r]; }
        GRange* dr = (GRange*)(g.dev.p + o_ranges);
        GAgg* agg = (GAgg*)(g.dev.p + o_agg); GAgg* off = (GAgg*)(g.dev.p + o_off);
        RangesD rs; rs.r = dr; rs.n = n_ranges; rs.N = (uint32_t)N;
        ProbeD pd; pd.ring = L->ring; pd.K = L->K; pd.arena = L->arena; pd.arena_bytes = (uint64_t)L->seg_bytes * L->nseg;
        pd.oldest = seglog_oldest_resident(L); pd.floor = L->d_floor;
        RangeOutD od; od.refs = (rafting_entry_ref_t*)d_refs; od.blob_cap = blob_cap; od.req = (GatherReq*)(g.dev.p + o_req);
        od.miss = (uint32_t*)(hdev + g.o_miss);
        const uint32_t blocks = (uint32_t)((N + 1 + 255) / 256);
        const uint64_t copy_blocks = (N * 8 + 255) / 256;
        CU(cudaMemcpyAsync(dr, hr, (size_t)n_ranges * sizeof(GRange), cudaMemcpyHostToDevice, L->s_log));
        CU(cudaEventRecord(g.t0, L->s_log));
        range_probe_kernel<<<blocks, 256, 0, L->s_log>>>(rs, pd, agg);
        size_t tb = scan_tmp;
        CU(cub::DeviceScan::ExclusiveScan(g.dev.p + o_tmp, tb, agg, off, GAggSum(), GAgg{0, 0, 0}, (int)(N + 1), L->s_log));
        range_emit_kernel<<<blocks, 256, 0, L->s_log>>>(rs, pd, off, od);
        step_gather_copy_kernel<<<(uint32_t)(copy_blocks < 1056 ? copy_blocks : 1056), 256, 0, L->s_log>>>(
            od.req, off + N, pd.ring, pd.K, pd.arena, pd.arena_bytes, pd.oldest, (uint32_t*)(g.dev.p + o_lens), d_blob);
        CU(cudaGetLastError());
        CU(cudaEventRecord(g.t1, L->s_log));
        CU(cudaMemcpyAsync(g.host.p + sizeof(GAgg), off + N, sizeof(GAgg), cudaMemcpyDeviceToHost, L->s_log));
    } else {
        ((GAgg*)g.host.p)[1] = GAgg{0, 0, 0};
    }
    CU(cudaEventRecord(g.ev, L->s_log));
    g.refs = refs_out; g.refs_cap = refs_cap; g.blob = (uint8_t*)blob_out; g.blob_cap = blob_cap; g.plans = nullptr; g.plans_cap = 0;
    L->ticket_busy[ticket] = true; L->gathers++;
    return RAFTING_OK;
}

extern "C" int rafting_log_gather_wait(rafting_engine_t* e, uint32_t ticket, uint32_t* n_refs, size_t* bytes, uint32_t* host_served) {
    using namespace rafting;
    if (!e || ticket >= RAFTING_GATHER_TICKETS) return fail(RAFTING_E_INVAL, "bad argument");
    SegLog* L = e->seglog;
    if (!L || !L->ticket_busy[ticket]) return fail(RAFTING_E_INVAL, "ticket %u has no gather in flight", ticket);
    CU(cudaSetDevice(e->cfg.device));
    StepGather& g = *L->ticket[ticket];
    CU(cudaEventSynchronize(g.ev));
    L->ticket_busy[ticket] = false; L->gathers--;
    const GAgg t1 = ((const GAgg*)g.host.p)[0], t2 = ((const GAgg*)g.host.p)[1];   // (refs, 0), (device bytes, misses, hits)
    uint64_t need; bool fits;
    if (int rc = gather_finish(e, g, t1, t2, nullptr, &need, &fits)) return rc;
    if (n_refs) *n_refs = (uint32_t)t1.a;
    if (bytes) *bytes = (size_t)need;
    if (host_served) *host_served = (uint32_t)t2.b;
    if (!fits)
        return fail(RAFTING_E_CAPACITY, "ticket %u: the ranges need %llu bytes (blob_cap %zu)", ticket, (unsigned long long)need, g.blob_cap);
    return RAFTING_OK;
}

// Garbage collection behind RaftLog.flush (RocksLog.java:228-242: deleteRange below the new epoch): index entries below
// a group's lowest stored key are dropped, and a cold (pinned host) segment whose last live record went away is freed.
// A segment with no live record is also never spilled in the first place (seglog_spill_for).
extern "C" int rafting_log_trim(rafting_engine_t* e, uint32_t first_gid, uint32_t count, uint64_t* dropped_entries, uint64_t* freed_cold_bytes) {
    if (!e || !e->seglog) return fail(RAFTING_E_INVAL, "entry buffer not configured (rafting_log_config)");
    if ((uint64_t)first_gid + count > e->G) return fail(RAFTING_E_CAPACITY, "gid range beyond max_groups");
    if (e->seglog->gathers) return fail(RAFTING_E_BUSY, "a gather has not been waited for (rafting_log_gather_wait / _step_wait)");
    SegLog* L = e->seglog;
    CU(cudaSetDevice(e->cfg.device));
    std::vector<uint64_t> meta(count); std::vector<int64_t> lo(count), hi(count);
    { int rc0 = seglog_after_tables(e, L); if (rc0) return rc0; }
    if (count) {
        CU(cudaMemcpyAsync(meta.data(), e->T.g_meta + first_gid, (size_t)count * 8, cudaMemcpyDeviceToHost, L->s_log));
        CU(cudaMemcpyAsync(lo.data(), e->T.g_lo + first_gid, (size_t)count * 8, cudaMemcpyDeviceToHost, L->s_log));
        CU(cudaMemcpyAsync(hi.data(), e->T.g_hi + first_gid, (size_t)count * 8, cudaMemcpyDeviceToHost, L->s_log));
        CU(cudaStreamSynchronize(L->s_log));
    }
    uint64_t dropped = 0, freed = 0;
    for (uint32_t k = 0; k < count; k++) {
        rafting::GroupIdx& gi = L->index[first_gid + k];
        if (gi.v.empty()) continue;
        const bool empty = (((uint32_t)meta[k] >> rafting::W_NRUNS_SH) & 0xf) == 0;
        // entries below the lowest stored key are gone for good (an empty store after a flush beyond its end: everything
        // up to the old end); a truncated suffix is NOT dropped here — re-appends overwrite it
        const int64_t keep_from = empty ? hi[k] + 1 : lo[k];
        int64_t cut = keep_from - gi.base;
        if (cut <= 0) continue;
        if (cut > (int64_t)gi.v.size()) cut = (int64_t)gi.v.size();
        for (int64_t i = 0; i < cut; i++) {
            const HostLoc& h = gi.v[(size_t)i];
            if (h.len == 0xffffffffu) continue;
            seglog_drop(L, h); dropped++;
        }
        gi.v.erase(gi.v.begin(), gi.v.begin() + cut);
        gi.base += cut;
        seglog_floor(L, first_gid + k, gi.base, 0);
    }
    if (int rc = seglog_floor_flush(L)) return rc;
    for (size_t s = 0; s < L->cold.size(); s++) {
        if (!L->cold[s] || (s < L->seg_live.size() && L->seg_live[s] != 0)) continue;
        CU(cudaEventSynchronize(L->cold_ready[s]));
        cudaFreeHost(L->cold[s]); L->cold[s] = nullptr;
        cudaEventDestroy(L->cold_ready[s]); L->cold_ready[s] = nullptr;
        freed += L->seg_bytes;
    }
    L->trimmed += dropped; L->cold_freed_bytes += freed;
    if (dropped_entries) *dropped_entries = dropped;
    if (freed_cold_bytes) *freed_cold_bytes = freed;
    return RAFTING_OK;
}

extern "C" int rafting_log_stats(rafting_engine_t* e, uint64_t* out, uint32_t n) {
    if (!e || !e->seglog || !out) return fail(RAFTING_E_INVAL, "entry buffer not configured");
    SegLog* L = e->seglog;
    const uint64_t v[] = {L->appended, L->head, L->spilled_bytes, L->hbm_hits, L->cold_hits, L->indexed,
                          (uint64_t)(L->last_gather_kernel_ms * 1e6), L->last_gather_bytes,
                          L->trimmed, L->cold_freed_bytes, L->spills_skipped};
    for (uint32_t i = 0; i < n && i < 11; i++) out[i] = v[i];
    return 11;
}

// ---------------------------------------------------------------------------------------------------------------------
// Durable tier (SURVEY §8(f)-1: "crash-durable spill file replacing flushWal(true)", RocksLog.java:87,195).  Every appended
// record is framed into an append-only file BEFORE it is scattered into HBM (write-ahead); rafting_log_sync is the one
// durability barrier per step (fdatasync) the pump issues before it releases the step's replies.  Truncations and
// compactions — which in the engine are pure metadata (the stored key range lives in the step kernel's tables) — are
// logged as RANGE / EPOCH marks by the pump, so that recovery does not resurrect a truncated suffix.  Little-endian frames:
//     { magic 'RLE1', kind, gid, len, a, b, crc32c(header[0..32) ++ payload), pad }  + payload padded to 8 bytes
//     PUT a = index, b = term | RANGE a = lowest stored key, b = highest (a > b: empty) | EPOCH a = epoch.index, b = epoch.term
// The file is also the coldest read tier (pread), which is what allows the pinned pool to be bounded.
// ---------------------------------------------------------------------------------------------------------------------
namespace {
constexpr uint32_t WAL_MAGIC = 0x31454C52u;   // "RLE1"
enum { WAL_PUT = 1, WAL_RANGE = 2, WAL_EPOCH = 3 };
struct WalHdr { uint32_t magic, kind, gid, len; int64_t a, b; uint32_t crc, pad; };
static_assert(sizeof(WalHdr) == 40, "entry file frame header");
uint32_t wal_crc_table[256]; bool wal_crc_ready = false;
uint32_t wal_crc32c(const void* p, size_t n, uint32_t c) {
    if (!wal_crc_ready) {
        for (uint32_t i = 0; i < 256; i++) { uint32_t v = i; for (int k = 0; k < 8; k++) v = (v & 1) ? (v >> 1) ^ 0x82F63B78u : v >> 1; wal_crc_table[i] = v; }
        wal_crc_ready = true;
    }
    const uint8_t* b = (const uint8_t*)p; c = ~c;
    for (size_t i = 0; i < n; i++) c = wal_crc_table[(c ^ b[i]) & 0xff] ^ (c >> 8);
    return ~c;
}
void wal_frame(std::vector<uint8_t>& buf, uint32_t kind, uint32_t gid, uint32_t len, int64_t a, int64_t b, const uint8_t* payload) {
    WalHdr h; h.magic = WAL_MAGIC; h.kind = kind; h.gid = gid; h.len = len; h.a = a; h.b = b; h.pad = 0;
    h.crc = wal_crc32c(payload, len, wal_crc32c(&h, 32, 0));
    const size_t at = buf.size(), padded = ((size_t)len + 7) & ~(size_t)7;
    buf.resize(at + sizeof(h) + padded, 0);
    memcpy(buf.data() + at, &h, sizeof(h));
    if (len) memcpy(buf.data() + at + sizeof(h), payload, len);
}
bool wal_write_all(int fd, const uint8_t* p, size_t n) {
    while (n) { const ssize_t w = write(fd, p, n); if (w < 0) { if (errno == EINTR) continue; return false; } p += w; n -= (size_t)w; }
    return true;
}
}  // namespace

static int seglog_wal_flush(SegLog* L) {
    if (L->wal_buf.empty()) return RAFTING_OK;
    if (L->wal_failed) return fail(RAFTING_E_CUDA, "entry file is failed (an earlier write error): reopen the store");
    if (!wal_write_all(L->wal_fd, L->wal_buf.data(), L->wal_buf.size())) {
        // the index already points into the unwritten tail: no later record may be acknowledged as durable
        L->wal_failed = true;
        return fail(RAFTING_E_CUDA, "entry file write failed: %s", strerror(errno));
    }
    L->wal_buf.clear();
    return RAFTING_OK;
}
static int seglog_wal_put(SegLog* L, const rafting_entry_ref_t* refs, uint32_t n, const uint8_t* blob, std::vector<uint64_t>& file_offs) {
    if (L->wal_failed) return fail(RAFTING_E_CUDA, "entry file is failed (an earlier write error): reopen the store");
    file_offs.resize(n);
    for (uint32_t i = 0; i < n; i++) {
        file_offs[i] = L->wal_bytes + sizeof(WalHdr);
        wal_frame(L->wal_buf, WAL_PUT, refs[i].gid, refs[i].len, refs[i].index, refs[i].term, blob + refs[i].blob_off);
        L->wal_bytes += sizeof(WalHdr) + (((uint64_t)refs[i].len + 7) & ~7ull);
    }
    if (L->wal_buf.size() > (8u << 20)) return seglog_wal_flush(L);
    return RAFTING_OK;
}

// opens (creates) the entry file and replays what it holds into the host index: the HBM arena starts empty, recovered
// records are served from the file.  cold_max_segments bounds the pinned-host pool (0 = unbounded).
extern "C" int rafting_log_store_open(rafting_engine_t* e, const char* path, uint32_t cold_max_segments, uint64_t* recovered_records) {
    if (!e || !e->seglog || !path) return fail(RAFTING_E_INVAL, "entry buffer not configured (rafting_log_config)");
    SegLog* L = e->seglog;
    if (L->wal_fd >= 0) return fail(RAFTING_E_INVAL, "entry file already open");
    if (L->gathers) return fail(RAFTING_E_BUSY, "a gather has not been waited for (rafting_log_gather_wait / _step_wait)");
    if (L->appended) return fail(RAFTING_E_INVAL, "open the entry file before the first append");
    try {
        const int fd = open(path, O_RDWR | O_CREAT, 0644);
        if (fd < 0) return fail(RAFTING_E_CUDA, "open %s: %s", path, strerror(errno));
        uint64_t pos = 0, recs = 0;
        std::vector<uint8_t> pay;
        for (;;) {
            WalHdr h;
            if (pread(fd, &h, sizeof(h), (off_t)pos) != (ssize_t)sizeof(h)) break;
            if (h.magic != WAL_MAGIC || h.kind < WAL_PUT || h.kind > WAL_EPOCH || h.gid >= e->G || h.len > L->seg_bytes) break;
            const size_t padded = ((size_t)h.len + 7) & ~(size_t)7;
            pay.resize(padded);
            if (padded && pread(fd, pay.data(), padded, (off_t)(pos + sizeof(h))) != (ssize_t)padded) break;
            if (wal_crc32c(pay.data(), h.len, wal_crc32c(&h, 32, 0)) != h.crc) break;
            rafting::GroupIdx& gi = L->index[h.gid];
            if (h.kind == WAL_PUT) {
                if (h.a <= 0) break;
                HostLoc hl; hl.off = rafting::NO_ARENA; hl.len = h.len; hl.term = h.b; hl.file_off = pos + sizeof(h);
                seglog_put(L, h.gid, h.a, hl, 0);
            } else if (h.kind == WAL_RANGE) {
                for (size_t k = 0; k < gi.v.size(); k++) {
                    const int64_t idx = gi.base + (int64_t)k;
                    if ((idx < h.a || idx > h.b) && gi.v[k].len != 0xffffffffu) { seglog_drop(L, gi.v[k]); gi.v[k].len = 0xffffffffu; }
                }
            } else { gi.epoch_index = h.a; gi.epoch_term = h.b; }
            pos += sizeof(h) + padded; recs++;
        }
        if (ftruncate(fd, (off_t)pos) != 0 || lseek(fd, (off_t)pos, SEEK_SET) < 0) { close(fd); return fail(RAFTING_E_CUDA, "cannot position the entry file: %s", strerror(errno)); }
        L->wal_fd = fd; L->wal_bytes = pos; L->wal_synced = pos; L->cold_max = cold_max_segments;
        if (recovered_records) *recovered_records = recs;
    } catch (const std::exception& ex) { return fail(RAFTING_E_NOMEM, "rafting_log_store_open: %s", ex.what()); }
    return RAFTING_OK;
}
// the durability barrier of a step: everything appended / marked so far is on stable storage when this returns 0
extern "C" int rafting_log_sync(rafting_engine_t* e) {
    if (!e || !e->seglog) return fail(RAFTING_E_INVAL, "entry buffer not configured");
    SegLog* L = e->seglog;
    if (L->wal_fd < 0) return fail(RAFTING_E_INVAL, "no entry file (rafting_log_store_open)");
    int rc = seglog_wal_flush(L); if (rc) return rc;
    if (L->wal_synced == L->wal_bytes) return RAFTING_OK;
    if (fdatasync(L->wal_fd) != 0) { L->wal_failed = true; return fail(RAFTING_E_CUDA, "fdatasync of the entry file failed: %s", strerror(errno)); }
    L->wal_synced = L->wal_bytes; L->wal_syncs++;
    return RAFTING_OK;
}
// RocksLog.truncate / flush are deleteRange calls (RocksLog.java:219-242): the pump logs the group's new stored key range
// (and epoch) so that recovery agrees with the tables.  lo > hi: the store is empty.
extern "C" int rafting_log_mark(rafting_engine_t* e, uint32_t gid, int64_t lo, int64_t hi, int64_t epoch_index, int64_t epoch_term) {
    if (!e || !e->seglog || gid >= e->G) return fail(RAFTING_E_INVAL, "bad argument");
    SegLog* L = e->seglog;
    if (L->wal_fd < 0) return fail(RAFTING_E_INVAL, "no entry file (rafting_log_store_open)");
    if (L->wal_failed) return fail(RAFTING_E_CUDA, "entry file is failed: reopen the store");
    try {
        wal_frame(L->wal_buf, WAL_RANGE, gid, 0, lo, hi, nullptr); L->wal_bytes += sizeof(WalHdr);
        wal_frame(L->wal_buf, WAL_EPOCH, gid, 0, epoch_index, epoch_term, nullptr); L->wal_bytes += sizeof(WalHdr);
        L->index[gid].epoch_index = epoch_index; L->index[gid].epoch_term = epoch_term;
    } catch (const std::exception& ex) { return fail(RAFTING_E_NOMEM, "rafting_log_mark: %s", ex.what()); }
    return RAFTING_OK;
}
// what RaftContext.initialize needs from a recovered log (RaftContext.java:91-113): epoch, stored key range, last term and
// the index->term runs (oldest first) for rafting_group_open + rafting_group_load_runs.  *n_runs > cap: RAFTING_E_CAPACITY.
extern "C" int rafting_log_recovered(rafting_engine_t* e, uint32_t gid, rafting_group_init_t* init, rafting_i64x2_t* runs, uint32_t cap, uint32_t* n_runs) {
    if (!e || !e->seglog || gid >= e->G || !init || !n_runs) return fail(RAFTING_E_INVAL, "bad argument");
    const rafting::GroupIdx& gi = e->seglog->index[gid];
    memset(init, 0, sizeof(*init));
    init->ballot = -1; init->epoch_index = gi.epoch_index; init->epoch_term = gi.epoch_term; init->first_index = 1; init->last_index = 0;
    *n_runs = 0;
    // the stored range is the CONTIGUOUS run of records that ends at the highest one (RocksLog keeps its keys contiguous)
    int64_t hi = -1;
    for (size_t k = gi.v.size(); k-- > 0;) if (gi.v[k].len != 0xffffffffu) { hi = gi.base + (int64_t)k; break; }
    if (hi < 0) return RAFTING_OK;
    int64_t lo = hi;
    while (lo - 1 >= gi.base && gi.v[(size_t)(lo - 1 - gi.base)].len != 0xffffffffu) lo--;
    init->first_index = lo; init->last_index = hi; init->last_term = gi.v[(size_t)(hi - gi.base)].term;
    uint32_t nr = 0; int64_t t = 0;
    for (int64_t i = lo; i <= hi; i++) {
        const int64_t ti = gi.v[(size_t)(i - gi.base)].term;
        if (i == lo || ti != t) { if (runs && nr < cap) { runs[nr].x = i; runs[nr].y = ti; } nr++; t = ti; }
    }
    *n_runs = nr;
    return nr > cap && runs ? fail(RAFTING_E_CAPACITY, "%u term runs, room for %u", nr, cap) : RAFTING_OK;
}
// one stored entry in the reference's RocksDB layout (RocksLog.java:82-89,259-280): key = 8-byte big-endian index,
// value = 8-byte big-endian term || payload — what src/test/java/.../cluster/LogChecker.java iterates over
extern "C" int rafting_log_export_kv(rafting_engine_t* e, uint32_t gid, int64_t index, uint8_t key_out[8], void* val_out, size_t val_cap, size_t* val_len) {
    if (!e || !e->seglog || gid >= e->G || !key_out || !val_out || !val_len) return fail(RAFTING_E_INVAL, "bad argument");
    SegLog* L = e->seglog;
    CU(cudaSetDevice(e->cfg.device));
    const HostLoc* hl = seglog_find(L, gid, index);
    if (!hl) return fail(RAFTING_E_INVAL, "no such entry");
    if (val_cap < 8 + (size_t)hl->len) return fail(RAFTING_E_CAPACITY, "value needs %zu bytes", 8 + (size_t)hl->len);
    for (int i = 0; i < 8; i++) { key_out[i] = (uint8_t)((uint64_t)index >> (56 - 8 * i)); ((uint8_t*)val_out)[i] = (uint8_t)((uint64_t)hl->term >> (56 - 8 * i)); }
    if (hl->len) { int rc = seglog_fetch(e, L, *hl, (uint8_t*)val_out + 8); if (rc) return rc; CU(cudaStreamSynchronize(L->s_log)); }
    *val_len = 8 + hl->len;
    return RAFTING_OK;
}
extern "C" int rafting_log_store_stats(rafting_engine_t* e, uint64_t out[6]) {
    if (!e || !e->seglog || !out) return fail(RAFTING_E_INVAL, "entry buffer not configured");
    SegLog* L = e->seglog;
    out[0] = L->wal_bytes; out[1] = L->wal_synced; out[2] = L->wal_syncs; out[3] = L->file_hits; out[4] = L->cold_evicted;
    uint64_t live = 0; for (auto p : L->cold) if (p) live++;
    out[5] = live;
    return RAFTING_OK;
}
