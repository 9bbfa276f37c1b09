// timers.cuh — the list of groups whose timers are due (include/rafting_b200.h, rafting_timers_due_begin).
//
// A sweep row at time t (rafting_inbox_t.row_now[r] = t) fires the implied RAFTING_OP_TIMEOUT of every listed group for which
//     alive && (leader ? timer <= t : timer > 0 && timer != INT64_MAX && timer <= t)
// holds (step_body.inc, pair_kernel.cuh).  A pump that runs steps over active lists needs to know, without holding the timers
// on the host, which groups a sweep at t would fire.  Three launches on the engine's step stream (so a query sees every step
// begun before it) answer that from g_meta and g_timer:
//
//   due_scan_kernel   one thread per group reads its two 8-byte words (16 B per group): the due bit goes into a 32-bit warp
//                     mask, and each block leaves (number due, earliest armed deadline after t) for the scan
//   cub::DeviceScan   exclusive scan of the block pairs (sum, min): every block's first output position, and from the last
//                     block the count and next deadline of the whole shard
//   due_emit_kernel   one thread per group again, from the masks only (1 bit per group): the due gids, in increasing order,
//                     at their positions below cap; the last block writes (count, next deadline)
//
// The order-preserving compaction is a two-pass block scan instead of CUB DeviceSelect: DeviceSelect cannot stop at cap
// entries (it writes every selected item), and the min-reduction of the deadlines would be a second pass over the 16 B per
// group; here the scan carries the count and the minimum together, and the second pass reads 4 B per 32 groups.
// The list is written where the caller reads it: into the caller's buffer directly when it is mapped pinned memory (every
// cudaHostAlloc / pinned allocation on a 64-bit host), else into a mapped pinned staging block of the query slot, copied into the
// caller's buffer at the wait.  Either way only the n_due entries cross PCIe, not cap; DESIGN.md "Timers" has the measurement.
//
// Included at the end of engine.cu (same translation unit: it uses rafting_engine, HostPath, fail(), CU()).
#pragma once
#include <cub/device/device_scan.cuh>

namespace rafting {

constexpr uint32_t DUE_TPB = 256;

struct DueAgg { uint32_t count, _pad; int64_t next; };      // due groups of a block, earliest armed deadline after `until`
struct DueAggOp {
    __host__ __device__ DueAgg operator()(const DueAgg& a, const DueAgg& b) const {
        DueAgg r; r.count = a.count + b.count; r._pad = 0; r.next = a.next < b.next ? a.next : b.next; return r;
    }
};
struct DueResult { uint32_t n_due, _pad; int64_t next; };   // what the wait reports, written by the last block of due_emit_kernel

__global__ void __launch_bounds__(DUE_TPB) due_scan_kernel(Tables T, int64_t until, uint32_t* __restrict__ mask, DueAgg* __restrict__ agg) {
    __shared__ uint32_t wcnt[DUE_TPB / 32];
    __shared__ int64_t wmin[DUE_TPB / 32];
    const uint32_t g = blockIdx.x * DUE_TPB + threadIdx.x;
    bool due = false; int64_t next = I64MAX;
    if (g < T.G) {
        const uint32_t w = (uint32_t)T.g_meta[g];
        const int64_t timer = T.g_timer[g];
        const bool alive = (w & W_ALIVE) != 0, leader = (w & W_ROLE_MASK) == RAFTING_ROLE_LEADER;
        // the sweep's predicate at t = until; a deadline it would fire at a later t is armed
        const bool armed = alive && (leader || (timer > 0 && timer != I64MAX));
        due = armed && timer <= until;
        if (armed && timer > until) next = timer;
    }
    const uint32_t lane = threadIdx.x & 31u, wq = threadIdx.x >> 5;
    const uint32_t m = __ballot_sync(0xffffffffu, due);
    for (int o = 16; o > 0; o >>= 1) { const int64_t v = __shfl_down_sync(0xffffffffu, next, o); next = v < next ? v : next; }
    if (lane == 0) { mask[(size_t)blockIdx.x * (DUE_TPB / 32) + wq] = m; wcnt[wq] = __popc(m); wmin[wq] = next; }
    __syncthreads();
    if (threadIdx.x == 0) {
        DueAgg a; a.count = 0; a._pad = 0; a.next = I64MAX;
        for (uint32_t k = 0; k < DUE_TPB / 32; k++) { a.count += wcnt[k]; if (wmin[k] < a.next) a.next = wmin[k]; }
        agg[blockIdx.x] = a;
    }
}

__global__ void __launch_bounds__(DUE_TPB) due_emit_kernel(const uint32_t* __restrict__ mask, const DueAgg* __restrict__ agg,
                                                           const DueAgg* __restrict__ off, uint32_t nblocks, uint32_t* __restrict__ out,
                                                           uint32_t cap, DueResult* __restrict__ res) {
    __shared__ uint32_t wbase[DUE_TPB / 32];
    const uint32_t lane = threadIdx.x & 31u, wq = threadIdx.x >> 5;
    const uint32_t* bm = mask + (size_t)blockIdx.x * (DUE_TPB / 32);
    if (threadIdx.x == 0) {
        uint32_t b = off[blockIdx.x].count;
        for (uint32_t k = 0; k < DUE_TPB / 32; k++) { wbase[k] = b; b += __popc(bm[k]); }
    }
    __syncthreads();
    const uint32_t m = bm[wq];
    if ((m >> lane) & 1u) {
        const uint32_t pos = wbase[wq] + __popc(m & ((1u << lane) - 1u));
        if (pos < cap) out[pos] = blockIdx.x * DUE_TPB + threadIdx.x;
    }
    if (blockIdx.x == nblocks - 1 && threadIdx.x == 0) {
        const DueAgg t = DueAggOp()(off[blockIdx.x], agg[blockIdx.x]);
        DueResult r; r.n_due = t.count; r._pad = 0; r.next = t.next;
        *res = r;
    }
}

// ---- the tail of a step begun with rafting_step_begin_compact_due ----
// The step's list is the host's gids (positions 0 .. n_host) followed by a tail of cap gids chosen on the step stream, after
// the slot's H2D copy and before unpack_kernel, so the choice sees the state the step itself will see:
//   tail_member_kernel   one thread per host position sets its gid's bit in a G-bit mask (zeroed by a memset before it)
//   tail_scan_kernel     one thread per group, due_scan_kernel's predicate: a due-unlisted and an idle-unlisted bit go into two
//                        warp masks, and each block leaves its two counts packed in one word, due << 32 | idle, so that one
//                        cub::DeviceScan sum carries both (each count stays below 2^32: no carry crosses)
//   tail_emit_kernel     due gids from tail position 0, then idle ones (fillers) from min(due total, cap), both in increasing
//                        order, stopping at cap; one thread writes the due total (counts[3])
// Fillers keep the step's n host-known, so unpack / step / pack run unchanged over the device-written gids column: a listed
// group with no event whose timer is not due is left untouched by a sweep row.  DueAgg does not fit here (two counts, no
// deadline), hence the packed sum.
constexpr uint32_t TAIL_WARPS = DUE_TPB / 32;

__global__ void tail_member_kernel(const uint32_t* __restrict__ gids, uint32_t n_host, uint32_t* __restrict__ member) {
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k < n_host) { const uint32_t g = gids[k]; atomicOr(member + (g >> 5), 1u << (g & 31u)); }
}

__global__ void __launch_bounds__(DUE_TPB) tail_scan_kernel(Tables T, int64_t until, const uint32_t* __restrict__ member,
                                                            uint32_t* __restrict__ mask, uint64_t* __restrict__ agg) {
    __shared__ uint32_t wdue[TAIL_WARPS], widle[TAIL_WARPS];
    const uint32_t g = blockIdx.x * DUE_TPB + threadIdx.x;
    bool due = false, idle = false;
    if (g < T.G) {
        const uint32_t w = (uint32_t)T.g_meta[g];
        const int64_t timer = T.g_timer[g];
        const bool alive = (w & W_ALIVE) != 0, leader = (w & W_ROLE_MASK) == RAFTING_ROLE_LEADER;
        const bool armed = alive && (leader || (timer > 0 && timer != I64MAX));
        const bool listed = (member[g >> 5] >> (g & 31u)) & 1u;
        due = !listed && armed && timer <= until;
        idle = !listed && !due;
    }
    const uint32_t lane = threadIdx.x & 31u, wq = threadIdx.x >> 5;
    const uint32_t md = __ballot_sync(0xffffffffu, due), mi = __ballot_sync(0xffffffffu, idle);
    if (lane == 0) {
        const size_t at = ((size_t)blockIdx.x * TAIL_WARPS + wq) * 2;
        mask[at] = md; mask[at + 1] = mi; wdue[wq] = __popc(md); widle[wq] = __popc(mi);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        uint64_t d = 0, i = 0;
        for (uint32_t k = 0; k < TAIL_WARPS; k++) { d += wdue[k]; i += widle[k]; }
        agg[blockIdx.x] = (d << 32) | i;
    }
}

__global__ void __launch_bounds__(DUE_TPB) tail_emit_kernel(const uint32_t* __restrict__ mask, const uint64_t* __restrict__ agg,
                                                            const uint64_t* __restrict__ off, uint32_t nblocks,
                                                            uint32_t* __restrict__ tail, uint32_t cap, uint32_t* __restrict__ n_due) {
    __shared__ uint32_t bdue[TAIL_WARPS], bidle[TAIL_WARPS];
    const uint64_t total = off[nblocks - 1] + agg[nblocks - 1];
    const uint32_t due_total = (uint32_t)(total >> 32), first_filler = due_total < cap ? due_total : cap;
    if (blockIdx.x == 0 && threadIdx.x == 0) *n_due = due_total;
    const uint64_t o = off[blockIdx.x];
    const uint32_t od = (uint32_t)(o >> 32), oi = (uint32_t)o;
    if (od >= cap && (uint64_t)first_filler + oi >= cap) return;          // every entry of this block lies past the tail
    const uint32_t* bm = mask + (size_t)blockIdx.x * TAIL_WARPS * 2;
    if (threadIdx.x == 0) {
        uint32_t d = od, i = oi;
        for (uint32_t k = 0; k < TAIL_WARPS; k++) { bdue[k] = d; bidle[k] = i; d += __popc(bm[2 * k]); i += __popc(bm[2 * k + 1]); }
    }
    __syncthreads();
    const uint32_t lane = threadIdx.x & 31u, wq = threadIdx.x >> 5, below = (1u << lane) - 1u;
    const uint32_t md = bm[2 * wq], mi = bm[2 * wq + 1];
    const uint32_t g = blockIdx.x * DUE_TPB + threadIdx.x;
    if ((md >> lane) & 1u) {
        const uint32_t pos = bdue[wq] + __popc(md & below);
        if (pos < cap) tail[pos] = g;
    } else if ((mi >> lane) & 1u) {
        const uint64_t pos = (uint64_t)first_filler + bidle[wq] + __popc(mi & below);
        if (pos < cap) tail[pos] = g;
    }
}

}  // namespace rafting

// device scratch of one tail selection over G groups: member mask, warp masks, block counts, their scan, CUB's scratch
struct TailLayout { size_t member, mask, agg, off, tmp, total; uint32_t nblocks; };
static int tail_layout(uint32_t G, TailLayout& L) {
    using namespace rafting;
    L.nblocks = (G + DUE_TPB - 1) / DUE_TPB;
    size_t scan_tmp = 0;
    CU(cub::DeviceScan::ExclusiveSum(nullptr, scan_tmp, (const uint64_t*)nullptr, (uint64_t*)nullptr, (int)L.nblocks));
    Carve c;
    L.member = c.take((size_t)L.nblocks * TAIL_WARPS * 4); L.mask = c.take((size_t)L.nblocks * TAIL_WARPS * 8);
    L.agg = c.take((size_t)L.nblocks * 8); L.off = c.take((size_t)L.nblocks * 8); L.tmp = c.take(scan_tmp);
    L.total = c.o;
    return RAFTING_OK;
}
static int tail_reserve(rafting_engine* e, Blk& scratch) {
    TailLayout L;
    if (int rc = tail_layout(e->G, L)) return rc;
    return blk_reserve(scratch, L.total, false);
}

// Enqueues the tail selection on the engine's stream: list[0 .. n_host) is the host's part (device copy), the tail goes to
// list[n_host .. n_host + cap), the due total to *n_due.  scratch holds tail_layout(G).total bytes.
static int tail_select(rafting_engine* e, uint8_t* scratch, int64_t until, uint32_t* list, uint32_t n_host, uint32_t cap, uint32_t* n_due) {
    using namespace rafting;
    TailLayout L;
    if (int rc = tail_layout(e->G, L)) return rc;
    uint32_t* member = (uint32_t*)(scratch + L.member); uint32_t* mask = (uint32_t*)(scratch + L.mask);
    uint64_t* agg = (uint64_t*)(scratch + L.agg); uint64_t* off = (uint64_t*)(scratch + L.off);
    CU(cudaMemsetAsync(member, 0, (size_t)L.nblocks * TAIL_WARPS * 4, e->stream));
    if (n_host) tail_member_kernel<<<(n_host + 255u) / 256u, 256, 0, e->stream>>>(list, n_host, member);
    tail_scan_kernel<<<L.nblocks, DUE_TPB, 0, e->stream>>>(e->T, until, member, mask, agg);
    size_t tb = L.total - L.tmp;
    CU(cub::DeviceScan::ExclusiveSum(scratch + L.tmp, tb, agg, off, (int)L.nblocks, e->stream));
    tail_emit_kernel<<<L.nblocks, DUE_TPB, 0, e->stream>>>(mask, agg, off, L.nblocks, list + n_host, cap, n_due);
    CU(cudaGetLastError());
    return RAFTING_OK;
}

// One query slot: device scratch, a pinned (so mapped) block for the result (and the list when the caller's buffer is not mapped)
struct DueSlot {
    Blk dev;                                               // mask, block pairs, their scan, CUB's scratch
    Blk host;                                              // DueResult, then the staged list
    cudaEvent_t ev = nullptr;
    bool inflight = false;
    uint32_t* user = nullptr; uint32_t cap = 0;            // the caller's buffer; staged: copy from host + 256 at the wait
    bool staged = false;
};
struct DuePath { DueSlot slot[RAFTING_HOST_SLOTS]; };

static void due_release(rafting_engine* e) {
    if (!e->due) return;
    for (DueSlot& s : e->due->slot) {
        blk_free(s.dev, false);
        blk_free(s.host, true);
        if (s.ev) cudaEventDestroy(s.ev);
    }
    delete e->due; e->due = nullptr;
}

extern "C" int rafting_timers_due_begin(rafting_engine_t* e, uint32_t slot, int64_t until_ms, uint32_t* gids_out, uint32_t cap) {
    using namespace rafting;
    if (!e || slot >= RAFTING_HOST_SLOTS || (cap && !gids_out)) return fail(RAFTING_E_INVAL, "bad argument");
    CU(cudaSetDevice(e->cfg.device));
    if (!e->due) e->due = new DuePath();
    DueSlot& S = e->due->slot[slot];
    if (S.inflight) return fail(RAFTING_E_BUSY, "due-query slot %u has a query in flight", slot);
    if (!S.ev) CU(cudaEventCreateWithFlags(&S.ev, cudaEventDisableTiming));
    const uint32_t nblocks = (e->G + DUE_TPB - 1) / DUE_TPB;
    size_t scan_tmp = 0;
    CU(cub::DeviceScan::ExclusiveScan(nullptr, scan_tmp, (DueAgg*)nullptr, (DueAgg*)nullptr, DueAggOp(), DueAgg{0, 0, I64MAX}, (int)nblocks));
    Carve c;
    const size_t o_mask = c.take((size_t)nblocks * (DUE_TPB / 32) * 4), o_agg = c.take((size_t)nblocks * sizeof(DueAgg));
    const size_t o_off = c.take((size_t)nblocks * sizeof(DueAgg)), o_tmp = c.o;
    if (int rc = blk_reserve(S.dev, o_tmp + scan_tmp, false)) return rc;
    // the caller's buffer, if the device can write it (mapped pinned memory); else the slot's staging block
    void* dst = nullptr;
    bool staged = false;
    if (cap) {
        cudaPointerAttributes pa;
        if (cudaPointerGetAttributes(&pa, gids_out) == cudaSuccess && pa.type == cudaMemoryTypeHost && pa.devicePointer) dst = pa.devicePointer;
        else { cudaGetLastError(); staged = true; }
    }
    if (int rc = blk_reserve(S.host, 256 + (staged ? (size_t)cap * 4 : 0), true)) return rc;
    uint8_t* hdev = nullptr;
    CU(cudaHostGetDevicePointer((void**)&hdev, S.host.p, 0));
    if (staged) dst = hdev + 256;
    uint32_t* mask = (uint32_t*)(S.dev.p + o_mask); DueAgg* agg = (DueAgg*)(S.dev.p + o_agg); DueAgg* off = (DueAgg*)(S.dev.p + o_off);
    due_scan_kernel<<<nblocks, DUE_TPB, 0, e->stream>>>(e->T, until_ms, mask, agg);
    size_t tb = scan_tmp;
    CU(cub::DeviceScan::ExclusiveScan(S.dev.p + o_tmp, tb, agg, off, DueAggOp(), DueAgg{0, 0, I64MAX}, (int)nblocks, e->stream));
    due_emit_kernel<<<nblocks, DUE_TPB, 0, e->stream>>>(mask, agg, off, nblocks, (uint32_t*)dst, cap, (DueResult*)hdev);
    CU(cudaGetLastError());
    CU(cudaEventRecord(S.ev, e->stream));
    S.user = gids_out; S.cap = cap; S.staged = staged;
    S.inflight = true;
    return RAFTING_OK;
}

extern "C" int rafting_timers_due_wait(rafting_engine_t* e, uint32_t slot, uint32_t* n_due, int64_t* next_deadline_ms) {
    using namespace rafting;
    if (!e || slot >= RAFTING_HOST_SLOTS) return fail(RAFTING_E_INVAL, "bad argument");
    if (!e->due || !e->due->slot[slot].inflight) return fail(RAFTING_E_INVAL, "due-query slot %u has no query in flight", slot);
    CU(cudaSetDevice(e->cfg.device));
    DueSlot& S = e->due->slot[slot];
    CU(cudaEventSynchronize(S.ev));
    S.inflight = false;
    const DueResult* r = (const DueResult*)S.host.p;
    if (S.staged) memcpy(S.user, S.host.p + 256, (size_t)(r->n_due < S.cap ? r->n_due : S.cap) * 4);
    if (n_due) *n_due = r->n_due;
    if (next_deadline_ms) *next_deadline_ms = r->next;
    return RAFTING_OK;
}
