// timers.cuh — the groups whose timers are due: the due query (include/rafting_b200.h, rafting_timers_due_begin) and the tail
// of a due step (rafting_step_begin_compact_due, compact.cuh).
//
// A sweep row at time t (rafting_inbox_t.row_now[r] = t) fires the implied RAFTING_OP_TIMEOUT of every listed group for which
// timer_fires (handlers.cuh) holds.  A pump that runs steps over active lists needs to know, without holding the timers on the
// host, which groups a sweep at t would fire.  due_select answers that from g_meta and g_timer with launches on the engine's
// step stream (so it sees every step begun before it):
//
//   due_member_kernel  only when a host list is given: one thread per listed gid sets its bit in a G-bit mask (zeroed before)
//   due_scan_kernel    one thread per group reads its two 8-byte words (16 B per group): an unlisted group is due or idle, each
//                      bit goes into a 32-bit warp mask (the idle one only with fillers), and each block leaves a DueAgg (number due, number idle, earliest armed
//                      deadline after t)
//   cub::DeviceScan    exclusive scan of the block aggregates (sum, sum, min): every block's first due and first idle position
//   due_emit_kernel    one thread per group again, from the masks only: the due gids in increasing order at [0, cap), then,
//                      when asked for, the idle ones (fillers) from min(due total, cap); the last block writes the due total and
//                      the next deadline
//
// The order-preserving compaction is a two-pass block scan instead of CUB DeviceSelect: DeviceSelect cannot stop at cap
// entries (it writes every selected item), and the min-reduction of the deadlines would be a second pass over the 16 B per
// group; here the scan carries the counts and the minimum together, and the second pass reads 4 B per 32 groups (8 B with
// fillers).  Fillers are a template parameter of the scan and emit kernels, so the query, which never asks for them, neither
// ballots nor stores nor reads the idle mask.
//
// The query lists nothing and asks for no fillers.  Its list is written where the caller reads it: into the caller's buffer
// directly when it is mapped pinned memory (every cudaHostAlloc / pinned allocation on a 64-bit host), else into a mapped pinned
// staging block of the query slot, copied into the caller's buffer at the wait.  Either way only the n_due entries cross PCIe,
// not cap; DESIGN.md "Timers" has the measurement.
// A due step lists the host's gids and asks for fillers: they keep the step's n host-known, so unpack / step / pack run unchanged
// over the device-written gids column, and a listed group with no event whose timer is not due is left untouched by a sweep row.
//
// Included at the end of engine.cu (same translation unit: it uses rafting_engine, HostPath, fail(), CU()).
#pragma once
#include <cub/device/device_scan.cuh>

namespace rafting {

constexpr uint32_t DUE_TPB = 256, DUE_WARPS = DUE_TPB / 32;

// unlisted groups due at `until`, unlisted groups not due, earliest armed deadline after `until` (of a block, then of a prefix)
struct DueAgg { uint32_t due, idle; int64_t next; };
struct DueAggOp {
    __host__ __device__ DueAgg operator()(const DueAgg& a, const DueAgg& b) const {
        return DueAgg{a.due + b.due, a.idle + b.idle, a.next < b.next ? a.next : b.next};
    }
};
struct DueResult { uint32_t n_due, _pad; int64_t next; };   // what the query's wait reports, written by due_emit_kernel

__global__ void due_member_kernel(const uint32_t* __restrict__ gids, uint32_t n_host, uint32_t* __restrict__ member) {
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k < n_host) { const uint32_t g = gids[k]; atomicOr(member + (g >> 5), 1u << (g & 31u)); }
}

// member: the G-bit mask of the listed groups, or null when nothing is listed.  FILL: the idle groups are counted and get a
// second warp mask (mask holds 2 words per warp, else 1); without it a block's idle count is 0.
template <bool FILL>
__global__ void __launch_bounds__(DUE_TPB) due_scan_kernel(Tables T, int64_t until, const uint32_t* __restrict__ member,
                                                           uint32_t* __restrict__ mask, DueAgg* __restrict__ agg) {
    __shared__ uint32_t wdue[DUE_WARPS], widle[DUE_WARPS];
    __shared__ int64_t wmin[DUE_WARPS];
    const uint32_t g = blockIdx.x * DUE_TPB + threadIdx.x;
    bool due = false, idle = false; int64_t next = I64MAX;
    if (g < T.G) {
        const uint32_t w = (uint32_t)T.g_meta[g];
        const int64_t timer = T.g_timer[g];
        const bool listed = member && ((member[g >> 5] >> (g & 31u)) & 1u);
        due = !listed && timer_fires(w, timer, until);
        idle = !listed && !due;
        if (timer_armed(w, timer) && timer > until) next = timer;            // a later sweep would fire it
    }
    const uint32_t lane = threadIdx.x & 31u, wq = threadIdx.x >> 5;
    const uint32_t md = __ballot_sync(0xffffffffu, due), mi = FILL ? __ballot_sync(0xffffffffu, idle) : 0u;
    for (int o = 16; o > 0; o >>= 1) { const int64_t v = __shfl_down_sync(0xffffffffu, next, o); next = v < next ? v : next; }
    if (lane == 0) {
        const size_t at = (size_t)blockIdx.x * DUE_WARPS + wq;
        if (FILL) { mask[2 * at] = md; mask[2 * at + 1] = mi; } else mask[at] = md;
        wdue[wq] = __popc(md); widle[wq] = __popc(mi); wmin[wq] = next;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        DueAgg a{0, 0, I64MAX};
        for (uint32_t k = 0; k < DUE_WARPS; k++) a = DueAggOp()(a, DueAgg{wdue[k], widle[k], wmin[k]});
        agg[blockIdx.x] = a;
    }
}

// out[0, cap): the due gids, then (FILL) the idle ones, each in increasing order; the last block writes *n_due and, unless next
// is null, *next.  A block whose positions all lie past cap returns once the totals are out.
template <bool FILL>
__global__ void __launch_bounds__(DUE_TPB) due_emit_kernel(const uint32_t* __restrict__ mask, const DueAgg* __restrict__ agg,
                                                           const DueAgg* __restrict__ off, uint32_t nblocks, uint32_t* __restrict__ out,
                                                           uint32_t cap, uint32_t* __restrict__ n_due, int64_t* __restrict__ next) {
    constexpr uint32_t MW = FILL ? 2 : 1;                                  // mask words per warp
    __shared__ uint32_t bdue[DUE_WARPS], bidle[DUE_WARPS];
    if (blockIdx.x == nblocks - 1 && threadIdx.x == 0) {
        const DueAgg t = DueAggOp()(off[blockIdx.x], agg[blockIdx.x]);
        *n_due = t.due;
        if (next) *next = t.next;
    }
    uint32_t first_filler = 0;
    if (FILL) { const uint32_t d = off[nblocks - 1].due + agg[nblocks - 1].due; first_filler = d < cap ? d : cap; }
    const DueAgg o = off[blockIdx.x];
    if (o.due >= cap && (!FILL || (uint64_t)first_filler + o.idle >= cap)) return;
    const uint32_t* bm = mask + (size_t)blockIdx.x * DUE_WARPS * MW;
    if (threadIdx.x == 0) {
        uint32_t d = o.due, i = o.idle;
        for (uint32_t k = 0; k < DUE_WARPS; k++) {
            bdue[k] = d; d += __popc(bm[MW * k]);
            if (FILL) { bidle[k] = i; i += __popc(bm[MW * k + 1]); }
        }
    }
    __syncthreads();
    const uint32_t lane = threadIdx.x & 31u, wq = threadIdx.x >> 5, below = (1u << lane) - 1u;
    const uint32_t md = bm[MW * wq];
    const uint32_t g = blockIdx.x * DUE_TPB + threadIdx.x;
    if ((md >> lane) & 1u) {
        const uint32_t pos = bdue[wq] + __popc(md & below);
        if (pos < cap) out[pos] = g;
    } else if (FILL) {
        const uint32_t mi = bm[MW * wq + 1];
        if ((mi >> lane) & 1u) {
            const uint64_t pos = (uint64_t)first_filler + bidle[wq] + __popc(mi & below);
            if (pos < cap) out[pos] = g;
        }
    }
}

}  // namespace rafting

// device scratch of one selection over G groups: member mask, warp masks, block aggregates, their scan, CUB's scratch
struct DueLayout { size_t member, mask, agg, off, tmp, total; uint32_t nblocks; };
static int due_layout(uint32_t G, DueLayout& L) {
    using namespace rafting;
    L.nblocks = (G + DUE_TPB - 1) / DUE_TPB;
    size_t scan_tmp = 0;
    CU(cub::DeviceScan::ExclusiveScan(nullptr, scan_tmp, (DueAgg*)nullptr, (DueAgg*)nullptr, DueAggOp(), DueAgg{0, 0, I64MAX}, (int)L.nblocks));
    Carve c;
    L.member = c.take((size_t)L.nblocks * DUE_WARPS * 4); L.mask = c.take((size_t)L.nblocks * DUE_WARPS * 8);
    L.agg = c.take((size_t)L.nblocks * sizeof(DueAgg)); L.off = c.take((size_t)L.nblocks * sizeof(DueAgg)); L.tmp = c.take(scan_tmp);
    L.total = c.o;
    return RAFTING_OK;
}

// Enqueues the selection on the engine's stream: the groups a sweep at `until` fires, except the n_host gids of list (device
// memory), go to out[0 .. cap) and, when `fill`, the groups that are neither listed nor due after them; the due total goes to
// *n_due and, unless next is null, the earliest armed deadline after `until` (INT64_MAX: none) to *next.  scratch holds L.total
// bytes, L = due_layout(G).
static int due_select(rafting_engine* e, const DueLayout& L, uint8_t* scratch, int64_t until, const uint32_t* list, uint32_t n_host,
                      uint32_t* out, uint32_t cap, bool fill, uint32_t* n_due, int64_t* next) {
    using namespace rafting;
    uint32_t* member = nullptr;
    if (n_host) {
        member = (uint32_t*)(scratch + L.member);
        CU(cudaMemsetAsync(member, 0, (size_t)L.nblocks * DUE_WARPS * 4, e->stream));
        due_member_kernel<<<(n_host + 255u) / 256u, 256, 0, e->stream>>>(list, n_host, member);
    }
    uint32_t* mask = (uint32_t*)(scratch + L.mask); DueAgg* agg = (DueAgg*)(scratch + L.agg); DueAgg* off = (DueAgg*)(scratch + L.off);
    auto scan = fill ? due_scan_kernel<true> : due_scan_kernel<false>;
    auto emit = fill ? due_emit_kernel<true> : due_emit_kernel<false>;
    scan<<<L.nblocks, DUE_TPB, 0, e->stream>>>(e->T, until, member, mask, agg);
    size_t tb = L.total - L.tmp;
    CU(cub::DeviceScan::ExclusiveScan(scratch + L.tmp, tb, agg, off, DueAggOp(), DueAgg{0, 0, I64MAX}, (int)L.nblocks, e->stream));
    emit<<<L.nblocks, DUE_TPB, 0, e->stream>>>(mask, agg, off, L.nblocks, out, cap, n_due, next);
    CU(cudaGetLastError());
    return RAFTING_OK;
}

// One query slot: device scratch, a pinned (so mapped) block for the result (and the list when the caller's buffer is not mapped)
struct DueSlot {
    Blk dev;                                               // due_layout(G).total bytes
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
    DueLayout L;
    if (int rc = due_layout(e->G, L)) return rc;
    if (int rc = blk_reserve(S.dev, L.total, false)) return rc;
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
    DueResult* res = (DueResult*)hdev;
    if (int rc = due_select(e, L, S.dev.p, until_ms, nullptr, 0, (uint32_t*)dst, cap, false, &res->n_due, &res->next)) return rc;
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
