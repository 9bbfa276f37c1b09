// engine.cu — C-ABI implementation (include/rafting_b200.h) over the sm_90a step kernel.
//
// Host-side responsibilities only: table allocation in HBM, pinned staging for the lease/step
// path, kernel dispatch, state export for parity checks, and the NCCL all-gather of the commit
// column.  There is NO CPU fallback: without a CUDA device engine_create fails with
// RAFTING_E_NODEVICE.  Nothing here includes or links oracle/.
#include <cuda_runtime.h>
#include <dlfcn.h>
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <string>
#include <vector>

#include "step_kernel.cuh"

using namespace rafting;

#ifndef RAFTING_HOST_SLOTS
#define RAFTING_HOST_SLOTS 4        // steps that may be in flight on the host path
#endif

static thread_local char g_err[512] = "";
static int fail(int code, const char* fmt, ...) {
    va_list ap; va_start(ap, fmt); vsnprintf(g_err, sizeof(g_err), fmt, ap); va_end(ap);
    return code;
}
#define CU(call)                                                                                  \
    do {                                                                                          \
        cudaError_t _e = (call);                                                                  \
        if (_e != cudaSuccess)                                                                    \
            return fail(RAFTING_E_CUDA, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(_e), __FILE__, __LINE__); \
    } while (0)

// ---- NCCL through dlopen: no link-time dependency, the torch-bundled or system libnccl works ----
typedef struct { char internal[128]; } nccl_uid_t;
typedef void* nccl_comm_t;
struct NcclApi {
    void* h = nullptr;
    int (*GetUniqueId)(nccl_uid_t*) = nullptr;
    int (*CommInitRank)(nccl_comm_t*, int, nccl_uid_t, int) = nullptr;
    int (*AllGather)(const void*, void*, size_t, int, nccl_comm_t, cudaStream_t) = nullptr;
    int (*CommDestroy)(nccl_comm_t) = nullptr;
    int (*GroupStart)() = nullptr;
    int (*GroupEnd)() = nullptr;
    const char* (*GetErrorString)(int) = nullptr;
};
static NcclApi g_nccl;
static int nccl_load() {
    if (g_nccl.h) return 0;
    const char* names[] = {"libnccl.so.2", "libnccl.so"};
    for (const char* n : names) { g_nccl.h = dlopen(n, RTLD_NOW | RTLD_GLOBAL); if (g_nccl.h) break; }
    if (!g_nccl.h) return fail(RAFTING_E_NCCL, "dlopen(libnccl.so.2) failed: %s", dlerror());
    *(void**)&g_nccl.GetUniqueId = dlsym(g_nccl.h, "ncclGetUniqueId");
    *(void**)&g_nccl.CommInitRank = dlsym(g_nccl.h, "ncclCommInitRank");
    *(void**)&g_nccl.AllGather = dlsym(g_nccl.h, "ncclAllGather");
    *(void**)&g_nccl.CommDestroy = dlsym(g_nccl.h, "ncclCommDestroy");
    *(void**)&g_nccl.GetErrorString = dlsym(g_nccl.h, "ncclGetErrorString");
    *(void**)&g_nccl.GroupStart = dlsym(g_nccl.h, "ncclGroupStart");
    *(void**)&g_nccl.GroupEnd = dlsym(g_nccl.h, "ncclGroupEnd");
    if (!g_nccl.GetUniqueId || !g_nccl.CommInitRank || !g_nccl.AllGather)
        return fail(RAFTING_E_NCCL, "libnccl lacks required symbols");
    return 0;
}

struct HostPath;
namespace rafting { struct SegLog; }
struct rafting_engine {
    rafting_cfg_t cfg;
    CfgD dcfg;
    CfgD* d_cfg = nullptr;            // device copy for the slow path (the fast path reads the kernel-param copy)
    Tables T;
    uint32_t G, F;
    cudaStream_t stream = nullptr;
    int64_t* gather[2] = {nullptr, nullptr};   // [world * G] x 2: cross-shard commitIndex summaries, alternating
    uint64_t gather_seq = 0;
    int rank = 0, world = 1;
    nccl_comm_t comm = nullptr;
    cudaStream_t s_comm = nullptr;     // the summary all-gather runs here, off the kernels' critical path
    cudaEvent_t ev_step = nullptr, ev_gather[2] = {nullptr, nullptr};
    struct HostPath* host = nullptr;  // slots, copy streams (created on first use)
    struct rafting::SegLog* seglog = nullptr;   // HBM entry buffer (seglog.cuh), created by rafting_log_config
    cudaEvent_t ev_seg = nullptr;
    uint64_t launches = 0, events = 0;
    bool follows_step = false;         // the launch being made directly follows a step kernel of the same sequence on its stream
    uint32_t lease_counter = 0;
    uint32_t* d_perm = nullptr;        // [NCLS * G] class-sorted positions of the step being launched (classify_kernel)
    uint32_t* d_perm_cnt = nullptr;    // class sizes
    std::vector<void*> dev_allocs;
    std::vector<size_t> dev_bytes;
    std::vector<char>  dev_is_state;   // parallel to dev_allocs: 1 = protocol state (tables, in-flight table), 0 = scratch
    std::vector<void*> shadow;         // rafting_checkpoint copies, parallel to dev_allocs (null for scratch)
    bool alloc_state = true;           // what dalloc marks new allocations as
    struct CompactState* compact = nullptr;   // in-flight table of the compact host path (compact.cuh), created on first use
    struct DuePath* due = nullptr;             // query slots of rafting_timers_due_begin (timers.cuh), created on first use
    struct EditPath* edit = nullptr;           // staging of rafting_group_edit_begin, created on first use
};

template <typename T>
static int dalloc(rafting_engine* e, T** p, size_t count) {
    void* q = nullptr;
    size_t bytes = count * sizeof(T); if (bytes == 0) bytes = 16;
    CU(cudaMalloc(&q, bytes));
    CU(cudaMemset(q, 0, bytes));
    e->dev_allocs.push_back(q);
    e->dev_bytes.push_back(bytes);
    e->dev_is_state.push_back(e->alloc_state ? 1 : 0);
    *p = (T*)q;
    return 0;
}

static void rafting_hostpath_release(rafting_engine* e);
static void seglog_release(rafting_engine* e);
static void compact_release(rafting_engine* e);
static void due_release(rafting_engine* e);
static void edit_release(rafting_engine* e);
static int compact_state(rafting_engine* e);
static uint32_t* compact_bits(rafting_engine* e);
static bool compact_owns(const rafting_engine* e, const void* p);
static int quiesce_for_table_edit(rafting_engine* e, const char* who);
extern "C" uint32_t rafting_abi_version(void) { return RAFTING_ABI_VERSION; }
extern "C" const char* rafting_last_error(void) { return g_err; }

extern "C" int rafting_engine_create(const rafting_cfg_t* cfg, rafting_engine_t** out) {
    if (!cfg || !out) return fail(RAFTING_E_INVAL, "null argument");
    if (cfg->struct_size != sizeof(rafting_cfg_t)) return fail(RAFTING_E_INVAL, "cfg.struct_size %u != %zu", cfg->struct_size, sizeof(rafting_cfg_t));
    if (cfg->flags & ~(uint32_t)(RAFTING_CFG_STRICT_CANDIDATE_VOTE | RAFTING_CFG_LENIENT_FOLLOWER_COMMIT))
        return fail(RAFTING_E_INVAL, "cfg.flags 0x%x: only RAFTING_CFG_STRICT_CANDIDATE_VOTE (1) and RAFTING_CFG_LENIENT_FOLLOWER_COMMIT (2) are defined", cfg->flags);
    if (cfg->replicas < 2 || cfg->replicas > RAFTING_MAX_REPLICAS || cfg->local_slot >= cfg->replicas || cfg->max_groups == 0)
        return fail(RAFTING_E_INVAL, "bad replicas/local_slot/max_groups");
    int ndev = 0;
    cudaError_t ce = cudaGetDeviceCount(&ndev);
    if (ce != cudaSuccess || ndev == 0)
        return fail(RAFTING_E_NODEVICE, "no CUDA device (%s): the engine has no CPU path", cudaGetErrorString(ce));
    if (cfg->device < 0 || cfg->device >= ndev) return fail(RAFTING_E_INVAL, "device %d out of range", cfg->device);
    CU(cudaSetDevice(cfg->device));
    rafting_engine* e = new rafting_engine();
    e->cfg = *cfg;
    e->G = cfg->max_groups; e->F = cfg->replicas - 1;
    e->dcfg.replicas = cfg->replicas; e->dcfg.local_slot = cfg->local_slot;
    e->dcfg.pre_vote = cfg->pre_vote; e->dcfg.avail_critical_point = cfg->avail_critical_point;
    e->dcfg.recovery_cool_down_ms = cfg->recovery_cool_down_ms; e->dcfg.heartbeat_ms = cfg->heartbeat_ms;
    e->dcfg.election_ms = cfg->election_ms; e->dcfg.timer_seed = cfg->timer_seed;
    e->dcfg.flags = cfg->flags; e->dcfg._pad = 0;
    int rc = 0;
    Tables& T = e->T; const size_t G = e->G, F = e->F;
    T.G = e->G; T.F = e->F;
    if ((rc = dalloc(e, &T.g_meta, G)) || (rc = dalloc(e, &T.g_term, G)) || (rc = dalloc(e, &T.g_commit, G)) ||
        (rc = dalloc(e, &T.g_lo, G)) || (rc = dalloc(e, &T.g_hi, G)) || (rc = dalloc(e, &T.g_timer, G)) ||
        (rc = dalloc(e, &T.g_epoch, G)) || (rc = dalloc(e, &T.g_elect, G)) || (rc = dalloc(e, &T.g_err, G)) ||
        (rc = dalloc(e, &T.g_runs, G * KRUNS)) || (rc = dalloc(e, &T.l_nm, G * F)) || (rc = dalloc(e, &T.l_es, G * F)) ||
        (rc = dalloc(e, &T.l_fr, G * F)) || (rc = dalloc(e, &T.l_cnt, G * F))) {
        rafting_engine_destroy(e); return rc;
    }
    e->alloc_state = false;
    if ((rc = dalloc(e, &e->d_cfg, 1)) || (rc = dalloc(e, &e->d_perm, NCLS * G)) || (rc = dalloc(e, &e->d_perm_cnt, NCLS))) { rafting_engine_destroy(e); return rc; }
    if (cudaMemcpy(e->d_cfg, &e->dcfg, sizeof(CfgD), cudaMemcpyHostToDevice) != cudaSuccess) {
        rafting_engine_destroy(e); return fail(RAFTING_E_CUDA, "cfg upload failed");
    }
    if (cudaStreamCreateWithFlags(&e->stream, cudaStreamNonBlocking) != cudaSuccess) {
        rafting_engine_destroy(e); return fail(RAFTING_E_CUDA, "cudaStreamCreate failed");
    }
    *out = e;
    return RAFTING_OK;
}

extern "C" int rafting_engine_destroy(rafting_engine_t* e) {
    if (!e) return RAFTING_OK;
    cudaSetDevice(e->cfg.device);
    if (e->stream) { cudaStreamSynchronize(e->stream); }
    if (e->s_comm) {
        cudaStreamSynchronize(e->s_comm); cudaStreamDestroy(e->s_comm); cudaEventDestroy(e->ev_step);
        for (int p = 0; p < 2; p++) if (e->ev_gather[p]) cudaEventDestroy(e->ev_gather[p]);
    }
    if (e->comm && g_nccl.CommDestroy) g_nccl.CommDestroy(e->comm);
    for (void* p : e->dev_allocs) cudaFree(p);
    for (void* p : e->shadow) if (p) cudaFree(p);
    compact_release(e);
    due_release(e);
    edit_release(e);
    rafting_hostpath_release(e);
    seglog_release(e);
    if (e->ev_seg) cudaEventDestroy(e->ev_seg);
    if (e->stream) cudaStreamDestroy(e->stream);
    delete e;
    return RAFTING_OK;
}

// One group's rows as an open writes them: g_meta, g_term, g_commit, g_lo, g_hi, g_timer, g_epoch and the g_runs planes (newest
// run first); g_elect, g_err and the l_* planes of its lanes are zero.  rafting_group_open_bulk copies them column by column,
// rafting_group_edit_begin ships them to group_edit_kernel as records, so the two paths compute them in one place.
struct EditRow { uint32_t gid, kind; uint64_t meta; int64_t term, commit, lo, hi, timer; i64x2 epoch; i64x2 runs[KRUNS]; };

// ContextManager.buildContext + RaftContext.initialize (RaftContext.java:91-113): the group starts
// as Follower(restore.term, restore.ballot) — first RaftMember construction (incarnation 1) — with
// an armed election timer: resetTimer with a null ticket gives max(0 + 1, now + timeout)
// (RaftRoutine.java:95-107).
static int open_row(const rafting_engine* e, uint32_t gid, const rafting_group_init_t& g, EditRow& r) {
    const bool has = g.last_index >= g.first_index;
    if (has && g.first_index != g.epoch_index && g.first_index != g.epoch_index + 1)
        return fail(RAFTING_E_INVAL, "group %u: first_index must be epoch_index or epoch_index+1", gid);
    if (g.ballot < -1 || g.ballot >= (int)e->cfg.replicas) return fail(RAFTING_E_INVAL, "group %u: bad ballot", gid);
    memset(&r, 0, sizeof(r));
    r.gid = gid; r.kind = RAFTING_EDIT_OPEN;
    const uint32_t word = RAFTING_ROLE_FOLLOWER | W_ALIVE | ((uint32_t)(g.ballot + 1) << W_BALLOT_SH) | ((has ? 1u : 0u) << W_NRUNS_SH);
    r.meta = (uint64_t)word | (1ull << 32);
    r.term = g.term; r.commit = g.commit_index;
    r.lo = has ? g.first_index : 1; r.hi = has ? g.last_index : 0;
    const int64_t draw = g.rand_ms != 0 ? g.rand_ms : rafting_draw(e->cfg.timer_seed, gid, 1, e->cfg.election_ms);
    const int64_t b = (INT64_MAX - draw < g.now_ms) ? INT64_MAX : g.now_ms + draw;
    r.timer = b > 1 ? b : 1;
    r.epoch.x = g.epoch_index; r.epoch.y = g.epoch_term;
    r.runs[0].x = has ? g.first_index : 0; r.runs[0].y = has ? g.last_term : 0;
    return RAFTING_OK;
}
// rafting_group_load_runs' checks of 1..KRUNS runs (oldest first) against a stored log [lo, hi] whose last term is last_term;
// out gets them newest first, as g_runs keeps them
static int runs_rows(int64_t lo, int64_t hi, int64_t last_term, const rafting_i64x2_t* runs, uint32_t n, i64x2* out) {
    if (runs[0].x != lo || runs[n - 1].y != last_term) return fail(RAFTING_E_INVAL, "runs do not match the opened log (first index / last term)");
    for (uint32_t k = 1; k < n; k++)
        if (runs[k].x <= runs[k - 1].x || runs[k].x > hi || runs[k].y == runs[k - 1].y) return fail(RAFTING_E_INVAL, "runs must start at increasing indices inside the log and change term");
    for (uint32_t k = 0; k < n; k++) { out[k].x = runs[n - 1 - k].x; out[k].y = runs[n - 1 - k].y; }
    return RAFTING_OK;
}
static uint64_t with_nruns(uint64_t m, uint32_t n) { return (m & ~((uint64_t)0xf << W_NRUNS_SH)) | ((uint64_t)n << W_NRUNS_SH); }

extern "C" int rafting_group_open_bulk(rafting_engine_t* e, uint32_t first, uint32_t count, const rafting_group_init_t* in) {
    if (!e || !in) return fail(RAFTING_E_INVAL, "null argument");
    if ((uint64_t)first + count > e->G) return fail(RAFTING_E_CAPACITY, "gid range beyond max_groups");
    if (count == 0) return RAFTING_OK;
    CU(cudaSetDevice(e->cfg.device));
    // e->stream is non-blocking: the legacy-stream copies below are NOT ordered against queued step kernels, and a dense
    // step loads and writes back the hot columns of every gid.  Opening is rare (ContextManager.buildContext is
    // synchronized): drain the step stream first, and refuse while a host-path step is still in flight.
    if (int rc = quiesce_for_table_edit(e, "rafting_group_open")) return rc;
    const size_t F = e->F;
    std::vector<uint64_t> meta(count); std::vector<int64_t> term(count), commit(count), lo(count), hi(count), timer(count);
    std::vector<i64x2> epoch(count), elect(count), run0(count); std::vector<uint32_t> err(count, 0);
    for (uint32_t k = 0; k < count; k++) {
        EditRow r;
        if (int rc = open_row(e, first + k, in[k], r)) return rc;
        meta[k] = r.meta; term[k] = r.term; commit[k] = r.commit; lo[k] = r.lo; hi[k] = r.hi; timer[k] = r.timer;
        epoch[k] = r.epoch; elect[k].x = 0; elect[k].y = 0; run0[k] = r.runs[0];
    }
    Tables& T = e->T;
    CU(cudaMemcpy(T.g_meta + first, meta.data(), count * 8, cudaMemcpyHostToDevice));
    CU(cudaMemcpy(T.g_term + first, term.data(), count * 8, cudaMemcpyHostToDevice));
    CU(cudaMemcpy(T.g_commit + first, commit.data(), count * 8, cudaMemcpyHostToDevice));
    CU(cudaMemcpy(T.g_lo + first, lo.data(), count * 8, cudaMemcpyHostToDevice));
    CU(cudaMemcpy(T.g_hi + first, hi.data(), count * 8, cudaMemcpyHostToDevice));
    CU(cudaMemcpy(T.g_timer + first, timer.data(), count * 8, cudaMemcpyHostToDevice));
    CU(cudaMemcpy(T.g_epoch + first, epoch.data(), count * 16, cudaMemcpyHostToDevice));
    CU(cudaMemcpy(T.g_elect + first, elect.data(), count * 16, cudaMemcpyHostToDevice));
    CU(cudaMemcpy(T.g_err + first, err.data(), count * 4, cudaMemcpyHostToDevice));
    CU(cudaMemcpy(T.g_runs + first, run0.data(), count * 16, cudaMemcpyHostToDevice));
    for (int k = 1; k < KRUNS; k++) CU(cudaMemset(T.g_runs + (size_t)k * e->G + first, 0, (size_t)count * 16));
    CU(cudaMemset(T.l_nm + (size_t)first * F, 0, (size_t)count * F * 16));
    CU(cudaMemset(T.l_es + (size_t)first * F, 0, (size_t)count * F * 16));
    CU(cudaMemset(T.l_fr + (size_t)first * F, 0, (size_t)count * F * 16));
    CU(cudaMemset(T.l_cnt + (size_t)first * F, 0, (size_t)count * F * 16));
    return RAFTING_OK;
}
extern "C" int rafting_group_open(rafting_engine_t* e, uint32_t gid, const rafting_group_init_t* init) {
    return rafting_group_open_bulk(e, gid, 1, init);
}
extern "C" int rafting_group_load_runs(rafting_engine_t* e, uint32_t gid, const rafting_i64x2_t* runs, uint32_t n) {
    if (!e || !runs || gid >= e->G) return fail(RAFTING_E_INVAL, "bad argument");
    if (n == 0 || n > (uint32_t)KRUNS) return fail(RAFTING_E_CAPACITY, "%u term runs: the engine keeps at most %d per group", n, KRUNS);
    CU(cudaSetDevice(e->cfg.device));
    CU(cudaStreamSynchronize(e->stream));
    uint64_t m; int64_t lo, hi; i64x2 newest;
    CU(cudaMemcpy(&m, e->T.g_meta + gid, 8, cudaMemcpyDeviceToHost));
    CU(cudaMemcpy(&lo, e->T.g_lo + gid, 8, cudaMemcpyDeviceToHost));
    CU(cudaMemcpy(&hi, e->T.g_hi + gid, 8, cudaMemcpyDeviceToHost));
    CU(cudaMemcpy(&newest, e->T.g_runs + gid, 16, cudaMemcpyDeviceToHost));
    if (!(m & W_ALIVE) || ((uint32_t)(m >> W_NRUNS_SH) & 0xf) != 1 || hi < lo) return fail(RAFTING_E_INVAL, "group %u is not a freshly opened group with a stored log", gid);
    i64x2 rows[KRUNS];
    if (int rc = runs_rows(lo, hi, newest.y, runs, n, rows)) return rc;
    for (uint32_t k = 0; k < n; k++) CU(cudaMemcpy(e->T.g_runs + (size_t)k * e->G + gid, &rows[k], 16, cudaMemcpyHostToDevice));   // newest run first in the table
    m = with_nruns(m, n);
    CU(cudaMemcpy(e->T.g_meta + gid, &m, 8, cudaMemcpyHostToDevice));
    return RAFTING_OK;
}
extern "C" int rafting_group_close(rafting_engine_t* e, uint32_t gid) {
    if (!e || gid >= e->G) return fail(RAFTING_E_INVAL, "bad gid");
    CU(cudaSetDevice(e->cfg.device));
    if (int rc = quiesce_for_table_edit(e, "rafting_group_close")) return rc;   // host read-modify-write of g_meta
    uint64_t m;
    CU(cudaMemcpy(&m, e->T.g_meta + gid, 8, cudaMemcpyDeviceToHost));
    m &= ~(uint64_t)W_ALIVE;
    CU(cudaMemcpy(e->T.g_meta + gid, &m, 8, cudaMemcpyHostToDevice));
    return RAFTING_OK;
}

// ---------------------------------------------------------------------------------------------
// kernel dispatch
// ---------------------------------------------------------------------------------------------
// follower-slot bound FT and staging depth NST per replica count: R=2 -> <1,3>, R=3 -> <2,3>,
// R<=5 -> <4,3>, R<=9 -> <8,2>, larger clusters keep their slots in local memory and read the inbox directly
template <int FT, int NST, bool FIX>
static int launch_t(rafting_engine* e, const InboxD& in, const OutboxD& out, cudaStream_t st) {
    const size_t smem = (size_t)NST * sizeof(Stage<FT>);
    static bool configured[64] = {false};
    if (smem > 0 && !configured[e->cfg.device & 63]) {
        CU(cudaFuncSetAttribute(unrolled::step_kernel<FT, NST, FIX>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        configured[e->cfg.device & 63] = true;
    }
    const uint32_t blocks = (in.n + TPB - 1) / TPB + (in.perm ? (uint32_t)NCLS : 0u);   // + NCLS: every class is padded to a block
    if (in.n == 0) return RAFTING_OK;
    unrolled::step_kernel<FT, NST, FIX><<<blocks, TPB, smem, st>>>(e->T, in, out, e->d_cfg, e->dcfg);
    return RAFTING_OK;
}
// R = 3, a step launched without a class sort (the leader stream): one thread per (group, follower) (pair_kernel.cuh, v7),
// which measured faster than the thread-per-group kernel (v6) on an H100 (DESIGN.md §5)
static int launch_pair(rafting_engine* e, const InboxD& in0, const OutboxD& out, cudaStream_t st) {
    constexpr int NSTP = 3;
    const size_t smem = (size_t)NSTP * sizeof(pair::PStage);
    static bool configured[64] = {false};
    if (!configured[e->cfg.device & 63]) {
        CU(cudaFuncSetAttribute(pair::pair_kernel<NSTP>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        configured[e->cfg.device & 63] = true;
    }
    if (in0.perm) return fail(RAFTING_E_INVAL, "launch_pair: pair_kernel takes only steps launched without a class sort");
    if (in0.n == 0) return RAFTING_OK;
    const uint32_t blocks = (in0.n + TPB - 1) / TPB;
    // Directly behind the previous step's kernel, the launch is programmatic (Hopper PDL): its blocks take the SMs the
    // previous launch's blocks free, and stage their first inbox rows while its last blocks finish; griddepcontrol.wait
    // holds every table / outbox access until the previous grid has completed and its writes are visible.
    cudaLaunchConfig_t lc = {};
    lc.gridDim = dim3(blocks); lc.blockDim = dim3(pair::PTPB); lc.dynamicSmemBytes = smem; lc.stream = st;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization; at[0].val.programmaticStreamSerializationAllowed = 1;
    lc.attrs = at; lc.numAttrs = e->follows_step ? 1u : 0u;
    CU(cudaLaunchKernelEx(&lc, pair::pair_kernel<NSTP>, e->T, in0, out, (const CfgD*)e->d_cfg, e->dcfg));
    return RAFTING_OK;
}
template <bool FIX>
static int launch_looped(rafting_engine* e, const InboxD& in, const OutboxD& out, cudaStream_t st) {
    const uint32_t blocks = (in.n + TPB - 1) / TPB;
    if (blocks == 0) return RAFTING_OK;
    looped::step_kernel<32, 0, FIX><<<blocks, TPB, 0, st>>>(e->T, in, out, e->d_cfg, e->dcfg);
    return RAFTING_OK;
}
// FIX: the kernels run with the opt-in protocol fixes compiled in (handlers.cuh).  Only the handlers of inbound requests
// differ between the instantiations, so a step that carries none computes the same on both.
template <bool FIX>
static int launch_step_t(rafting_engine* e, const InboxD& in0, const OutboxD& out, cudaStream_t st) {
    int rc;
    const uint32_t F = e->F;
    InboxD in = in0; in.perm = nullptr; in.perm_cnt = nullptr;
    // A step that may hold inbound requests mixes steady-state leaders with groups that need the generic handlers;
    // one slow lane stalls its whole warp, so such steps are launched class-sorted (DESIGN.md §5)
    if (!(in.flags & RAFTING_INBOX_NO_REQUESTS) && in.op_meta && in.n >= 2048 && F <= 8) {
        CU(cudaMemsetAsync(e->d_perm_cnt, 0, NCLS * 4, st));
        classify_kernel<<<(in.n + 255) / 256, 256, 0, st>>>(e->T, in, e->d_perm, e->d_perm_cnt);
        in.perm = e->d_perm; in.perm_cnt = e->d_perm_cnt;
    }
    // at F = 2..4 the slow classes run in a kernel of their own, with their own register cap
    if (in.perm && F >= 2 && F <= 4) {
        const uint32_t sb = (in.n + unrolled::SLOW_TPB - 1) / unrolled::SLOW_TPB + (uint32_t)NCLS;
        if (F == 2) unrolled::slow_kernel<2, 4, FIX><<<sb, unrolled::SLOW_TPB, 0, st>>>(e->T, in, out, e->d_cfg);
        else unrolled::slow_kernel<4, 4, FIX><<<sb, unrolled::SLOW_TPB, 0, st>>>(e->T, in, out, e->d_cfg);
        in.flags |= INBOX_INTERNAL_SLOW_ELSEWHERE;
    }
    if (F == 1) rc = launch_t<1, 3, FIX>(e, in, out, st);
#ifndef RAFTING_NST2
#define RAFTING_NST2 3
#endif
    else if (F == 2) {
        // v7 (pair_kernel.cuh) measured faster than v6 on the leader stream on an H100 and slower on class-sorted steps
        // (config #5), same-call A/Bs (DESIGN.md §5): it runs the steps launched without a class sort.  pair_kernel has no
        // FIX instantiation: with flags it takes only the steps that promise no inbound request, and the others run unsorted
        // in the FIX step kernel
        const bool pair = !in.perm && (!FIX || (in.flags & RAFTING_INBOX_NO_REQUESTS));
        rc = pair ? launch_pair(e, in, out, st) : launch_t<2, RAFTING_NST2, FIX>(e, in, out, st);
    }
    else if (F <= 4) rc = launch_t<4, 3, FIX>(e, in, out, st);
    else if (F <= 8) rc = launch_t<8, 2, FIX>(e, in, out, st);
    else rc = launch_looped<FIX>(e, in, out, st);
    if (rc) return rc;
    e->launches++;
    CU(cudaGetLastError());
    return RAFTING_OK;
}
// Every step entry point (host, lease and leased steps, every compact begin, rafting_step_device and _seq) reaches the step
// kernels here: the one place that picks the instantiation for the engine's cfg.flags
static int launch_step(rafting_engine* e, const InboxD& in0, const OutboxD& out, cudaStream_t st) {
    if ((uint64_t)in0.rows * in0.n * e->F >= (1ull << 32)) return fail(RAFTING_E_CAPACITY, "rows * groups * followers must stay below 2^32 per step");
    return e->cfg.flags != 0 ? launch_step_t<true>(e, in0, out, st) : launch_step_t<false>(e, in0, out, st);
}

static void to_dev_views(const rafting_inbox_t* in, const rafting_outbox_t* out, uint32_t G, uint32_t* flags, InboxD& di, OutboxD& dout) {
    di.rows = in->rows; di.n = in->gids ? in->n_active : G; di.gids = in->gids; di.row_now = in->row_now;
    di.op_meta = in->op_meta; di.op_nr = (const i64x2*)in->op_nr; di.op_ab = (const i64x2*)in->op_ab;
    di.op_cd = (const i64x2*)in->op_cd; di.op_e = in->op_e; di.ent_terms = in->ent_terms; di.ent_count = in->ent_count; di.flags = in->flags;
    di.ev_meta = in->ev_meta; di.ev_tn = (const i64x2*)in->ev_tn; di.ev_el = (const i64x2*)in->ev_el;
    dout.rep_meta = out->rep_meta; dout.rep_term = out->rep_term; dout.plan_meta = out->plan_meta;
    dout.plan_pp = (i64x2*)out->plan_pp; dout.plan_lc = (i64x2*)out->plan_lc; dout.plan_epoch = out->plan_epoch;
    dout.ballot_meta = out->ballot_meta; dout.ballot_term = out->ballot_term; dout.ballot_last = (i64x2*)out->ballot_last;
    dout.commit_index = out->commit_index; dout.current_term = out->current_term; dout.role_word = out->role_word;
    dout.incarnation = out->incarnation; dout.err_word = out->err_word; dout.last_entry = (i64x2*)out->last_entry; dout.flags = flags;
}

extern "C" int rafting_step_device(rafting_engine_t* e, const rafting_inbox_t* in, const rafting_outbox_t* out, void* stream) {
    if (!e || !in || !out) return fail(RAFTING_E_INVAL, "null argument");
    if (in->gids && in->n_active > e->G) return fail(RAFTING_E_CAPACITY, "n_active > max_groups");
    CU(cudaSetDevice(e->cfg.device));
    InboxD di; OutboxD dout;
    to_dev_views(in, out, e->G, nullptr, di, dout);
    return launch_step(e, di, dout, stream ? (cudaStream_t)stream : e->stream);
}

extern "C" int rafting_allgather_commit_from(rafting_engine_t* e, const int64_t* dev_src, int64_t* host_out, void** dev_out);
extern "C" int rafting_step_device_seq(rafting_engine_t* e, const rafting_inbox_t* ins, const rafting_outbox_t* outs, uint32_t n,
                                       int gather, void* stream) {
    if (!e || !ins || !outs) return fail(RAFTING_E_INVAL, "null argument");
    if (gather && stream && (cudaStream_t)stream != e->stream) return fail(RAFTING_E_INVAL, "gathers follow the engine's own stream");
    if (gather && !e->gather[0]) return fail(RAFTING_E_NCCL, "communicator not initialised (rafting_comm_init)");
    // every launch is checked before any is enqueued: a refused call leaves the stream, the tables and the outboxes alone
    for (uint32_t k = 0; k < n; k++) {
        const rafting_inbox_t& in = ins[k];
        if (in.gids && in.n_active > e->G) return fail(RAFTING_E_CAPACITY, "launch %u: n_active > max_groups", k);
        if ((uint64_t)in.rows * (in.gids ? in.n_active : e->G) * e->F >= (1ull << 32))
            return fail(RAFTING_E_CAPACITY, "launch %u: rows * groups * followers must stay below 2^32 per step", k);
        // a gather copies max_groups entries of the launch's commit column: only a whole-shard launch writes all of them
        if (gather && in.gids) return fail(RAFTING_E_INVAL, "launch %u: a gathering sequence takes whole-shard launches only", k);
    }
    for (uint32_t k = 0; k < n; k++) {
        // without gathers, launch k's only predecessor on the stream is launch k-1's step kernel: none of them writes an inbox
        e->follows_step = k > 0 && !gather;
        int rc = rafting_step_device(e, &ins[k], &outs[k], stream);
        e->follows_step = false;
        if (rc) return rc;
        if (gather) { rc = rafting_allgather_commit_from(e, outs[k].commit_index, nullptr, nullptr); if (rc) return rc; }
    }
    return RAFTING_OK;
}

// ---------------------------------------------------------------------------------------------
// host path.  Two SLOTS, each with its own device staging (and, for leases, engine-owned pinned
// buffers), and three streams: H2D copies, the step kernel, D2H copies.  A step in slot s is
//   s_h2d: inbox columns -> device staging          (event h2d[s])
//   stream: wait h2d[s]; step kernel                (event kernel[s])
//   s_d2h: wait kernel[s]; outbox columns -> host   (event done[s])
// so while slot A's kernel runs, slot B's inputs travel up and the previous outbox travels down (PCIe
// is full duplex).  Kernels of successive steps stay ordered on `stream`: that is the serial order.
// ---------------------------------------------------------------------------------------------
enum { PER_GI = 0, PER_LI = 1, PER_ACTIVE = 2, PER_ROW = 3, PER_ENT = 4, PER_G = 5 };
struct ColDesc { size_t off; uint32_t elem; int per; };
#define INCOL(f, elem, per) {offsetof(rafting_inbox_t, f), elem, per}
#define OUTCOL(f, elem, per) {offsetof(rafting_outbox_t, f), elem, per}
static const ColDesc IN_COLS[] = {
    INCOL(gids, 4, PER_ACTIVE), INCOL(row_now, 8, PER_ROW), INCOL(op_meta, 8, PER_GI), INCOL(op_nr, 16, PER_GI),
    INCOL(op_ab, 16, PER_GI), INCOL(op_cd, 16, PER_GI), INCOL(op_e, 8, PER_GI), INCOL(ent_terms, 8, PER_ENT),
    INCOL(ev_meta, 8, PER_LI), INCOL(ev_tn, 16, PER_LI), INCOL(ev_el, 16, PER_LI)};
static const ColDesc OUT_COLS[] = {
    OUTCOL(rep_meta, 4, PER_GI), OUTCOL(rep_term, 8, PER_GI), OUTCOL(plan_meta, 8, PER_LI), OUTCOL(plan_pp, 16, PER_LI),
    OUTCOL(plan_lc, 16, PER_LI), OUTCOL(plan_epoch, 8, PER_LI), OUTCOL(ballot_meta, 8, PER_GI), OUTCOL(ballot_term, 8, PER_GI),
    OUTCOL(ballot_last, 16, PER_GI), OUTCOL(commit_index, 8, PER_G), OUTCOL(current_term, 8, PER_G), OUTCOL(role_word, 4, PER_G),
    OUTCOL(incarnation, 4, PER_G), OUTCOL(err_word, 4, PER_G), OUTCOL(last_entry, 16, PER_G)};
constexpr int N_IN = sizeof(IN_COLS) / sizeof(IN_COLS[0]), N_OUT = sizeof(OUT_COLS) / sizeof(OUT_COLS[0]);

static size_t col_bytes(const ColDesc& c, size_t rows, size_t n, size_t F, size_t G, size_t nact, size_t ent) {
    switch (c.per) {
        case PER_GI: return rows * n * c.elem;
        case PER_LI: return rows * n * F * c.elem;
        case PER_ACTIVE: return nact * c.elem;
        case PER_ROW: return rows * c.elem;
        case PER_ENT: return ent * c.elem;
        default: return G * c.elem;
    }
}
template <typename S> static const void*& in_ptr(S* st, const ColDesc& c) { return *(const void**)((char*)st + c.off); }
template <typename S> static void*& out_ptr(S* st, const ColDesc& c) { return *(void**)((char*)st + c.off); }

// Staging layout of one step: every column gets a 256-byte aligned offset inside ONE block, in an order that
// keeps what a typical step carries adjacent (op + event families first; dense outbox columns before the
// sparse payload columns).  The device block and — for leases — the pinned host block use the same offsets,
// so adjacent columns travel in a single cudaMemcpyAsync (a leased leader step is 1 copy up, 1 copy down).
static const int IN_ORDER[N_IN]   = {2, 3, 8, 9, 10, 4, 5, 6, 7, 0, 1};     // op_meta op_nr ev_meta ev_tn ev_el op_ab op_cd op_e ent gids row_now
static const int OUT_ORDER[N_OUT] = {0, 2, 3, 4, 5, 6, 9, 10, 11, 12, 13, 14, 1, 7, 8};   // ... dense ..., then rep_term ballot_term ballot_last
// carves one block into 256-byte aligned parts: take(bytes) returns the next part's offset, o is where the block ends so far
struct Carve { size_t o = 0; size_t take(size_t bytes) { const size_t at = o; o += (bytes + 255) & ~(size_t)255; return at; } };
struct Layout { size_t in_off[N_IN], out_off[N_OUT], flags_off, in_total, out_total; };
// gcols = entries of a per-group outbox column: max_groups, or n under RAFTING_INBOX_COMPACT_GROUPS
static Layout make_layout(size_t rows, size_t n, size_t F, size_t gcols, size_t nact, size_t ent) {
    const size_t G = gcols;
    Layout L; Carve in, out;
    for (int q = 0; q < N_IN; q++) { const int k = IN_ORDER[q]; L.in_off[k] = in.take(col_bytes(IN_COLS[k], rows, n, F, G, nact, ent + 1)); }
    L.in_total = in.o;
    for (int q = 0; q < N_OUT; q++) {
        const int k = OUT_ORDER[q];
        if (q == N_OUT - 3) L.flags_off = out.take(16);                    // the two flag words sit right after the dense columns
        L.out_off[k] = out.take(col_bytes(OUT_COLS[k], rows, n, F, G, 0, 0));
    }
    L.out_total = out.o;
    return L;
}
// Device staging views of one step in the blocks carved by make_layout.  The inbox view has every column at its offset; the
// caller nulls the ones its step does not carry.  The outbox view has the columns `want` has (every one when want is null),
// except that without an op or a sweep row nothing can produce replies or plans, so those columns stay null.
static rafting_inbox_t stage_inbox(const Layout& L, uint8_t* blk) {
    rafting_inbox_t v; memset(&v, 0, sizeof(v));
    for (int k = 0; k < N_IN; k++) in_ptr(&v, IN_COLS[k]) = blk + L.in_off[k];
    return v;
}
static rafting_outbox_t stage_outbox(const Layout& L, uint8_t* blk, const rafting_outbox_t* want, bool ops) {
    rafting_outbox_t v; memset(&v, 0, sizeof(v));
    for (int k = 0; k < N_OUT; k++) {
        const ColDesc& c = OUT_COLS[k];
        const bool repOrPlan = c.off <= offsetof(rafting_outbox_t, plan_epoch);
        if ((!want || out_ptr(want, c)) && (ops || !repOrPlan)) out_ptr(&v, c) = blk + L.out_off[k];
    }
    return v;
}
struct Blk { uint8_t* p = nullptr; size_t cap = 0; };
static void blk_free(Blk& b, bool pinned) { if (b.p) { if (pinned) cudaFreeHost(b.p); else cudaFree(b.p); b.p = nullptr; b.cap = 0; } }
static int blk_reserve(Blk& b, size_t bytes, bool pinned) {
    if (bytes <= b.cap) return 0;
    blk_free(b, pinned);
    const size_t cap = bytes + bytes / 4 + 4096;
    if (pinned) { CU(cudaHostAlloc((void**)&b.p, cap, cudaHostAllocDefault)); memset(b.p, 0, cap); }
    else { CU(cudaMalloc((void**)&b.p, cap)); CU(cudaMemset(b.p, 0, cap)); }   // column padding and never-written plan fields travel in the one-block D2H copy: defined bytes
    if (!pinned) CU(cudaStreamSynchronize(0));        // that memset runs on the legacy stream, which the engine's non-blocking streams do not wait for
    b.cap = cap;
    return 0;
}

struct Slot {
    Blk din, dout;                            // device staging (both paths)
    Blk cin, cout, chin, chout;               // compact path: device wire blocks + pinned landing block of the small items
    Blk creq, creqw;                          // compact path: request list + entry pool, and its scan scratch
    bool compact_step = false;                // the step in flight came through one of the rafting_step_begin_compact* calls
    rafting_coutbox_t c_host; uint32_t* c_counts_pinned = nullptr; void* c_esc_dev = nullptr;
    Blk ctail;                                // rafting_step_begin_compact_due: the tail selection's scratch, due_layout (timers.cuh)
    uint32_t* c_tail_user = nullptr; uint32_t c_tail_n = 0;   // where the wait copies the tail (landed at chout + 256)
    Blk hin, hout;                            // pinned host staging (leases only), same layout as din / dout
    uint32_t* h_flags = nullptr;              // pinned landing place of the flag words on the caller-owned path
    cudaEvent_t ev_h2d = nullptr, ev_kernel = nullptr, ev_done = nullptr;
    bool leased = false, inflight = false;
    uint32_t rows = 0, n = 0, ent = 0; bool list = false, compact = false;
    void* lease_key = nullptr;                // the lease's commit_index pointer + its generation identify it
    uint32_t lease_gen = 0;
    // of the step in flight (for the sparse columns fetched at wait time)
    rafting_outbox_t host_out; rafting_outbox_t dev_out; size_t rows_ = 0, n_ = 0; const uint32_t* flags_host = nullptr;
    const uint32_t* c_gids = nullptr;         // device list of the compact step (null: whole shard), due tail included
    struct StepGather* gather = nullptr;      // rafting_log_gather_step_begin (seglog.cuh), created on first use
    bool gathering = false;                   // a gather of this slot's plans has not been waited for: no step may reuse the slot
};
struct HostPath {
    Slot slot[RAFTING_HOST_SLOTS];
    cudaStream_t s_h2d = nullptr, s_d2h = nullptr;
    bool ready = false;
};
static HostPath* hp(rafting_engine* e) { if (!e->host) e->host = new HostPath(); return e->host; }
static void step_gather_release(Slot& s);

// Host-side edits of the tables (group open / close / load_runs) must not interleave with step kernels: RAFTING_E_BUSY
// while a host-path step has been begun and not waited for, then the step stream is drained.
static int quiesce_for_table_edit(rafting_engine* e, const char* who) {
    if (e->host)
        for (int k = 0; k < RAFTING_HOST_SLOTS; k++)
            if (e->host->slot[k].inflight) return fail(RAFTING_E_BUSY, "%s: slot %d has a step in flight (wait for it first)", who, k);
    CU(cudaStreamSynchronize(e->stream));
    return RAFTING_OK;
}

static int hostpath_init(rafting_engine* e) {
    HostPath* H = hp(e);
    if (H->ready) return 0;
    CU(cudaStreamCreateWithFlags(&H->s_h2d, cudaStreamNonBlocking));
    CU(cudaStreamCreateWithFlags(&H->s_d2h, cudaStreamNonBlocking));
    for (Slot& s : H->slot) {
        CU(cudaEventCreateWithFlags(&s.ev_h2d, cudaEventDisableTiming));
        CU(cudaEventCreateWithFlags(&s.ev_kernel, cudaEventDisableTiming));
        CU(cudaEventCreateWithFlags(&s.ev_done, cudaEventDisableTiming));
        CU(cudaHostAlloc((void**)&s.h_flags, 16, cudaHostAllocDefault));
    }
    H->ready = true;
    return 0;
}
static void hostpath_free(rafting_engine* e) {
    HostPath* H = hp(e);
    for (Slot& s : H->slot) {
        for (Blk* b : {&s.din, &s.dout, &s.cin, &s.cout, &s.creq, &s.creqw, &s.ctail}) blk_free(*b, false);
        for (Blk* b : {&s.hin, &s.hout, &s.chin, &s.chout}) blk_free(*b, true);
        if (s.ev_h2d) cudaEventDestroy(s.ev_h2d);
        if (s.ev_kernel) cudaEventDestroy(s.ev_kernel);
        if (s.ev_done) cudaEventDestroy(s.ev_done);
        if (s.h_flags) cudaFreeHost(s.h_flags);
        step_gather_release(s);
    }
    if (H->s_h2d) cudaStreamDestroy(H->s_h2d);
    if (H->s_d2h) cudaStreamDestroy(H->s_d2h);
}
static void rafting_hostpath_release(rafting_engine* e) { if (e->host) { hostpath_free(e); delete e->host; e->host = nullptr; } }

// copy list with merging: entries of the engine's own pinned block `hb` (a lease) whose host and device addresses
// advance by the same amount, with at most one alignment gap between them, become one cudaMemcpyAsync.  Caller-owned
// buffers are never merged: two of them may be adjacent in the address space and still be separate registrations.
struct CopyItem { uint8_t* h; uint8_t* d; size_t bytes; };
static int issue_copies(std::vector<CopyItem>& v, bool to_device, cudaStream_t st, const Blk& hb) {
    auto own = [&](const CopyItem& c) { return hb.p && c.h >= hb.p && c.h + c.bytes <= hb.p + hb.cap; };
    size_t i = 0;
    while (i < v.size()) {
        uint8_t* h0 = v[i].h; uint8_t* d0 = v[i].d; size_t len = v[i].bytes; size_t j = i + 1;
        while (own(v[i]) && j < v.size() && own(v[j]) && v[j].h - h0 == v[j].d - d0 && v[j].h >= h0 + len && (size_t)(v[j].h - (h0 + len)) < 256) {
            len = (size_t)(v[j].h - h0) + v[j].bytes; j++;
        }
        if (to_device) CU(cudaMemcpyAsync(d0, h0, len, cudaMemcpyHostToDevice, st));
        else CU(cudaMemcpyAsync(h0, d0, len, cudaMemcpyDeviceToHost, st));
        i = j;
    }
    return RAFTING_OK;
}

// enqueue one step in `slot`: `in` / `out` hold HOST pointers (pinned for real overlap)
static int step_enqueue(rafting_engine* e, uint32_t slot, const rafting_inbox_t* in, const rafting_outbox_t* out) {
    HostPath* H = hp(e); Slot& S = H->slot[slot];
    if (S.inflight) return fail(RAFTING_E_BUSY, "slot %u has a step in flight", slot);
    if (S.gathering) return fail(RAFTING_E_BUSY, "slot %u: the gather of its plans has not been waited for", slot);
    const size_t rows = in->rows, F = e->F, G = e->G;
    const bool list = in->gids != nullptr;
    const size_t n = list ? in->n_active : G;
    if (rows == 0 || rows > e->cfg.max_rows) return fail(RAFTING_E_CAPACITY, "rows %zu beyond max_rows %u", rows, e->cfg.max_rows);
    if (n > G) return fail(RAFTING_E_CAPACITY, "n_active > max_groups");
    if (in->ent_count > e->cfg.entry_pool_cap) return fail(RAFTING_E_CAPACITY, "ent_count > entry_pool_cap");
    bool sweep = false;
    if (in->row_now) for (size_t r = 0; r < rows; r++) sweep |= in->row_now[r] != 0;
    if (in->op_meta && !in->op_nr) return fail(RAFTING_E_INVAL, "op_meta without op_nr");
    if (in->ev_meta && !in->ev_tn) return fail(RAFTING_E_INVAL, "ev_meta without ev_tn");
    // a leased step keeps the layout of its lease (the pinned block was carved with it)
    const bool compact = list && (in->flags & RAFTING_INBOX_COMPACT_GROUPS);
    if (S.leased && compact != S.compact) return fail(RAFTING_E_INVAL, "COMPACT_GROUPS differs from the lease");
    const size_t gcols = compact ? n : G;
    const Layout L = S.leased ? make_layout(S.rows, S.n, F, S.compact ? S.n : G, S.list ? S.n : 0, S.ent)
                              : make_layout(rows, n, F, gcols, in->n_active, in->ent_count);
    int rc;
    if ((rc = blk_reserve(S.din, L.in_total, false)) || (rc = blk_reserve(S.dout, L.out_total, false))) return rc;
    rafting_inbox_t din = *in;
    // ---- H2D ----
    std::vector<CopyItem> up;
    for (int q = 0; q < N_IN; q++) {
        const int k = IN_ORDER[q]; const ColDesc& c = IN_COLS[k];
        const void* hsrc = in_ptr(in, c);
        bool use = hsrc != nullptr;
        if (c.per == PER_GI && !in->op_meta) use = false;                    // op family absent
        if (c.per == PER_LI && !in->ev_meta) use = false;                    // event family absent
        if (c.per == PER_ROW && !sweep) use = false;
        if (c.per == PER_ENT && (in->ent_count == 0 || !in->op_meta)) use = false;
        const size_t bytes = use ? col_bytes(c, rows, n, F, G, in->n_active, in->ent_count) : 0;
        if (!use || bytes == 0) { in_ptr(&din, c) = nullptr; continue; }
        CopyItem it; it.h = (uint8_t*)hsrc; it.d = S.din.p + L.in_off[k]; it.bytes = bytes;
        up.push_back(it);
        in_ptr(&din, c) = it.d;
    }
    if ((rc = issue_copies(up, true, H->s_h2d, S.hin))) return rc;
    CU(cudaEventRecord(S.ev_h2d, H->s_h2d));
    // ---- kernel ----
    rafting_outbox_t dout = stage_outbox(L, S.dout.p, out, din.op_meta || din.row_now);
    uint32_t* d_flags = (uint32_t*)(S.dout.p + L.flags_off);
    CU(cudaStreamWaitEvent(e->stream, S.ev_h2d, 0));
    CU(cudaMemsetAsync(d_flags, 0, 16, e->stream));
    InboxD di; OutboxD dov;
    to_dev_views(&din, &dout, e->G, d_flags, di, dov);
    rc = launch_step(e, di, dov, e->stream);
    if (rc) { cudaStreamSynchronize(H->s_h2d); return rc; }                  // no copy of this step may outlive the failed call
    CU(cudaEventRecord(S.ev_kernel, e->stream));
    // ---- D2H: dense columns always; the payload of the SPARSE families (rep_term, ballot_term, ballot_last —
    //      meaningful only where a reply / ballot exists, i.e. never in leader steady state) only if the kernel
    //      counted any, which the host learns from two flag words at wait time ----
    CU(cudaStreamWaitEvent(H->s_d2h, S.ev_kernel, 0));
    std::vector<CopyItem> down;
    for (int q = 0; q < N_OUT - 3; q++) {
        const int k = OUT_ORDER[q]; const ColDesc& c = OUT_COLS[k];
        uint8_t* dsrc = (uint8_t*)out_ptr(&dout, c);
        if (!dsrc) continue;
        CopyItem it; it.h = (uint8_t*)out_ptr(out, c); it.d = dsrc; it.bytes = col_bytes(c, rows, n, F, gcols, 0, 0);
        down.push_back(it);
    }
    // flag words: into the lease's own pinned block when the outbox is leased (merges with the columns), else aside
    uint32_t* hf = S.h_flags;
    if (S.leased && S.hout.p && out->commit_index == (int64_t*)(S.hout.p + L.out_off[9])) hf = (uint32_t*)(S.hout.p + L.flags_off);
    { CopyItem it; it.h = (uint8_t*)hf; it.d = (uint8_t*)d_flags; it.bytes = 16; down.push_back(it); }
    if ((rc = issue_copies(down, false, H->s_d2h, S.hout))) return rc;
    CU(cudaEventRecord(S.ev_done, H->s_d2h));
    S.host_out = *out; S.dev_out = dout; S.rows_ = rows; S.n_ = n; S.flags_host = hf;
    S.compact_step = false;
    S.inflight = true;
    return RAFTING_OK;
}
static int slot_wait(rafting_engine* e, uint32_t slot) {
    HostPath* H = hp(e); Slot& S = H->slot[slot];
    if (!S.inflight) return RAFTING_OK;
    if (S.compact_step) return fail(RAFTING_E_INVAL, "slot %u holds a compact step (use rafting_step_wait_compact)", slot);
    CU(cudaEventSynchronize(S.ev_done));
    S.inflight = false;
    // sparse families: fetch their payload columns only when the step produced ballots / valid replies
    const size_t gi_cnt = S.rows_ * S.n_;
    const uint32_t f0 = S.flags_host[0], f1 = S.flags_host[1];
    if (f0) {
        if (S.dev_out.ballot_term) CU(cudaMemcpyAsync(S.host_out.ballot_term, S.dev_out.ballot_term, gi_cnt * 8, cudaMemcpyDeviceToHost, H->s_d2h));
        if (S.dev_out.ballot_last) CU(cudaMemcpyAsync(S.host_out.ballot_last, S.dev_out.ballot_last, gi_cnt * 16, cudaMemcpyDeviceToHost, H->s_d2h));
    }
    if (f1 && S.dev_out.rep_term)
        CU(cudaMemcpyAsync(S.host_out.rep_term, S.dev_out.rep_term, gi_cnt * 8, cudaMemcpyDeviceToHost, H->s_d2h));
    if (f0 || f1) CU(cudaStreamSynchronize(H->s_d2h));
    return RAFTING_OK;
}

extern "C" int rafting_step_begin_host(rafting_engine_t* e, uint32_t slot, const rafting_inbox_t* in_host, const rafting_outbox_t* out_host) {
    if (!e || !in_host || !out_host || slot >= RAFTING_HOST_SLOTS) return fail(RAFTING_E_INVAL, "bad argument");
    CU(cudaSetDevice(e->cfg.device));
    int rc = hostpath_init(e); if (rc) return rc;
    if (hp(e)->slot[slot].leased) return fail(RAFTING_E_BUSY, "slot %u is held by an outstanding lease", slot);
    return step_enqueue(e, slot, in_host, out_host);
}
extern "C" int rafting_step_wait_slot(rafting_engine_t* e, uint32_t slot) {
    if (!e || slot >= RAFTING_HOST_SLOTS) return fail(RAFTING_E_INVAL, "bad argument");
    CU(cudaSetDevice(e->cfg.device));
    return slot_wait(e, slot);
}

// lease = engine-owned pinned columns of a free slot, carved from one pinned block with the staging layout
extern "C" int rafting_lease_ex(rafting_engine_t* e, uint32_t rows, uint32_t n_active, uint32_t ent_count, uint32_t flags, rafting_lease_t* out) {
    if (!e || !out) return fail(RAFTING_E_INVAL, "null argument");
    const bool compact = (flags & RAFTING_INBOX_COMPACT_GROUPS) != 0;
    if (compact && n_active == 0) return fail(RAFTING_E_INVAL, "COMPACT_GROUPS needs an active list");
    if (rows == 0 || rows > e->cfg.max_rows) return fail(RAFTING_E_CAPACITY, "rows %u > max_rows %u", rows, e->cfg.max_rows);
    if (n_active > e->G) return fail(RAFTING_E_CAPACITY, "n_active > max_groups");
    if (ent_count > e->cfg.entry_pool_cap) return fail(RAFTING_E_CAPACITY, "ent_count > entry_pool_cap");
    CU(cudaSetDevice(e->cfg.device));
    int rc = hostpath_init(e); if (rc) return rc;
    HostPath* H = hp(e);
    int sl = -1;
    for (int k = 0; k < RAFTING_HOST_SLOTS; k++) if (!H->slot[k].leased && !H->slot[k].inflight) { sl = k; break; }
    if (sl < 0) return fail(RAFTING_E_BUSY, "every slot is leased or in flight");
    Slot& S = H->slot[sl];
    const size_t n = n_active ? n_active : e->G, F = e->F, G = e->G;
    const Layout L = make_layout(rows, n, F, compact ? n : G, n_active, ent_count);
    if ((rc = blk_reserve(S.hin, L.in_total, true)) || (rc = blk_reserve(S.hout, L.out_total, true))) return rc;
    memset(out, 0, sizeof(*out));
    out->in = stage_inbox(L, S.hin.p);
    if (n_active == 0) out->in.gids = nullptr;
    memset((void*)out->in.row_now, 0, (size_t)rows * 8);                   // row_now: no sweep unless the caller sets it
    out->out = stage_outbox(L, S.hout.p, nullptr, true);
    out->in.rows = rows; out->in.n_active = n_active; out->in.ent_count = ent_count; out->in.flags = flags;
    S.compact = compact;
    S.leased = true; S.rows = rows; S.n = (uint32_t)n; S.ent = ent_count; S.list = n_active != 0;
    S.lease_key = out->out.commit_index;
    S.lease_gen = ++e->lease_counter; if (S.lease_gen == 0) S.lease_gen = ++e->lease_counter;
    out->generation = S.lease_gen;
    return RAFTING_OK;
}
extern "C" int rafting_lease(rafting_engine_t* e, uint32_t rows, uint32_t n_active, uint32_t ent_count, rafting_lease_t* out) {
    return rafting_lease_ex(e, rows, n_active, ent_count, 0, out);
}
static int lease_slot(rafting_engine* e, const rafting_lease_t* L) {
    HostPath* H = hp(e);
    for (int k = 0; k < RAFTING_HOST_SLOTS; k++)
        if (H->slot[k].leased && L->out.commit_index == (int64_t*)H->slot[k].lease_key && L->generation == H->slot[k].lease_gen) return k;
    return -1;
}
// give back a lease that will not be stepped (or whose step has been waited for already: then it is a no-op error)
extern "C" int rafting_lease_release(rafting_engine_t* e, rafting_lease_t* L) {
    if (!e || !L) return fail(RAFTING_E_INVAL, "null argument");
    if (!e->host) return fail(RAFTING_E_INVAL, "not an outstanding lease");
    CU(cudaSetDevice(e->cfg.device));
    const int sl = lease_slot(e, L);
    if (sl < 0) return fail(RAFTING_E_INVAL, "not an outstanding lease");
    Slot& S = hp(e)->slot[sl];
    if (S.inflight) { int rc = slot_wait(e, (uint32_t)sl); if (rc) return rc; }   // begun but never waited for: finish it
    S.leased = false; S.lease_key = nullptr; L->generation = 0;
    return RAFTING_OK;
}
extern "C" int rafting_step_begin(rafting_engine_t* e, rafting_lease_t* L) {
    if (!e || !L) return fail(RAFTING_E_INVAL, "null argument");
    CU(cudaSetDevice(e->cfg.device));
    const int sl = lease_slot(e, L);
    if (sl < 0) return fail(RAFTING_E_INVAL, "not an outstanding lease");
    Slot& S = hp(e)->slot[sl];
    if (L->in.rows == 0 || L->in.rows > S.rows) return fail(RAFTING_E_CAPACITY, "rows beyond the lease");
    if (L->in.ent_count > S.ent) return fail(RAFTING_E_CAPACITY, "ent_count beyond the lease");
    if (S.list != (L->in.gids != nullptr)) return fail(RAFTING_E_INVAL, "active-list lease without gids (or the reverse)");
    if (S.list && L->in.n_active > S.n) return fail(RAFTING_E_CAPACITY, "n_active beyond the lease");
    return step_enqueue(e, (uint32_t)sl, &L->in, &L->out);
}
extern "C" int rafting_step_wait(rafting_engine_t* e, rafting_lease_t* L) {
    if (!e || !L) return fail(RAFTING_E_INVAL, "null argument");
    CU(cudaSetDevice(e->cfg.device));
    const int sl = lease_slot(e, L);
    if (sl < 0) return fail(RAFTING_E_INVAL, "not an outstanding lease");
    int rc = slot_wait(e, (uint32_t)sl);
    if (rc) return rc;                                                       // the lease stays valid: wait again or release it
    hp(e)->slot[sl].leased = false; hp(e)->slot[sl].lease_key = nullptr;     // the lease ends with its step
    L->generation = 0;
    return rc;
}
extern "C" int rafting_step(rafting_engine_t* e, rafting_lease_t* L) {
    int rc = rafting_step_begin(e, L);
    if (rc) return rc;
    return rafting_step_wait(e, L);
}

// ---------------------------------------------------------------------------------------------
// group edits in step-stream order (rafting_group_edit_begin): the records' rows are built and checked on the host by the
// functions the synchronous calls use, travel up in one copy on the step stream, and one kernel writes them, so they take
// effect between the steps begun before the call and those begun after it.
// ---------------------------------------------------------------------------------------------
// one thread per record; the gids of a call are distinct, so no two threads touch the same row
__global__ void __launch_bounds__(256) group_edit_kernel(Tables T, const EditRow* __restrict__ rows, uint32_t n, uint32_t* __restrict__ bits) {
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n) return;
    const EditRow& r = rows[k];
    const size_t g = r.gid, F = T.F;
    if (r.kind == RAFTING_EDIT_CLOSE) {
        T.g_meta[g] &= ~(uint64_t)W_ALIVE;
    } else {
        const i64x2 z = {0, 0};
        T.g_meta[g] = r.meta; T.g_term[g] = r.term; T.g_commit[g] = r.commit; T.g_lo[g] = r.lo; T.g_hi[g] = r.hi;
        T.g_timer[g] = r.timer; T.g_epoch[g] = r.epoch; T.g_elect[g] = z; T.g_err[g] = 0;
        for (int q = 0; q < KRUNS; q++) T.g_runs[(size_t)q * T.G + g] = r.runs[q];
        for (size_t f = 0; f < F; f++) {
            T.l_nm[g * F + f] = z; T.l_es[g * F + f] = z; T.l_fr[g * F + f] = z; T.l_cnt[g * F + f] = make_int4(0, 0, 0, 0);
        }
    }
    if (bits)                                      // the compact path's in-flight table: the old life's tags are free again
        for (size_t f = 0; f < F; f++) bits[g * F + f] = 0;
}

// Pinned blocks the records travel from, used in turn, each reused once the event recorded behind its edit has fired, and one
// device block the copies land in: every copy and launch is on the step stream, so the next copy cannot overtake a launch.
constexpr int EDIT_STAGES = RAFTING_HOST_SLOTS;
struct EditPath { Blk host[EDIT_STAGES]; cudaEvent_t ev[EDIT_STAGES] = {}; Blk dev; uint32_t next = 0; };
static void edit_release(rafting_engine* e) {
    if (!e->edit) return;
    for (int k = 0; k < EDIT_STAGES; k++) { blk_free(e->edit->host[k], true); if (e->edit->ev[k]) cudaEventDestroy(e->edit->ev[k]); }
    blk_free(e->edit->dev, false);
    delete e->edit; e->edit = nullptr;
}
static int edit_row(const rafting_engine* e, uint32_t k, const rafting_group_edit_t& d, uint32_t prev_gid, EditRow& r) {
    if (d.gid >= e->G) return fail(RAFTING_E_CAPACITY, "edit %u: gid %u beyond max_groups", k, d.gid);
    if (k > 0 && d.gid <= prev_gid) return fail(RAFTING_E_INVAL, "edit %u: gid %u after gid %u (gids must increase strictly)", k, d.gid, prev_gid);
    if (d.kind == RAFTING_EDIT_CLOSE) { memset(&r, 0, sizeof(r)); r.gid = d.gid; r.kind = d.kind; return RAFTING_OK; }
    if (d.kind != RAFTING_EDIT_OPEN) return fail(RAFTING_E_INVAL, "edit %u: unknown kind %u", k, d.kind);
    if (int rc = open_row(e, d.gid, d.init, r)) return rc;
    if (d.n_runs == 0) return RAFTING_OK;
    if (d.n_runs > (uint32_t)KRUNS) return fail(RAFTING_E_CAPACITY, "edit %u: %u term runs: the engine keeps at most %d per group", k, d.n_runs, KRUNS);
    if (r.hi < r.lo) return fail(RAFTING_E_INVAL, "edit %u: group %u has term runs but no stored log", k, d.gid);
    if (int rc = runs_rows(r.lo, r.hi, d.init.last_term, d.runs, d.n_runs, r.runs)) return rc;
    r.meta = with_nruns(r.meta, d.n_runs);
    return RAFTING_OK;
}
extern "C" int rafting_group_edit_begin(rafting_engine_t* e, uint32_t n, const rafting_group_edit_t* edits) {
    if (!e) return fail(RAFTING_E_INVAL, "null argument");
    if (n == 0) return RAFTING_OK;
    if (!edits) return fail(RAFTING_E_INVAL, "null argument");
    if (n > e->G) return fail(RAFTING_E_CAPACITY, "%u edits: more than max_groups", n);
    CU(cudaSetDevice(e->cfg.device));
    if (!e->edit) {
        e->edit = new EditPath();
        for (int k = 0; k < EDIT_STAGES; k++) CU(cudaEventCreateWithFlags(&e->edit->ev[k], cudaEventDisableTiming));
    }
    EditPath& P = *e->edit;
    const uint32_t st = P.next;
    const size_t bytes = (size_t)n * sizeof(EditRow);
    CU(cudaEventSynchronize(P.ev[st]));                     // the stage's previous edit has run (a fresh event counts as fired)
    int rc;
    if ((rc = blk_reserve(P.host[st], bytes, true))) return rc;
    EditRow* rows = (EditRow*)P.host[st].p;
    for (uint32_t k = 0; k < n; k++)
        if ((rc = edit_row(e, k, edits[k], k ? edits[k - 1].gid : 0, rows[k]))) return rc;
    if (bytes > P.dev.cap) {                                 // growing frees the block an earlier edit may still read
        CU(cudaStreamSynchronize(e->stream));
        if ((rc = blk_reserve(P.dev, bytes, false))) return rc;
    }
    CU(cudaMemcpyAsync(P.dev.p, rows, bytes, cudaMemcpyHostToDevice, e->stream));
    group_edit_kernel<<<(n + 255) / 256, 256, 0, e->stream>>>(e->T, (const EditRow*)P.dev.p, n, compact_bits(e));
    CU(cudaGetLastError());
    CU(cudaEventRecord(P.ev[st], e->stream));
    P.next = (st + 1) % EDIT_STAGES;
    return RAFTING_OK;
}

// ---------------------------------------------------------------------------------------------
// state export (parity checks / checkpoint)
// ---------------------------------------------------------------------------------------------
static uint64_t fnv1a(uint64_t h, uint64_t v) {
    for (int i = 0; i < 8; i++) { h ^= (v >> (8 * i)) & 0xff; h *= 0x100000001B3ull; }
    return h;
}
extern "C" int rafting_state_export_bulk(rafting_engine_t* e, uint32_t first, uint32_t count, rafting_group_state_t* out) {
    if (!e || !out) return fail(RAFTING_E_INVAL, "null argument");
    if ((uint64_t)first + count > e->G) return fail(RAFTING_E_CAPACITY, "gid range beyond max_groups");
    if (count == 0) return RAFTING_OK;
    CU(cudaSetDevice(e->cfg.device));
    CU(cudaStreamSynchronize(e->stream));
    const size_t F = e->F; const Tables& T = e->T;
    std::vector<uint64_t> meta(count); std::vector<int64_t> term(count), commit(count), lo(count), hi(count), timer(count);
    std::vector<i64x2> epoch(count), elect(count), runs((size_t)count * KRUNS), nm(count * F), es(count * F), fr(count * F);
    std::vector<int4> cnt(count * F); std::vector<uint32_t> err(count);
    CU(cudaMemcpy(meta.data(), T.g_meta + first, count * 8, cudaMemcpyDeviceToHost));
    CU(cudaMemcpy(term.data(), T.g_term + first, count * 8, cudaMemcpyDeviceToHost));
    CU(cudaMemcpy(commit.data(), T.g_commit + first, count * 8, cudaMemcpyDeviceToHost));
    CU(cudaMemcpy(lo.data(), T.g_lo + first, count * 8, cudaMemcpyDeviceToHost));
    CU(cudaMemcpy(hi.data(), T.g_hi + first, count * 8, cudaMemcpyDeviceToHost));
    CU(cudaMemcpy(timer.data(), T.g_timer + first, count * 8, cudaMemcpyDeviceToHost));
    CU(cudaMemcpy(epoch.data(), T.g_epoch + first, count * 16, cudaMemcpyDeviceToHost));
    CU(cudaMemcpy(elect.data(), T.g_elect + first, count * 16, cudaMemcpyDeviceToHost));
    CU(cudaMemcpy(err.data(), T.g_err + first, count * 4, cudaMemcpyDeviceToHost));
    for (int k = 0; k < KRUNS; k++)
        CU(cudaMemcpy(runs.data() + (size_t)k * count, T.g_runs + (size_t)k * e->G + first, count * 16, cudaMemcpyDeviceToHost));
    CU(cudaMemcpy(nm.data(), T.l_nm + (size_t)first * F, count * F * 16, cudaMemcpyDeviceToHost));
    CU(cudaMemcpy(es.data(), T.l_es + (size_t)first * F, count * F * 16, cudaMemcpyDeviceToHost));
    CU(cudaMemcpy(fr.data(), T.l_fr + (size_t)first * F, count * F * 16, cudaMemcpyDeviceToHost));
    CU(cudaMemcpy(cnt.data(), T.l_cnt + (size_t)first * F, count * F * 16, cudaMemcpyDeviceToHost));
    for (uint32_t k = 0; k < count; k++) {
        rafting_group_state_t& o = out[k];
        memset(&o, 0, sizeof(o));
        const uint32_t w = (uint32_t)meta[k];
        const int nr = (int)((w >> W_NRUNS_SH) & 0xf);
        o.alive = (w & W_ALIVE) ? 1 : 0; o.role = w & W_ROLE_MASK; o.current_term = term[k];
        o.voted_for = (int)((w >> W_BALLOT_SH) & 0xff) - 1; o.current_leader = (int)((w >> W_LEADER_SH) & 0xff) - 1;
        o.incarnation = (uint32_t)(meta[k] >> 32);
        o.timeout_detected = (w & W_TIMEOUT_DET) ? 1 : 0; o.leader_prepared = (w & W_PREPARED) ? 1 : 0;
        o.votes = (int32_t)((uint64_t)elect[k].y >> 32); o.elected_inc = (uint32_t)(uint64_t)elect[k].y;
        o.elected_aborted = (w & W_ELECT_ABORT) ? 1 : 0; o.elected_term = elect[k].x;
        o.timer = timer[k]; o.commit_index = commit[k]; o.epoch_index = epoch[k].x; o.epoch_term = epoch[k].y;
        uint64_t h = 0xCBF29CE484222325ull;
        if (nr > 0) {
            o.first_index = lo[k]; o.last_index = hi[k]; o.last_term = runs[k].y;
            for (int r = nr - 1; r >= 0; r--) {
                const i64x2& run = runs[(size_t)r * count + k];
                int64_t start = (r == nr - 1) ? lo[k] : run.x;    // the oldest run starts at the lowest stored key
                h = fnv1a(h, (uint64_t)start); h = fnv1a(h, (uint64_t)run.y);
            }
            h = fnv1a(h, (uint64_t)hi[k]);
        } else { o.first_index = 1; o.last_index = 0; o.last_term = 0; }
        o.term_runs = (uint32_t)nr; o.err_word = err[k]; o.log_digest = h; o.n_followers = (uint32_t)F;
        if (o.role == RAFTING_ROLE_LEADER && o.leader_prepared) {
            for (size_t f = 0; f < F; f++) {
                rafting_follower_state_t& d = o.followers[f]; const size_t li = (size_t)k * F + f;
                d.next_index = nm[li].x; d.match_index = nm[li].y; d.last_epoch = es[li].x; d.request_success = es[li].y;
                d.request_failure = fr[li].x; d.last_request = fr[li].y;
                d.request_in_flight = cnt[li].x; d.recent_rejection = cnt[li].y; d.recent_failure = cnt[li].z;
                d.pending_installation = cnt[li].w;
            }
        }
    }
    return RAFTING_OK;
}
extern "C" int rafting_state_export(rafting_engine_t* e, uint32_t gid, rafting_group_state_t* out) {
    return rafting_state_export_bulk(e, gid, 1, out);
}
extern "C" int rafting_state_digest(rafting_engine_t* e, uint32_t first, uint32_t count, uint64_t* digests) {
    if (!digests) return fail(RAFTING_E_INVAL, "null argument");
    const uint32_t chunk = 4096;
    std::vector<rafting_group_state_t> buf(chunk);
    for (uint32_t off = 0; off < count; off += chunk) {
        uint32_t c = count - off < chunk ? count - off : chunk;
        int rc = rafting_state_export_bulk(e, first + off, c, buf.data());
        if (rc) return rc;
        for (uint32_t k = 0; k < c; k++) {
            const unsigned char* p = (const unsigned char*)&buf[k];
            uint64_t h = 0xCBF29CE484222325ull;
            const size_t used = offsetof(rafting_group_state_t, followers) + sizeof(rafting_follower_state_t) * e->F;
            for (size_t b = 0; b < used; b++) { h ^= p[b]; h *= 0x100000001B3ull; }
            digests[off + k] = h;
        }
    }
    return RAFTING_OK;
}
extern "C" int rafting_log_term(rafting_engine_t* e, uint32_t gid, int64_t index, int64_t* term) {
    if (!e || gid >= e->G || !term) return fail(RAFTING_E_INVAL, "bad argument");
    CU(cudaSetDevice(e->cfg.device));
    CU(cudaStreamSynchronize(e->stream));
    uint64_t meta; int64_t lo, hi; i64x2 runs[KRUNS];
    CU(cudaMemcpy(&meta, e->T.g_meta + gid, 8, cudaMemcpyDeviceToHost));
    CU(cudaMemcpy(&lo, e->T.g_lo + gid, 8, cudaMemcpyDeviceToHost));
    CU(cudaMemcpy(&hi, e->T.g_hi + gid, 8, cudaMemcpyDeviceToHost));
    for (int k = 0; k < KRUNS; k++) CU(cudaMemcpy(&runs[k], e->T.g_runs + (size_t)k * e->G + gid, 16, cudaMemcpyDeviceToHost));
    const int nr = (int)(((uint32_t)meta >> W_NRUNS_SH) & 0xf);
    *term = -1;
    if (nr == 0 || index < lo || index > hi) return RAFTING_OK;
    for (int k = 0; k < nr; k++) if (index >= runs[k].x || k == nr - 1) { *term = runs[k].y; break; }
    return RAFTING_OK;
}

extern "C" int rafting_checkpoint(rafting_engine_t* e) {
    if (!e) return fail(RAFTING_E_INVAL, "null argument");
    CU(cudaSetDevice(e->cfg.device));
    e->shadow.resize(e->dev_allocs.size(), nullptr);
    for (size_t i = 0; i < e->dev_allocs.size(); i++) {
        if (!e->dev_is_state[i]) continue;
        if (!e->shadow[i]) CU(cudaMalloc(&e->shadow[i], e->dev_bytes[i]));
        CU(cudaMemcpyAsync(e->shadow[i], e->dev_allocs[i], e->dev_bytes[i], cudaMemcpyDeviceToDevice, e->stream));
    }
    CU(cudaStreamSynchronize(e->stream));
    return RAFTING_OK;
}
// The checkpoint copies the state allocations that existed when it was taken (the tables).  A state allocation created
// later (the compact path's in-flight table, on its first use) held nothing at the checkpoint: a restore zeroes it, so
// no tag handed out after the checkpoint survives the rollback.  Scratch (the gather buffers of rafting_comm_init,
// staging) is not state and is left alone.
static int restore_enqueue(rafting_engine* e) {
    if (e->shadow.empty()) return fail(RAFTING_E_INVAL, "no checkpoint taken");
    CU(cudaSetDevice(e->cfg.device));
    for (size_t i = 0; i < e->shadow.size(); i++)
        if (e->shadow[i]) CU(cudaMemcpyAsync(e->dev_allocs[i], e->shadow[i], e->dev_bytes[i], cudaMemcpyDeviceToDevice, e->stream));
    for (size_t i = e->shadow.size(); i < e->dev_allocs.size(); i++)
        if (e->dev_is_state[i]) CU(cudaMemsetAsync(e->dev_allocs[i], 0, e->dev_bytes[i], e->stream));
    return RAFTING_OK;
}
extern "C" int rafting_restore(rafting_engine_t* e) {
    if (!e) return fail(RAFTING_E_INVAL, "null argument");
    int rc = restore_enqueue(e); if (rc) return rc;
    CU(cudaStreamSynchronize(e->stream));
    return RAFTING_OK;
}
extern "C" int rafting_restore_async(rafting_engine_t* e) {          // enqueued on the step stream, no host synchronisation
    if (!e) return fail(RAFTING_E_INVAL, "null argument");
    return restore_enqueue(e);
}

// ---------------------------------------------------------------------------------------------
// exportable checkpoint (SURVEY §8(f)-4): the tables of a shard as ONE file that survives the process.
// RaftContext.initialize rebuilds a context from StableLock + RaftLog (RaftContext.java:91-113) and starts every group as a
// Follower; a planned restart of a pump (upgrade, rebalance to another GPU) can instead save the whole shard — roles, timers,
// Leadership.State, in-flight table — and load it into a fresh engine of the same shape.  Layout: header { magic, version,
// G, F, term runs, n blocks, total bytes } + { bytes, crc32c } per block + the blocks; written to <path>.tmp, fdatasync'ed,
// renamed over <path> (a crash leaves the old image or none, never a torn one).
// ---------------------------------------------------------------------------------------------
#include <errno.h>
#include <fcntl.h>
#include <sys/stat.h>
#include <unistd.h>
namespace {
struct ImgHdr { uint32_t magic, version, G, F, runs, nblocks; uint64_t total; };
constexpr uint32_t IMG_MAGIC = 0x31474D49u;     // "IMG1"
uint32_t img_crc_table[256]; bool img_crc_ready = false;
uint32_t img_crc32c(const void* p, size_t n) {
    if (!img_crc_ready) {
        for (uint32_t i = 0; i < 256; i++) { uint32_t v = i; for (int k = 0; k < 8; k++) v = (v & 1) ? (v >> 1) ^ 0x82F63B78u : v >> 1; img_crc_table[i] = v; }
        img_crc_ready = true;
    }
    const uint8_t* b = (const uint8_t*)p; uint32_t c = ~0u;
    for (size_t i = 0; i < n; i++) c = img_crc_table[(c ^ b[i]) & 0xff] ^ (c >> 8);
    return ~c;
}
bool img_write_all(int fd, const void* p, size_t n) {
    const uint8_t* b = (const uint8_t*)p;
    while (n) { const ssize_t w = write(fd, b, n); if (w < 0) { if (errno == EINTR) continue; return false; } b += w; n -= (size_t)w; }
    return true;
}
bool img_read_all(int fd, void* p, size_t n) {
    uint8_t* b = (uint8_t*)p;
    while (n) { const ssize_t r = read(fd, b, n); if (r < 0) { if (errno == EINTR) continue; return false; } if (r == 0) return false; b += r; n -= (size_t)r; }
    return true;
}
}  // namespace
extern "C" int rafting_state_save(rafting_engine_t* e, const char* path) {
    if (!e || !path) return fail(RAFTING_E_INVAL, "null argument");
    CU(cudaSetDevice(e->cfg.device));
    int rc = quiesce_for_table_edit(e, "rafting_state_save"); if (rc) return rc;
    std::vector<size_t> ids;
    for (size_t i = 0; i < e->dev_allocs.size(); i++) if (e->dev_is_state[i]) ids.push_back(i);
    ImgHdr h; h.magic = IMG_MAGIC; h.version = RAFTING_ABI_VERSION; h.G = e->G; h.F = e->F; h.runs = KRUNS; h.nblocks = (uint32_t)ids.size(); h.total = 0;
    for (size_t i : ids) h.total += e->dev_bytes[i];
    std::string tmp = std::string(path) + ".tmp";
    const int fd = open(tmp.c_str(), O_WRONLY | O_CREAT | O_TRUNC, 0644);
    if (fd < 0) return fail(RAFTING_E_CUDA, "open %s: %s", tmp.c_str(), strerror(errno));
    bool ok = img_write_all(fd, &h, sizeof(h));
    std::vector<uint8_t> buf;
    for (size_t i : ids) {
        if (!ok) break;
        buf.resize(e->dev_bytes[i]);
        if (cudaMemcpy(buf.data(), e->dev_allocs[i], buf.size(), cudaMemcpyDeviceToHost) != cudaSuccess) { close(fd); unlink(tmp.c_str()); return fail(RAFTING_E_CUDA, "copy of block %zu failed", i); }
        const uint64_t meta[2] = {(uint64_t)buf.size(), (uint64_t)img_crc32c(buf.data(), buf.size())};
        ok = img_write_all(fd, meta, sizeof(meta)) && img_write_all(fd, buf.data(), buf.size());
    }
    ok = ok && fdatasync(fd) == 0;
    close(fd);
    if (!ok || rename(tmp.c_str(), path) != 0) { const int err = errno; unlink(tmp.c_str()); return fail(RAFTING_E_CUDA, "writing %s failed: %s", path, strerror(err)); }
    return RAFTING_OK;
}
extern "C" int rafting_state_load(rafting_engine_t* e, const char* path) {
    if (!e || !path) return fail(RAFTING_E_INVAL, "null argument");
    CU(cudaSetDevice(e->cfg.device));
    int rc = quiesce_for_table_edit(e, "rafting_state_load"); if (rc) return rc;
    const int fd = open(path, O_RDONLY);
    if (fd < 0) return fail(RAFTING_E_INVAL, "open %s: %s", path, strerror(errno));
    ImgHdr h;
    if (!img_read_all(fd, &h, sizeof(h)) || h.magic != IMG_MAGIC) { close(fd); return fail(RAFTING_E_INVAL, "%s is not a shard image", path); }
    if (h.version != RAFTING_ABI_VERSION || h.G != e->G || h.F != e->F || h.runs != (uint32_t)KRUNS) {
        close(fd); return fail(RAFTING_E_INVAL, "image of a different shape (G %u F %u runs %u abi %u)", h.G, h.F, h.runs, h.version);
    }
    // an image taken after the compact path was used carries the in-flight table: create ours before matching blocks.  One
    // taken before carries none: it is loaded into the other blocks, and our table is zeroed (nothing in flight), as it was
    // when the image was saved
    std::vector<size_t> ids, cleared;
    for (size_t i = 0; i < e->dev_allocs.size(); i++) if (e->dev_is_state[i]) ids.push_back(i);
    if (h.nblocks == ids.size() + 3) { rc = compact_state(e); if (rc) { close(fd); return rc; } ids.clear(); for (size_t i = 0; i < e->dev_allocs.size(); i++) if (e->dev_is_state[i]) ids.push_back(i); }
    if (e->compact && h.nblocks + 3 == ids.size()) {
        std::vector<size_t> keep;
        for (size_t i : ids) (compact_owns(e, e->dev_allocs[i]) ? cleared : keep).push_back(i);
        ids.swap(keep);
    }
    if (h.nblocks != ids.size()) { close(fd); return fail(RAFTING_E_INVAL, "image holds %u blocks, the engine %zu", h.nblocks, ids.size()); }
    // read + verify everything first: a corrupt image must not leave the tables half loaded
    std::vector<std::vector<uint8_t>> blocks(h.nblocks);
    for (uint32_t k = 0; k < h.nblocks; k++) {
        uint64_t meta[2];
        if (!img_read_all(fd, meta, sizeof(meta)) || meta[0] != e->dev_bytes[ids[k]]) { close(fd); return fail(RAFTING_E_INVAL, "block %u: size mismatch / truncated image", k); }
        blocks[k].resize(meta[0]);
        if (!img_read_all(fd, blocks[k].data(), meta[0]) || img_crc32c(blocks[k].data(), meta[0]) != (uint32_t)meta[1]) { close(fd); return fail(RAFTING_E_INVAL, "block %u: checksum mismatch", k); }
    }
    close(fd);
    for (uint32_t k = 0; k < h.nblocks; k++) CU(cudaMemcpy(e->dev_allocs[ids[k]], blocks[k].data(), blocks[k].size(), cudaMemcpyHostToDevice));
    for (size_t i : cleared) CU(cudaMemsetAsync(e->dev_allocs[i], 0, e->dev_bytes[i], e->stream));
    CU(cudaStreamSynchronize(e->stream));
    return RAFTING_OK;
}

// ---------------------------------------------------------------------------------------------
// multi-GPU commitIndex summary
// ---------------------------------------------------------------------------------------------
// Shards are contiguous gid blocks: rank r owns global groups [r*G, (r+1)*G).  The only exchange between shards is one
// ncclAllGather of commitIndex[G] per step into a [world * G] buffer kept on every rank (two of them, alternating, so the
// consumer of step k's summary is not overwritten by step k+1's gather).
//   * the gather runs on its own stream (s_comm) behind the kernel that produced the column;
//   * SOURCE = a device column the caller names (normally the step's outbox commit_index column: an end-of-step
//     snapshot no later kernel writes, so the gathered vector is EXACTLY the state after that step on every rank), or the
//     live table column, in which case the step stream is made to wait for the gather before the next kernel may change it;
//   * after enqueuing gather k the step stream waits for gather k-1: a caller that rotates two (or more) outboxes
//     therefore never overwrites a column a gather is still reading, and the next step kernel never waits for the
//     gather of the step right before it.
extern "C" int rafting_commit_slice(rafting_engine_t* e, void** dev_ptr, uint32_t* count) {
    if (!e || !dev_ptr || !count) return fail(RAFTING_E_INVAL, "null argument");
    *dev_ptr = e->T.g_commit; *count = e->G;
    return RAFTING_OK;
}
extern "C" int rafting_comm_unique_id(void* out, size_t* len) {
    if (!out || !len || *len < sizeof(nccl_uid_t)) return fail(RAFTING_E_INVAL, "buffer too small (need 128)");
    int rc = nccl_load(); if (rc) return rc;
    nccl_uid_t id;
    int nr = g_nccl.GetUniqueId(&id);
    if (nr) return fail(RAFTING_E_NCCL, "ncclGetUniqueId: %s", g_nccl.GetErrorString ? g_nccl.GetErrorString(nr) : "?");
    memcpy(out, &id, sizeof(id)); *len = sizeof(id);
    return RAFTING_OK;
}
static int comm_prepare(rafting_engine* e, int rank, int world) {
    if (e->gather[0]) return fail(RAFTING_E_INVAL, "communicator already initialised");
    CU(cudaSetDevice(e->cfg.device));
    for (int p = 0; p < 2; p++) { int rc = dalloc(e, &e->gather[p], (size_t)world * e->G); if (rc) return rc; }
    CU(cudaStreamCreateWithFlags(&e->s_comm, cudaStreamNonBlocking));
    CU(cudaEventCreateWithFlags(&e->ev_step, cudaEventDisableTiming));
    for (int p = 0; p < 2; p++) CU(cudaEventCreateWithFlags(&e->ev_gather[p], cudaEventDisableTiming));
    e->rank = rank; e->world = world; e->gather_seq = 0;
    return RAFTING_OK;
}
// one process per GPU (torchrun shape): every rank calls this with the same unique id
extern "C" int rafting_comm_init(rafting_engine_t* e, int rank, int world, const void* uid, size_t id_len) {
    if (!e || world < 1 || rank < 0 || rank >= world) return fail(RAFTING_E_INVAL, "bad rank/world");
    if (world > 1 && (!uid || id_len != sizeof(nccl_uid_t))) return fail(RAFTING_E_INVAL, "unique id must be 128 bytes");
    int rc = comm_prepare(e, rank, world); if (rc) return rc;
    if (world > 1) {
        rc = nccl_load(); if (rc) return rc;
        nccl_uid_t id; memcpy(&id, uid, sizeof(id));
        int nr = g_nccl.CommInitRank(&e->comm, world, id, rank);
        if (nr) return fail(RAFTING_E_NCCL, "ncclCommInitRank: %s", g_nccl.GetErrorString ? g_nccl.GetErrorString(nr) : "?");
    }
    return RAFTING_OK;
}
// ONE process that owns several shards (the reference's host is one JVM: ContextManager.java:46 — one pump thread per
// shard): engines[r] becomes rank r of an n-rank communicator.  ncclCommInitRank blocks until every rank has joined, so
// the n calls are issued inside one ncclGroupStart / ncclGroupEnd from this single thread.
extern "C" int rafting_comm_init_all(rafting_engine_t** engines, int n) {
    if (!engines || n < 1) return fail(RAFTING_E_INVAL, "bad argument");
    for (int r = 0; r < n; r++) {
        if (!engines[r]) return fail(RAFTING_E_INVAL, "null engine");
        if (engines[r]->G != engines[0]->G) return fail(RAFTING_E_INVAL, "every shard must have the same max_groups");
        for (int q = 0; q < r; q++) if (engines[q]->cfg.device == engines[r]->cfg.device) return fail(RAFTING_E_INVAL, "two shards on device %d", engines[r]->cfg.device);
    }
    int rc;
    for (int r = 0; r < n; r++) if ((rc = comm_prepare(engines[r], r, n))) return rc;
    if (n == 1) return RAFTING_OK;
    rc = nccl_load(); if (rc) return rc;
    if (!g_nccl.GroupStart || !g_nccl.GroupEnd) return fail(RAFTING_E_NCCL, "libnccl lacks ncclGroupStart/End");
    nccl_uid_t id;
    int nr = g_nccl.GetUniqueId(&id);
    if (nr) return fail(RAFTING_E_NCCL, "ncclGetUniqueId: %s", g_nccl.GetErrorString ? g_nccl.GetErrorString(nr) : "?");
    g_nccl.GroupStart();
    for (int r = 0; r < n && !nr; r++) {
        cudaSetDevice(engines[r]->cfg.device);
        nr = g_nccl.CommInitRank(&engines[r]->comm, n, id, r);
    }
    const int ne = g_nccl.GroupEnd();
    if (nr || ne) return fail(RAFTING_E_NCCL, "ncclCommInitRank (grouped): %s", g_nccl.GetErrorString ? g_nccl.GetErrorString(nr ? nr : ne) : "?");
    return RAFTING_OK;
}
// enqueue half of one shard's gather (no host synchronisation)
static int gather_enqueue(rafting_engine* e, const int64_t* dev_src, int64_t** recv_out) {
    if (!e->gather[0]) return fail(RAFTING_E_NCCL, "communicator not initialised (rafting_comm_init)");
    CU(cudaSetDevice(e->cfg.device));
    const int p = (int)(e->gather_seq & 1);
    const int64_t* src = dev_src ? dev_src : e->T.g_commit;
    int64_t* recv = e->gather[p];
    CU(cudaEventRecord(e->ev_step, e->stream));
    CU(cudaStreamWaitEvent(e->s_comm, e->ev_step, 0));
    if (e->world > 1) {
        if (!e->comm) return fail(RAFTING_E_NCCL, "communicator not initialised");
        int nr = g_nccl.AllGather(src, recv, e->G, /*ncclInt64*/ 4, e->comm, e->s_comm);
        if (nr) return fail(RAFTING_E_NCCL, "ncclAllGather: %s", g_nccl.GetErrorString ? g_nccl.GetErrorString(nr) : "?");
    } else {
        CU(cudaMemcpyAsync(recv, src, (size_t)e->G * 8, cudaMemcpyDeviceToDevice, e->s_comm));
    }
    CU(cudaEventRecord(e->ev_gather[p], e->s_comm));
    // the live table column may change with the next kernel: that kernel waits for THIS gather; a snapshot column only
    // has to survive until the caller's rotation comes back to it: the step stream waits for the PREVIOUS gather
    if (!dev_src) CU(cudaStreamWaitEvent(e->stream, e->ev_gather[p], 0));
    else if (e->gather_seq > 0) CU(cudaStreamWaitEvent(e->stream, e->ev_gather[p ^ 1], 0));
    e->gather_seq++;
    *recv_out = recv;
    return RAFTING_OK;
}
static int gather_finish(rafting_engine* e, int64_t* recv, int64_t* host_out, void** dev_out) {
    if (dev_out) *dev_out = recv;
    if (host_out) {
        CU(cudaSetDevice(e->cfg.device));
        CU(cudaMemcpyAsync(host_out, recv, (size_t)e->world * e->G * 8, cudaMemcpyDeviceToHost, e->s_comm));
        CU(cudaStreamSynchronize(e->s_comm));
    }
    return RAFTING_OK;
}
extern "C" int rafting_allgather_commit_from(rafting_engine_t* e, const int64_t* dev_src, int64_t* host_out, void** dev_out) {
    if (!e) return fail(RAFTING_E_INVAL, "null argument");
    int64_t* recv = nullptr;
    int rc = gather_enqueue(e, dev_src, &recv); if (rc) return rc;
    return gather_finish(e, recv, host_out, dev_out);
}
extern "C" int rafting_allgather_commit(rafting_engine_t* e, int64_t* host_out, void** dev_out) {
    return rafting_allgather_commit_from(e, nullptr, host_out, dev_out);
}
// the same for every shard of a single-process communicator (rafting_comm_init_all): the n ncclAllGather calls are
// issued as one group; dev_srcs / host_outs / dev_outs may be NULL or hold NULL entries
extern "C" int rafting_allgather_commit_all(rafting_engine_t** engines, int n, const int64_t* const* dev_srcs,
                                            int64_t* const* host_outs, void** dev_outs) {
    if (!engines || n < 1) return fail(RAFTING_E_INVAL, "bad argument");
    for (int r = 0; r < n; r++) if (!engines[r] || engines[r]->world != n || engines[r]->rank != r) return fail(RAFTING_E_INVAL, "engines[%d] is not rank %d of an %d-shard communicator", r, r, n);
    std::vector<int64_t*> recv((size_t)n, nullptr);
    int rc = RAFTING_OK;
    if (n > 1) g_nccl.GroupStart();
    for (int r = 0; r < n && !rc; r++) rc = gather_enqueue(engines[r], dev_srcs ? dev_srcs[r] : nullptr, &recv[r]);
    if (n > 1) { const int ne = g_nccl.GroupEnd(); if (!rc && ne) rc = fail(RAFTING_E_NCCL, "ncclGroupEnd: %s", g_nccl.GetErrorString ? g_nccl.GetErrorString(ne) : "?"); }
    if (rc) return rc;
    for (int r = 0; r < n; r++) {
        rc = gather_finish(engines[r], recv[r], host_outs ? host_outs[r] : nullptr, dev_outs ? &dev_outs[r] : nullptr);
        if (rc) return rc;
    }
    return RAFTING_OK;
}
// the most recently gathered vector, copied to the host (synchronises the gather stream)
extern "C" int rafting_allgather_last(rafting_engine_t* e, int64_t* host_out) {
    if (!e || !host_out) return fail(RAFTING_E_INVAL, "null argument");
    if (!e->s_comm || e->gather_seq == 0) return fail(RAFTING_E_INVAL, "no gather has been issued");
    CU(cudaSetDevice(e->cfg.device));
    CU(cudaMemcpyAsync(host_out, e->gather[(e->gather_seq - 1) & 1], (size_t)e->world * e->G * 8, cudaMemcpyDeviceToHost, e->s_comm));
    CU(cudaStreamSynchronize(e->s_comm));
    return RAFTING_OK;
}
// makes the step stream wait for every all-gather enqueued so far (e.g. before a timing event or a restore)
extern "C" int rafting_allgather_join(rafting_engine_t* e) {
    if (!e) return fail(RAFTING_E_INVAL, "null argument");
    if (!e->s_comm || e->gather_seq == 0) return RAFTING_OK;
    CU(cudaSetDevice(e->cfg.device));
    CU(cudaStreamWaitEvent(e->stream, e->ev_gather[(e->gather_seq - 1) & 1], 0));
    return RAFTING_OK;
}

extern "C" int rafting_engine_stream(rafting_engine_t* e, void** s) {
    if (!e || !s) return fail(RAFTING_E_INVAL, "null argument");
    *s = e->stream; return RAFTING_OK;
}
extern "C" int rafting_engine_counters(rafting_engine_t* e, uint64_t* launches, uint64_t* events) {
    if (!e) return fail(RAFTING_E_INVAL, "null argument");
    if (launches) *launches = e->launches;
    if (events) *events = e->events;
    return RAFTING_OK;
}
// the kernel's integer form of round(ln(e + r)) (Leadership.java:105), exposed so a CPU test can check it against libm
extern "C" int64_t rafting_backoff_step(int32_t r) { return rafting::backoff_step(r); }
// compile-time layout facts for tests/test_abi.py
extern "C" int rafting_abi_sizes(uint32_t* out, uint32_t n) {
    const uint32_t v[] = {(uint32_t)sizeof(rafting_cfg_t), (uint32_t)sizeof(rafting_inbox_t), (uint32_t)sizeof(rafting_outbox_t),
                          (uint32_t)sizeof(rafting_group_init_t), (uint32_t)sizeof(rafting_follower_state_t),
                          (uint32_t)sizeof(rafting_group_state_t), (uint32_t)sizeof(rafting_lease_t)};
    for (uint32_t i = 0; i < n && i < 7; i++) out[i] = v[i];
    return 7;
}

#include "timers.cuh"
#include "compact.cuh"
#include "seglog.cuh"
