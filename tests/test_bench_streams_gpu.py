"""The streams and the launch pattern bench.py times, held to the CPU oracle (`-m gpu`).

bench.py's headline number comes from inboxes that the device generators of rafting_b200/csrc/workload.cu write straight
into HBM, replayed by rafting_step_device_seq with pair_kernel launched programmatically from the second launch on.  The
bench's own exactness checks (replay_ok, e2e_exact) compare the engine with itself.  This suite holds that path to the
oracle:

  1. every device generator writes, byte for byte, what its host twin writes: the same step from the same previous outbox
     (an oracle outbox), both sides' columns poisoned first, so a cell one side writes and the other leaves alone differs;
  2. config #2 at the bench's shape, launch by launch as run_engine drives it: the device election, 8 settle launches
     through one reused inbox, a recorded window of distinct inboxes, two timed replays, a per-launch replay into
     poisoned outboxes, and --dump-outputs;
  3. one shard of config #4 (rank 5 of 8) on one GPU through the same driver;
  4. tools/bench_secondary.py's closed loops for configs #3 and #5 at reduced sizes.

The bench reuses inboxes (its settle inbox, bench_secondary's single inbox) and the generators write a lane's payload only
where they write an event, so the engine here always consumes inboxes holding an earlier launch's payload under a zero
ev_meta while the oracle consumes fresh ones.  An outbox at the bench's shape is ~150 MB: launches that cannot be compared
with the oracle on the spot are compared through per-column hashes (payloads masked as abi.Outbox.equal masks them).
tests/test_bench_streams_cpu.py checks the run_engine recipe restated here against bench.py's source."""
import ctypes as C
import hashlib
import sys
import types

import numpy as np
import pytest

from oracle import binding
from rafting_b200 import abi, workload
from tests import harness

pytestmark = pytest.mark.gpu

# ---- run_engine's locals, restated -------------------------------------------------------------------------------------
SETTLE = 8                         # settle launches before the checkpoint


def bench_init(G, gid_base):
    """run_engine's open_bulk argument: a fresh Follower per group, terms keyed by the global group id."""
    return harness.init_array(G, terms=(gid_base + np.arange(G)) % 7)


ORACLE_THREADS = 16
POISON = harness.POISON
SEED2, SEED3, SEED5 = 0x5EED0002, 0x5EED0003, 0x5EED0005      # bench.SEED2, bench_secondary's seeds
IN_COLS = (("op_meta", np.uint64, False), ("op_nr", abi.I64X2, False), ("op_ab", abi.I64X2, False), ("op_cd", abi.I64X2, False),
           ("op_e", np.int64, False), ("ev_meta", np.uint64, True), ("ev_tn", abi.I64X2, True), ("ev_el", abi.I64X2, True))
ALL_COLS = tuple(name for name, _, _ in IN_COLS)
LEADER_COLS = ("op_meta", "op_nr", "op_ab", "ev_meta", "ev_tn", "ev_el")       # DevInbox(requests=False): the election too
BENCH_COLS = ("op_meta", "op_nr", "ev_meta", "ev_tn", "ev_el")                 # DevInbox(requests=False, unavail=False)


@pytest.fixture(scope="module")
def dev():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    yield torch.device("cuda", 0)
    torch.cuda.empty_cache()


def sync():
    import torch
    torch.cuda.synchronize()


# ---- generators --------------------------------------------------------------------------------------------------------
def generate(kind, w, step, prev_c, ic, on_device, stream=0):
    L = workload._bind()
    fn = {"leader": L.rafting_wl_leader_step, "election": L.rafting_wl_election_step,
          "vote": L.rafting_wl_vote_step, "mixed": L.rafting_wl_mixed_step}[kind]
    rc = fn(C.byref(w), step, None if prev_c is None else C.byref(prev_c), C.byref(ic), 1 if on_device else 0, C.c_void_p(stream))
    assert rc == 0, f"rafting_wl_{kind}_step rc={rc}"


def host_inbox(kind, w, step, prev, cols, gids=None, flags=0, fill=0):
    """The host generator's inbox of one step: the columns `cols` (the others absent), every byte `fill` beforehand; a mixed
    step carries the entry-term pool as mixed_inbox_host's does."""
    ib = abi.Inbox(w.rows, w.n, w.F, ent_cap=workload.POOL_TERMS if kind == "mixed" else 0, gids=gids)
    ib.flags = flags
    for name in ALL_COLS:
        if name in cols:
            getattr(ib, name).view(np.uint8).fill(fill)
        else:
            setattr(ib, name, None)
    if kind == "mixed":
        assert workload._bind().rafting_wl_fill_term_pool(ib.ent_terms.ctypes.data, workload.POOL_TERMS, 0, None) == 0
        ib.ent_count = workload.POOL_TERMS
    generate(kind, w, step, None if prev is None else prev.as_c(), ib.as_c(), False)
    return ib


def device_inbox(kind, w, step, dprev, cols, dev, gids=None, flags=0):
    """The device generator's inbox of the same step into a DevInbox whose columns `cols` start as POISON."""
    from rafting_b200 import devbatch
    din = devbatch.DevInbox(w.rows, w.n, w.F, dev, requests=True)
    din.t = {name: t.fill_(POISON) for name, t in din.t.items() if name in cols}
    din.flags, din.gids = flags, gids
    generate(kind, w, step, None if dprev is None else dprev.as_c(), din.as_c(), True)
    sync()
    return din


def device_outbox(ob, dev):
    """A DevOutbox holding the bytes of the host outbox ob."""
    import torch
    from rafting_b200 import devbatch
    d = devbatch.DevOutbox(ob.rows, ob.n, ob.F, ob.G, dev)
    for name, t in d.t.items():
        t.copy_(torch.from_numpy(np.ascontiguousarray(getattr(ob, name)).view(np.uint8).reshape(-1)))
    return d


def assert_inbox_equal(hib, din, where, written_only=False):
    """Every column of the device inbox din against the host inbox hib, byte for byte.  written_only: the lane payloads only
    under a non-zero ev_meta, the cells a generator writes (din is reused, hib fresh)."""
    for name, dt, lane in IN_COLS:
        h = getattr(hib, name)
        if name not in din.t:
            assert h is None, f"{where}: {name} present on the host only"
            continue
        assert h is not None, f"{where}: {name} present on the device only"
        d = din.t[name].cpu().numpy().view(dt).reshape(h.shape)
        if written_only and name in ("ev_tn", "ev_el"):
            m = hib.ev_meta != 0
            h, d = h[m], d[m]
        if h.size == 0:
            continue
        hb = np.ascontiguousarray(h).view(np.uint8).reshape(h.size, -1)
        db = np.ascontiguousarray(d).view(np.uint8).reshape(d.size, -1)
        bad = np.flatnonzero((hb != db).any(axis=1))
        if len(bad):
            at = bad[0] if h.ndim == 1 else np.unravel_index(bad[0], h.shape)
            raise AssertionError(f"{where}: inbox column {name} differs in {len(bad)} cells, first at {at}: "
                                 f"host {hb[bad[0]].tobytes().hex()} device {db[bad[0]].tobytes().hex()}")


def op_kinds(ib):
    return set(np.unique(ib.op_meta & np.uint64(0xFF)).tolist()) if ib.op_meta is not None else set()


def event_tags(ib):
    """(kind, outcome, lane) of every event of the inbox."""
    m = ib.ev_meta
    lanes = np.broadcast_to(np.arange(m.shape[-1], dtype=np.uint64), m.shape)
    tags = (m & np.uint64(0xF)) | (((m >> np.uint64(4)) & np.uint64(3)) << np.uint64(4)) | (lanes << np.uint64(8))
    return {(t & 0xF, (t >> 4) & 3, t >> 8) for t in np.unique(tags[(m & np.uint64(0xF)) != 0]).tolist()}


# ---- 1. device generators against host generators ----------------------------------------------------------------------
SHAPES_N = (1, 255, 256, 257, 777, 4096)
SHAPES_ROWS = (1, 3, 16)
GID_BASES = (0, 5 * 131072)        # the second: rank 5 of a 1 M-group config #4 shard


def check_stream(kind, F, n, rows, gid_base, dev, *, listed=None, local_slot=0, col_sets=None, seen=None):
    """Drives `kind`'s stream closed-loop on the oracle (host generator into fresh columns, oracle step) and, at chosen
    steps, generates the step again on the host and on the device from the same oracle outbox into poisoned columns.
    listed: None, "gids" (an active list, group columns by gid) or "compact" (RAFTING_INBOX_COMPACT_GROUPS).  Every step
    runs ~144 ticks into a mixed stream, past the 64-tick churn and 128-tick catch-up cycles; the vote and leader streams
    are checked from their first step."""
    import torch
    R = F + 1
    G = 2 * n + 5 if listed else n
    gids = np.sort(np.random.default_rng([n, rows, F]).choice(G, n, replace=False)).astype(np.uint32) if listed else None
    gids_d = None if gids is None else torch.from_numpy(gids).to(dev)
    lflag = abi.INBOX_COMPACT_GROUPS if listed == "compact" else 0
    seed = {"leader": SEED2, "election": SEED2, "vote": SEED3, "mixed": SEED5}[kind]
    cfg = abi.make_cfg(replicas=R, local_slot=local_slot, max_groups=G, max_rows=rows,
                       entry_pool_cap=workload.POOL_TERMS if kind == "mixed" else 0)
    o = binding.Oracle(cfg)
    if kind == "vote":
        init = harness.init_array(G, terms=1 + np.arange(G) % 5)
        init["last_index"] = 100 + np.arange(G) % 50
        init["last_term"] = 1 + np.arange(G) % 5
    else:
        init = bench_init(G, gid_base)
    o.open_bulk(0, init)
    col_sets = col_sets or ((LEADER_COLS if kind in ("leader", "election") else ALL_COLS),)
    flags = (abi.INBOX_NO_REQUESTS if kind in ("leader", "election") else 0) | lflag
    shape = f"{kind} F={F} n={n} rows={rows} gid_base={gid_base} list={listed} local_slot={local_slot}"

    def check(k, w, step, prev):
        dprev = None if prev is None else device_outbox(prev, dev)
        for cols in col_sets:
            hib = host_inbox(kind, w, step, prev, cols, gids, flags, fill=POISON)
            din = device_inbox(kind, w, step, dprev, cols, dev, gids_d, flags)
            assert_inbox_equal(hib, din, f"{shape}, step {k}, columns {cols}")
            if seen is not None:
                seen["ops"] |= op_kinds(hib)
                seen["events"] |= event_tags(hib)

    def over(w):
        return workload._over(w, gids)[0]

    prev = None
    if kind != "vote":                                  # the leader and mixed streams start from elected leaders
        w1 = over(workload.make_wl(seed, 1, G, F, gid_base=gid_base, local_slot=local_slot))
        for ph in (0, 1, 2):
            if kind == "election":
                check(ph, w1, ph, prev)
            prev = o.step(host_inbox("election", w1, ph, prev, LEADER_COLS, gids, abi.INBOX_NO_REQUESTS | lflag))
        if kind == "election":
            return
        prev = None
    w = over(workload.make_wl(seed, rows, G, F, gid_base=gid_base, local_slot=local_slot))
    steps = {"leader": 4, "vote": 6, "mixed": -(-144 // rows) + 1}[kind]
    at = set(range(steps)) if kind == "leader" else {0, steps // 2, steps - 2, steps - 1}
    for k in range(steps):
        if k in at:
            check(k, w, k, prev)
        prev = o.step(host_inbox(kind, w, k, prev, col_sets[0], gids, flags))
    o.close()


def new_seen():
    return {"ops": set(), "events": set()}


@pytest.mark.parametrize("gid_base", GID_BASES)
@pytest.mark.parametrize("F", (1, 2, 4))
def test_leader_generator_matches_host(dev, F, gid_base):
    """rafting_wl_leader_step on the device == on the host, with op_ab present and absent (the bench's unavail=False)."""
    seen = new_seen()
    for n in SHAPES_N:
        for rows in SHAPES_ROWS:
            check_stream("leader", F, n, rows, gid_base, dev, col_sets=(LEADER_COLS, BENCH_COLS), seen=seen)
    assert {abi.OP_SUBMIT, abi.OP_TIMEOUT} <= seen["ops"]
    outcomes = {(k, oc) for k, oc, _ in seen["events"]}
    assert {(abi.EV_AE_ACK, abi.OUT_OK), (abi.EV_AE_ACK, abi.OUT_ERROR), (abi.EV_AE_ACK, abi.OUT_CANCELED)} <= outcomes
    assert {f for _, _, f in seen["events"]} == set(range(F))


@pytest.mark.parametrize("gid_base", GID_BASES)
@pytest.mark.parametrize("F", (1, 2, 4))
def test_election_generator_matches_host(dev, F, gid_base):
    """rafting_wl_election_step, phases 0 (no previous outbox), 1 and 2."""
    seen = new_seen()
    for n in SHAPES_N:
        check_stream("election", F, n, 1, gid_base, dev, seen=seen)
    assert {abi.OP_TIMEOUT, abi.OP_NONE} <= seen["ops"]
    assert {abi.EV_PV_REPLY, abi.EV_RV_REPLY} <= {k for k, _, _ in seen["events"]}


@pytest.mark.parametrize("gid_base", GID_BASES)
@pytest.mark.parametrize("F,local_slot", [(4, 2), (4, 0), (2, 1), (1, 0)])
def test_vote_generator_matches_host(dev, F, local_slot, gid_base):
    """rafting_wl_vote_step (config #3: R = 5 with local_slot 2 as the bench runs it, and other slots)."""
    seen = new_seen()
    for n in SHAPES_N:
        for rows in SHAPES_ROWS:
            check_stream("vote", F, n, rows, gid_base, dev, local_slot=local_slot, seen=seen)
    assert {abi.OP_NONE, abi.OP_TIMEOUT, abi.OP_PREVOTE_REQ, abi.OP_VOTE_REQ} <= seen["ops"]
    outcomes = {(k, oc) for k, oc, _ in seen["events"]}
    assert {(abi.EV_PV_REPLY, abi.OUT_OK), (abi.EV_RV_REPLY, abi.OUT_OK), (abi.EV_PV_REPLY, abi.OUT_ERROR)} <= outcomes


@pytest.mark.parametrize("gid_base", GID_BASES)
@pytest.mark.parametrize("F", (1, 2, 4))
def test_mixed_generator_matches_host(dev, F, gid_base):
    """rafting_wl_mixed_step with the entry pool and op_cd / op_e, ~144 ticks into the stream: churn step-downs and follower
    AppendEntries, re-elections, FLUSH and, at F > 1, the catch-up class's lane-1 error rewrite."""
    seen = new_seen()
    for n in SHAPES_N:
        for rows in SHAPES_ROWS:
            check_stream("mixed", F, n, rows, gid_base, dev, seen=seen)
    assert {abi.OP_NONE, abi.OP_SUBMIT, abi.OP_TIMEOUT, abi.OP_AE_REQUEST, abi.OP_FLUSH} <= seen["ops"]
    kinds = {k for k, _, _ in seen["events"]}
    assert {abi.EV_AE_ACK, abi.EV_PV_REPLY, abi.EV_RV_REPLY} <= kinds
    if F > 1:
        assert (abi.EV_AE_ACK, abi.OUT_ERROR, 1) in seen["events"]


@pytest.mark.parametrize("listed", ["gids", "compact"])
@pytest.mark.parametrize("kind", ["leader", "election", "vote", "mixed"])
def test_generators_over_an_active_list(dev, kind, listed):
    """The gid / lgid branches of every cell: an active list, its group columns read by gid or (RAFTING_INBOX_COMPACT_GROUPS)
    by position."""
    seen = new_seen()
    for F in (2, 4):
        for n in (1, 255, 257, 4096):
            for rows in ((1,) if kind == "election" else (1, 16)):
                check_stream(kind, F, n, rows, 0, dev, listed=listed, local_slot=2 if kind == "vote" and F == 4 else 0, seen=seen)
    assert len(seen["ops"]) >= 2 and seen["events"]


@pytest.mark.parametrize("capacity", [workload.POOL_TERMS, workload.POOL_TERMS + 77])
def test_term_pool_matches_host(dev, capacity):
    """rafting_wl_fill_term_pool: the same 256 x 50 terms, nothing written past them."""
    import torch
    host = np.full(capacity, np.frombuffer(bytes([POISON]) * 8, np.int64)[0], dtype=np.int64)
    assert workload._bind().rafting_wl_fill_term_pool(host.ctypes.data, capacity, 0, None) == 0
    d = torch.full((capacity * 8,), POISON, dtype=torch.uint8, device=dev)
    assert workload._bind().rafting_wl_fill_term_pool(C.c_void_p(d.data_ptr()), capacity, 1, None) == 0
    sync()
    assert np.array_equal(d.cpu().numpy().view(np.int64), host)
    assert np.array_equal(host[:workload.POOL_TERMS], np.arange(workload.POOL_TERMS) // 50)


# ---- outboxes and states at the bench's shape --------------------------------------------------------------------------
def outbox_digest(ob):
    """Per-column hashes of an outbox under abi.Outbox.equal's rule: a payload cell whose meta marks it invalid counts as 0."""
    pm = (ob.plan_meta & np.uint64(0xF)) != 0
    masks = {"rep_term": (ob.rep_meta & 1) != 0, "plan_pp": pm, "plan_lc": pm, "plan_epoch": pm,
             "ballot_term": ob.ballot_meta != 0, "ballot_last": ob.ballot_meta != 0}
    out = {}
    for name, *_ in abi.Outbox.ROW_COLS + abi.Outbox.GROUP_COLS:
        a = np.ascontiguousarray(getattr(ob, name))
        b = a.view(np.uint8).reshape(a.shape + (-1,))
        if name in masks:
            b = b.copy()
            b[~masks[name]] = 0
        out[name] = hashlib.sha256(b).hexdigest()
    return out


def assert_digest_equal(want, got, where):
    bad = [name for name in want if want[name] != got[name]]
    assert not bad, f"outbox column(s) {bad} differ {where}"


FNV_OFFSET, FNV_PRIME = np.uint64(0xCBF29CE484222325), np.uint64(0x100000001B3)


def state_digest(states):
    """rafting_state_digest restated: FNV-1a 64 over each group's used state bytes (a [groups, bytes] uint8 array),
    vectorised across groups."""
    h = np.full(len(states), FNV_OFFSET, dtype=np.uint64)
    for b in range(states.shape[1]):
        h ^= states[:, b]
        h *= FNV_PRIME
    return h


def state_matrix(states, F):
    """[groups, used bytes] of exported group states, through harness.state_bytes."""
    rows = [harness.state_bytes(st, F) for st in states]
    return np.frombuffer(b"".join(rows), dtype=np.uint8).reshape(len(rows), -1)


def assert_shard_state(o, e, G, F, where):
    """The engine's whole shard against the oracle's: export_bulk byte for byte, and Engine.digest against the restated
    digest of the oracle's states."""
    want = state_matrix([o.export(g) for g in range(G)], F)
    got_states = e.export_bulk(0, G)
    got = state_matrix(got_states, F)
    bad = np.flatnonzero((want != got).any(axis=1))
    if len(bad):
        g = int(bad[0])
        da, db = o.export(g).as_dict(), got_states[g].as_dict()
        raise AssertionError(f"{len(bad)} group states differ {where}; group {g}: { {k: (da[k], db[k]) for k in da if da[k] != db[k]} }")
    digest = e.digest(0, G)
    restated = state_digest(want)
    bad = np.flatnonzero(digest != restated)
    assert not len(bad), f"rafting_state_digest differs from FNV-1a over the state bytes {where} in {len(bad)} groups, first {bad[0]}"
    return want


def bench_defaults(monkeypatch):
    import bench
    monkeypatch.setattr(sys, "argv", ["bench.py"])
    return bench, bench.parse()


def run_bench_window(monkeypatch, dev, tmp_path, *, G, gid_base, seed, launches, per_launch, comm):
    """bench.py run_engine's device path, launch for launch, against the oracle driven by the host generators."""
    import torch
    from rafting_b200 import devbatch, engine
    bench, args = bench_defaults(monkeypatch)
    R, rows = args.replicas, args.rows
    F = R - 1
    cfg = abi.make_cfg(replicas=R, max_groups=G, max_rows=rows, device=0)
    e, o = engine.Engine(cfg), binding.Oracle(cfg)
    init = bench_init(G, gid_base)
    e.open_bulk(0, init)
    o.open_bulk(0, init)
    if comm:
        e.comm_init(0, 1, None)                      # before anything else, so the checkpoint sees the bench's allocations
    stream = e.stream()
    w1 = workload.make_wl(seed, 1, G, F, gid_base=gid_base)
    w = workload.make_wl(seed, rows, G, F, gid_base=gid_base)

    def leader_host(k, prev):
        ib = workload.leader_inbox_host(w, k, prev)
        ib.op_ab = None                              # nobody unavailable: the column is absent, as in the bench's inboxes
        return ib

    # ---- the election, on the device through one reused inbox and outbox ----
    in1, out1 = devbatch.DevInbox(1, G, F, dev), devbatch.DevOutbox(1, G, F, G, dev)
    prev_c, oprev = None, None
    for ph in (0, 1, 2):
        ic = in1.as_c()
        workload.election_step(w1, ph, prev_c, ic, on_device=True, stream=stream)
        oc = out1.as_c()
        e.step_device(ic, oc, stream)
        prev_c = oc
        hib = workload.election_inbox_host(w1, ph, oprev)
        oprev = o.step(hib, threads=ORACLE_THREADS)
        sync()
        assert_inbox_equal(hib, in1, f"election phase {ph}", written_only=True)
        harness.assert_outbox_equal(oprev, out1.to_host(), where=f"at election phase {ph}")
    assert_shard_state(o, e, G, F, "after the election")

    # ---- settle: one reused inbox, two rotating outboxes ----
    outs = [devbatch.DevOutbox(rows, G, F, G, dev) for _ in range(2)]
    inboxes = [devbatch.DevInbox(rows, G, F, dev, unavail=False) for _ in range(launches)]
    assert inboxes[0].nbytes() == bench.inbox_bytes_per_launch(G, rows, F)
    settle = devbatch.DevInbox(rows, G, F, dev, unavail=False)
    prev_out, oprev = None, None
    for k in range(SETTLE):
        ic = settle.as_c()
        workload.leader_step(w, k, None if prev_out is None else prev_out.as_c(), ic, on_device=True, stream=stream)
        prev_out = outs[k % 2]
        e.step_device(ic, prev_out.as_c(), stream)
        hib = leader_host(k, oprev)
        oprev = o.step(hib, threads=ORACLE_THREADS)
        sync()
        assert_inbox_equal(hib, settle, f"settle launch {k}", written_only=True)
        harness.assert_outbox_equal(oprev, prev_out.to_host(), where=f"at settle launch {k}")
    start_out = devbatch.DevOutbox(rows, G, F, G, dev)
    for name in start_out.t:
        start_out.t[name].copy_(prev_out.t[name])
    sync()
    assert_shard_state(o, e, G, F, "after settling")
    e.checkpoint()

    # ---- the recorded window: distinct inboxes ----
    prev_out, want = start_out, []
    for k in range(launches):
        ic = inboxes[k].as_c()
        workload.leader_step(w, SETTLE + k, prev_out.as_c(), ic, on_device=True, stream=stream)
        prev_out = outs[k % 2]
        e.step_device(ic, prev_out.as_c(), stream)
        hib = leader_host(SETTLE + k, oprev)
        oprev = o.step(hib, threads=ORACLE_THREADS)
        sync()
        assert_inbox_equal(hib, inboxes[k], f"recorded launch {k}")
        harness.assert_outbox_equal(oprev, prev_out.to_host(), where=f"at recorded launch {k}")
        if k < per_launch or k >= launches - 2:
            want.append(outbox_digest(oprev))
        else:
            want.append(None)
    del start_out
    final = assert_shard_state(o, e, G, F, "at the end of the recording")
    last_oracle = oprev

    # ---- the timed replay, twice: restore(sync=False) + one step_device_seq over the window ----
    ics = (abi.InboxC * launches)(*[ib.as_c() for ib in inboxes])
    ocs = (abi.OutboxC * launches)(*[outs[k % 2].as_c() for k in range(launches)])
    for rep in range(2):
        e.restore(sync=False)
        e.step_device_seq(ics, ocs, launches, gather=False, stream=0)
        sync()
        for k in (launches - 2, launches - 1):
            assert_digest_equal(want[k], outbox_digest(outs[k % 2].to_host()), f"at launch {k} of replay {rep}")
        again = assert_shard_state(o, e, G, F, f"after replay {rep}")
        assert np.array_equal(again, final)

    # ---- per-launch replay of the first launches into distinct poisoned outboxes (multi-wave programmatic launches) ----
    K = min(per_launch, launches)
    pouts = [devbatch.DevOutbox(rows, G, F, G, dev, fill=POISON) for _ in range(K)]
    free, total = torch.cuda.mem_get_info()
    print(f"\nbench window G={G} launches={launches}: {(total - free) / 1e9:.1f} GB of HBM in use on the device")
    e.restore(sync=False)
    e.step_device_seq(ics, (abi.OutboxC * K)(*[p.as_c() for p in pouts]), K, gather=False, stream=0)
    sync()
    for k in range(K):
        assert_digest_equal(want[k], outbox_digest(pouts[k].to_host()), f"at launch {k} of the per-launch replay")
    del pouts

    # ---- --dump-outputs of the last launch: the engine's outbox and the oracle's give the same files ----
    e.restore(sync=False)
    e.step_device_seq(ics, ocs, launches, gather=False, stream=0)
    sync()
    oracle_box = types.SimpleNamespace(t={name: torch.from_numpy(np.ascontiguousarray(getattr(last_oracle, name)).view(np.uint8).reshape(-1))
                                          for name, *_ in abi.Outbox.ROW_COLS + abi.Outbox.GROUP_COLS})
    bench.dump_outputs(str(tmp_path / "engine"), outs[(launches - 1) % 2], rows, G, F)
    bench.dump_outputs(str(tmp_path / "oracle"), oracle_box, rows, G, F)
    names = sorted(p.name for p in (tmp_path / "engine").iterdir())
    assert names == sorted(p.name for p in (tmp_path / "oracle").iterdir()) and "commit_index.npy" in names
    for name in names:
        assert (tmp_path / "engine" / name).read_bytes() == (tmp_path / "oracle" / name).read_bytes(), name
    e.close()
    o.close()
    del inboxes, outs, settle, in1, out1
    torch.cuda.empty_cache()


def test_config2_bench_window_launch_by_launch(monkeypatch, dev, tmp_path):
    """config #2 exactly as bench.py times it: 64 K groups, R = 3, 16 rows, a 128-launch window, each pair_kernel grid
    several waves deep, so launch k+1's blocks stage their rows while launch k's last wave runs."""
    bench, args = bench_defaults(monkeypatch)
    G = bench.G_CONFIG2
    L = bench.window_launches(args, G)
    assert L == 128
    run_bench_window(monkeypatch, dev, tmp_path, G=G, gid_base=0, seed=bench.SEED2, launches=L, per_launch=32, comm=True)


def test_config4_shard_on_one_gpu(monkeypatch, dev, tmp_path):
    """Rank 5 of config #4 at 8 GPUs: 128 K groups from gid 5 x 128 K, SEED4, a 16-launch window."""
    bench, _ = bench_defaults(monkeypatch)
    G = bench.G_CONFIG4 // 8
    run_bench_window(monkeypatch, dev, tmp_path, G=G, gid_base=5 * G, seed=bench.SEED4, launches=16, per_launch=16, comm=False)


# ---- 4. bench_secondary's closed loops -----------------------------------------------------------------------------
@pytest.mark.parametrize("config", ["config3", "config5"])
def test_bench_secondary_closed_loop(dev, config):
    """tools/bench_secondary.run at reduced size: one reused DevInbox(requests=True), the device pool, for #5 the device
    election, prev reset to None, and a checkpoint / restore between the two passes.  Every step's outbox against the
    oracle's, and both passes end in the oracle's state."""
    import torch
    from rafting_b200 import devbatch, engine
    if config == "config3":
        G, R, rows, steps, seed, kind, local_slot, elect, pool = 16384, 5, 1, 8, SEED3, "vote", 2, False, False
    else:
        G, R, rows, steps, seed, kind, local_slot, elect, pool = 32768, 3, 4, 35, SEED5, "mixed", 0, True, True
    F = R - 1
    cfg = abi.make_cfg(replicas=R, local_slot=local_slot, max_groups=G, max_rows=rows, pre_vote=True,
                       entry_pool_cap=workload.POOL_TERMS if pool else 0)
    e, o = engine.Engine(cfg), binding.Oracle(cfg)
    if config == "config3":
        init = harness.init_array(G, terms=1 + np.arange(G) % 5)
        init["last_index"] = 100 + np.arange(G) % 50
        init["last_term"] = 1 + np.arange(G) % 5
    else:
        init = harness.init_array(G, terms=np.arange(G) % 7)
    e.open_bulk(0, init)
    o.open_bulk(0, init)
    stream = e.stream()
    ob = [devbatch.DevOutbox(rows, G, F, G, dev) for _ in range(2)]
    ib = devbatch.DevInbox(rows, G, F, dev, requests=True)
    pool_t = None
    if pool:
        pool_t = torch.zeros(workload.POOL_TERMS, dtype=torch.int64, device=dev)
        assert workload._bind().rafting_wl_fill_term_pool(C.c_void_p(pool_t.data_ptr()), workload.POOL_TERMS, 1, C.c_void_p(stream)) == 0
    if elect:
        w1 = workload.make_wl(seed, 1, G, F, local_slot=local_slot)
        ib1 = devbatch.DevInbox(1, G, F, dev, requests=False)
        ob1 = [devbatch.DevOutbox(1, G, F, G, dev) for _ in range(2)]
        prev, oprev = None, None
        for ph in (0, 1, 2):
            workload.election_step(w1, ph, prev, ib1.as_c(), on_device=True, stream=stream)
            oc = ob1[ph & 1].as_c()
            e.step_device(ib1.as_c(), oc, stream)
            prev = oc
            oprev = o.step(workload.election_inbox_host(w1, ph, oprev), threads=ORACLE_THREADS)
            sync()
            harness.assert_outbox_equal(oprev, ob1[ph & 1].to_host(), where=f"{config}: election phase {ph}")
    w = workload.make_wl(seed, rows, G, F, local_slot=local_slot)
    host = workload.vote_inbox_host if kind == "vote" else workload.mixed_inbox_host
    e.checkpoint()
    want, ends = [], []
    oprev = None
    for p in (0, 1):
        if p:
            e.restore()
        prev = None
        for k in range(steps):
            ic = ib.as_c()
            if pool:
                ic.ent_terms, ic.ent_count = pool_t.data_ptr(), workload.POOL_TERMS
            generate(kind, w, k, prev, ic, True, stream)
            oc = ob[k & 1].as_c()
            e.step_device(ic, oc, stream)
            prev = oc
            if p == 0:
                hib = host(w, k, oprev)
                oprev = o.step(hib, threads=ORACLE_THREADS)
            sync()
            got = ob[k & 1].to_host()
            if p == 0:
                assert_inbox_equal(hib, ib, f"{config}: step {k}", written_only=True)
                harness.assert_outbox_equal(oprev, got, where=f"{config}: step {k}")
                want.append(outbox_digest(oprev))
            else:
                assert_digest_equal(want[k], outbox_digest(got), f"{config}: step {k} of the second pass")
        ends.append(assert_shard_state(o, e, G, F, f"{config}: after pass {p}"))
    assert np.array_equal(ends[0], ends[1])
    e.close()
    o.close()
