"""rafting_log_gather_step_begin / _wait: the payloads of a compact step's AppendEntries plans, gathered on the device.

Every gather is held to the host path a pump would otherwise take: the step's AE ranges decoded from rafting_step_fetch_dense in
lane-slot order, then rafting_log_gather over them.  The refs must agree field by field (gid, index, term, len), every payload
byte for byte, and the plan records must be the decoded plans.  Before each gather the entries the step created get payloads of
random length (zero-length ones included), as a pump appends the payloads of its SUBMITs after the wait."""
import ctypes as C

import numpy as np
import pytest

from rafting_b200 import abi, compact, engine, workload
from tests import edit_pump
from tests import harness
from tests import timers_model as tm

pytestmark = pytest.mark.gpu


def dense_ranges(e: engine.Engine, slot: int, rows: int, n: int, gids):
    """(lane slots, gids, first indices, counts) of the AE plans with entries of the step last waited for in slot"""
    d = abi.Outbox(rows, n, e.F, n)
    e.step_fetch_dense(slot, d.as_c())
    m = d.plan_meta.reshape(-1)
    c = np.where((m & 0xF) == abi.PLAN_AE, (m >> 16) & 0xFFFF, 0).astype(np.int64)
    t = np.flatnonzero(c)
    pos = (t // e.F) % n
    g = pos if gids is None else np.asarray(gids, np.int64)[pos]
    return t, g, d.plan_pp.reshape(-1)["x"][t] + 1, c[t]


_PINNED = []                                       # the pinned tensors behind the views pinned() hands out


def pinned(nbytes: int, dtype) -> np.ndarray:
    import torch
    t = torch.zeros(max(nbytes, 16), dtype=torch.uint8, pin_memory=True)
    _PINNED.append(t)
    return t.numpy()[:nbytes].view(dtype)


def with_submits(peers: tm.Peers, share: float = 0.05):
    """tests/timers_model's stream carries heartbeats and elections only: add SUBMITs of 1..3 commands in the last row of a
    share of the groups, so that the leaders among them plan AppendEntries with entries"""
    inbox = peers.inbox

    def wrapped(k, planned, terms):
        ib = inbox(k, planned, terms)
        rng = np.random.default_rng(50_000 + k)
        r = ib.rows - 1
        for g in np.flatnonzero((rng.random(ib.n) < share) & (ib.op_meta[r] == 0)).tolist():
            ib.submit(r, g, peers.now(k), count=1 + g % 3)
        return ib
    peers.inbox = wrapped


class Payloads:
    """The pump's side: payloads for the entries a step created, and every gather held to rafting_log_gather."""

    def __init__(self, e: engine.Engine, seed: int = 7, max_len: int = 4096, small: float = 0.9):
        self.e, self.rng, self.max_len, self.small = e, np.random.default_rng(seed), max_len, small
        self.last = {}
        self.refs = self.plans = self.served = self.absent = 0

    def payload(self) -> bytes:
        r = self.rng.random()
        if r < 0.1:
            return b""
        cap = 256 if r < self.small else self.max_len
        return self.rng.bytes(int(self.rng.integers(1, cap + 1)))

    def append_created(self, cout: compact.CompactOutbox, gids, keep: int = 8):
        """entries up to last_entry of each listed group that were not appended yet (the newest `keep` of a longer run)"""
        g = np.arange(cout.n) if gids is None else np.asarray(gids, np.int64)
        hi = cout.last_entry["x"]
        ents = []
        for i in np.flatnonzero(hi > 0):
            gid, h = int(g[i]), int(hi[i])
            lo = max(self.last.get(gid, 0), h - keep)
            ents += [(gid, x, int(cout.current_term[i]), self.payload()) for x in range(lo + 1, h + 1)]
            self.last[gid] = max(h, self.last.get(gid, 0))
        if ents:
            self.e.log_append(ents)

    def check(self, slot: int, rows: int, n: int, gids, where: str, pin: bool = False):
        t, g, f, c = dense_ranges(self.e, slot, rows, n, gids)
        want, cap = [], 1 << 24
        while len(t):
            try:
                want = self.e.log_gather(list(zip(g.tolist(), f.tolist(), c.tolist())), blob_cap=cap)
                break
            except engine.RaftingError as ex:
                if ex.rc != -5:
                    raise
                cap *= 4
        if pin:
            nr, np_ = max(int(c.sum()), 1), max(len(t), 1)
            refs, plans = pinned(nr * 32, self.e.ENTRY_REF), pinned(np_ * 16, abi.PLAN_REF)
            blob = pinned(max(cap, 1 << 20), np.uint8)
            self.e.log_gather_step_begin(slot, refs, blob, plans)
            n_refs, _, n_plans, served = self.e.log_gather_step_wait(slot)
            got, pl = self.e._gathered(refs[:n_refs], blob), plans[:n_plans]
        else:
            got, pl, served = self.e.log_gather_step(slot, blob_cap=cap)
        assert len(got) == len(want), f"{where}: {len(got)} refs, rafting_log_gather {len(want)}"
        bad = [k for k, (a, b) in enumerate(zip(got, want)) if a != b]
        assert not bad, f"{where}: ref {bad[0]} {got[bad[0]][:3]} != {want[bad[0]][:3]} ({len(bad)} differ)"
        assert np.array_equal(pl["slot"], t) and np.array_equal(pl["count"], c), where
        assert np.array_equal(pl["first"], np.concatenate([[0], np.cumsum(c)[:-1]]) if len(c) else []), where
        self.refs += len(got)
        self.plans += len(t)
        self.served += served
        self.absent += sum(1 for x in got if x[3] is None)
        return served, got


def leader_engines(R: int, G: int, rows: int, seed: int, configure: bool = True, **log):
    cfg = abi.make_cfg(replicas=R, max_groups=G, max_rows=rows)
    ref, e = engine.Engine(cfg), engine.Engine(cfg)
    init = harness.init_array(G, terms=np.arange(G) % 7)
    ref.open_bulk(0, init)
    e.open_bulk(0, init)
    if configure:
        e.log_config(**(log or dict(segment_bytes=1 << 20, hbm_segments=64, ring_slots=64)))
    w1 = workload.make_wl(seed, 1, G, R - 1)
    for sut in (ref, e):
        last = harness.elect_all(sut, w1)
    return ref, e, workload.make_wl(seed, rows, G, R - 1), last


def run_leader(R, flags, shapes, steps=6, G=2048, rows=4, seed=0x5EED0002, pin=False, log=None, pay=None):
    """the leader stream of a dense reference, stepped by the engine under test as compact steps of the given shapes"""
    ref, e, w, last = leader_engines(R, G, rows, seed, **(log or {}))
    P = pay(e) if pay else Payloads(e, seed=R * 16 + flags)
    rng = np.random.default_rng(seed)
    for k in range(steps):
        ib = workload.leader_inbox_host(w, k, last)
        last = ref.step(ib)
        shape = shapes[k % len(shapes)]
        gids = None if shape == "whole" else np.sort(rng.choice(G, G // 3, replace=False)).astype(np.uint32)
        ci = compact.encode_inbox(ib if gids is None else tm.slice_inbox(ib, gids), None, None, None)
        cout = compact.CompactOutbox(rows, G if gids is None else len(gids), R - 1, esc_cap=rows * G * R, gids=gids)
        e.step_compact(ci, cout, flags=flags)
        P.append_created(cout, gids)
        P.check(0, rows, cout.n, gids, f"R={R} flags={flags} step {k} ({shape})", pin=pin and k % 2 == 1)
    return P, e


@pytest.mark.parametrize("R", [3, 5])
@pytest.mark.parametrize("flags", [0, 1, 4, 5])
def test_leader_stream_whole_and_active(R, flags):
    P, _ = run_leader(R, flags, ["whole", "active"])
    assert P.refs > 0 and P.plans > 0


def test_multi_row_prev_term_and_pinned_outputs():
    # the first compact steps carry no tags: their AE plans travel as escape records; later ones as words of kind 1 / 7
    P, _ = run_leader(3, abi.COMPACT_PREV_TERM, ["whole"], steps=8, rows=8, pin=True)
    assert P.refs > 0


def test_peers_stream_sweep_and_active_steps():
    """Whole-shard, active, whole-shard sweep and active sweep steps over tests/timers_model's 3-node stream (heartbeats,
    elections after a lost peer), flags cycling through 0, 1, 4 and 5."""
    G, rows = 4096, 3
    cfg = edit_pump.make_cfg(G)
    ref, e = engine.Engine(cfg), engine.Engine(cfg)
    init = edit_pump.init_all(G)
    ref.open_bulk(0, init)
    e.open_bulk(0, init)
    e.log_config(segment_bytes=1 << 20, hbm_segments=32, ring_slots=64)
    peers = tm.Peers(G, rows=rows, lost_at=20, t0=workload.T0_MS)
    with_submits(peers)
    pay = Payloads(e, seed=11)
    wants, terms = [], init["term"].astype(np.int64)
    shapes = ["whole", "active", "sweep", "active-sweep"]
    for k in range(48):
        ib = peers.inbox(k, wants[k - peers.DELAY] if k >= peers.DELAY else None, terms)
        want = ref.step(ib)
        wants.append(want)
        terms = want.current_term.copy()
        shape, flags = shapes[k % 4], (0, 1, 4, 5)[(k // 4) % 4]
        gids = tm.event_gids(ib).astype(np.uint32) if "active" in shape else None
        if gids is not None and len(gids) == 0:
            gids = np.arange(8, dtype=np.uint32)
        sib = ib if gids is None else tm.slice_inbox(ib, gids)
        ci = compact.encode_inbox(sib, None, None, None, sweep="sweep" in shape)
        n = G if gids is None else len(gids)
        cout = compact.CompactOutbox(rows, n, 2, esc_cap=rows * n * 2 + 2 * rows * n, gids=gids)
        e.step_compact(ci, cout, flags=flags)
        pay.append_created(cout, gids)
        pay.check(0, rows, n, gids, f"tick {k} ({shape}, flags {flags})")
    assert pay.plans > 0


@pytest.mark.parametrize("k_edits", [0, 256])
def test_due_pump_closed_loop(k_edits):
    """The 64 K x 3 due pump at d = 3; its on_wait hook appends the payloads and gathers, for plans from host-listed and
    device-chosen tail positions alike (and, with edits, for groups restarted by rafting_group_edit_begin)."""
    S = edit_pump.Stream(k_edits, every=10, first=5)
    with_submits(S.P)
    pump = edit_pump.DuePump(S, 3, "edit")
    pump.e.log_config(segment_bytes=1 << 22, hbm_segments=64, ring_slots=64)
    pay = Payloads(pump.e, seed=5, small=0.97)
    tails = []

    def on_wait(j, cout):
        pay.append_created(cout, cout.gids, keep=4)
        _, got = pay.check(j % 4, edit_pump.ROWS, cout.n, cout.gids, f"due tick {j}")
        tails.append(int(cout.counts[3]))

    pump.run(36 if k_edits else 170, on_wait=on_wait)             # without edits the node leads groups only after tick 150
    assert pay.plans > 0 and max(tails) > 0


def test_host_served_entries(tmp_path):
    """A ring of 4 slots, an arena of 4 segments spilling to a pinned pool of 2 segments over an entry file, and never-appended
    indices: the results still match, and host_served counts the entries the ring does not hold."""
    log = dict(segment_bytes=1 << 16, hbm_segments=4, ring_slots=4)

    class Spilling(Payloads):
        def __init__(self, e):
            e.log_store_open(str(tmp_path / "entries.log"), cold_max_segments=2)
            super().__init__(e, seed=3, max_len=2048)

        def append_created(self, cout, gids, keep=8):
            super().append_created(cout, gids, keep=3)        # older indices of a longer run stay never appended

    P, e = run_leader(3, 0, ["whole"], steps=6, G=512, log=log, pay=Spilling)
    st, fs = e.log_stats(), e.log_store_stats()
    assert P.served > P.absent > 0, (P.served, P.absent)
    assert st["spilled_bytes"] > 0 and (st["cold_hits"] + fs["file_hits"]) > 0
    # a roomy buffer holds every appended entry in the ring: only never-appended ones are served by the host
    P2, _ = run_leader(3, 0, ["whole"], steps=4, G=512, pay=lambda e: Payloads(e, seed=3, max_len=512))
    assert P2.served == P2.absent


def _one_step(G=1024, rows=2, log=True):
    """an engine after one compact leader step with AE plans (the second of the stream), and that step's outbox"""
    ref, e, w, last = leader_engines(3, G, rows, 0x5EED0002, configure=log)
    for k in range(2):
        ib = workload.leader_inbox_host(w, k, last)
        last = ref.step(ib)
        cout = compact.CompactOutbox(rows, G, 2, esc_cap=rows * G * 3)
        if k == 0:
            e.step_compact(compact.encode_inbox(ib, None, None, None), cout)
    return e, ib, cout


def test_refusals_and_lifetime():
    e, ib, cout = _one_step()
    refs, blob, plans = np.zeros(1 << 19, e.ENTRY_REF), np.zeros(1 << 26, np.uint8), np.zeros(1 << 14, abi.PLAN_REF)
    with pytest.raises(engine.RaftingError, match="E_INVAL"):                # no compact step in the slot yet
        e.log_gather_step_begin(1, refs, blob, plans)
    e.step_compact(compact.encode_inbox(ib, None, None, None), cout)
    P = Payloads(e, seed=1)
    P.append_created(cout, None)
    t, g, f, c = dense_ranges(e, 0, 2, 1024, None)
    assert len(t) > 0
    e.log_gather_step_begin(0, refs, blob, plans)
    with pytest.raises(engine.RaftingError, match="E_BUSY"):                 # one gather per slot
        e.log_gather_step_begin(0, refs, blob, plans)
    with pytest.raises(engine.RaftingError, match="E_BUSY"):                 # the slot's plans stay put until the wait
        e.step_begin_compact_ex(0, compact.encode_inbox(ib, None, None, None).as_c(), None, cout.as_c(), 0)
    with pytest.raises(engine.RaftingError, match="E_BUSY"):                 # so does the entry buffer's host index
        e.log_append([(0, 10**6, 1, b"x")])
    n, nb, npl, _ = e.log_gather_step_wait(0)
    assert n == int(c.sum()) and npl == len(t)
    with pytest.raises(engine.RaftingError, match="E_INVAL"):                # nothing in flight any more
        e.log_gather_step_wait(0)
    first = e._gathered(refs[:n], blob)
    # caps one too small: E_CAPACITY with the sizes needed, nothing past the caps written; a retry succeeds
    for rc_, bc_, pc_ in ((n - 1, nb, npl), (n, nb - 1, npl), (n, nb, npl - 1)):
        r2, b2, p2 = np.zeros(n, e.ENTRY_REF), np.full(nb + 64, 0xAB, np.uint8), np.zeros(npl + 1, abi.PLAN_REF)
        p2["slot"][-1] = 0xFFFFFFFF
        e.log_gather_step_begin(0, r2, b2, p2, refs_cap=rc_, blob_cap=bc_, plans_cap=pc_)
        with pytest.raises(engine.RaftingError, match="E_CAPACITY") as ex:
            e.log_gather_step_wait(0)
        assert ex.value.sizes[:3] == (n, nb, npl)
        assert (b2[bc_:] == 0xAB).all() and p2["slot"][pc_:].max() in (0, 0xFFFFFFFF) and p2["slot"][-1] == 0xFFFFFFFF
        if rc_ < n:
            assert r2[rc_:]["index"].max() == 0
    e.log_gather_step_begin(0, refs, blob, plans)
    assert e.log_gather_step_wait(0)[:3] == (n, nb, npl)
    assert e._gathered(refs[:n], blob) == first
    # the same through pinned outputs, written by the device directly
    pr, pb, pp = pinned(n * 32, e.ENTRY_REF), pinned(nb, np.uint8), pinned(npl * 16, abi.PLAN_REF)
    e.log_gather_step_begin(0, pr, pb, pp)
    assert e.log_gather_step_wait(0)[:3] == (n, nb, npl)
    assert e._gathered(pr, pb) == first and np.array_equal(pp, plans[:npl])
    # without an entry buffer
    e2, ib2, cout2 = _one_step(log=False)
    e2.step_compact(compact.encode_inbox(ib2, None, None, None), cout2)
    with pytest.raises(engine.RaftingError, match="E_INVAL"):
        e2.log_gather_step_begin(0, refs, blob, plans)


def test_gather_step_natives_through_the_jni_glue(tmp_path):
    from tests import jni_exec
    from tests.jni_exec import Buf, buf_of_array, fn
    L = jni_exec.build(str(tmp_path))
    if L is None:
        pytest.skip("no gcc")
    e, ib, cout = _one_step()
    e.step_compact(compact.encode_inbox(ib, None, None, None), cout)
    Payloads(e, seed=2).append_created(cout, None)
    want, want_plans, _ = e.log_gather_step(0)
    L.fake_reset()
    begin = fn(L, "logGatherStepBegin", None, C.c_int64, C.c_int32, C.POINTER(Buf), C.c_int32, C.POINTER(Buf), C.c_int64,
               C.POINTER(Buf), C.c_int32)
    wait = fn(L, "logGatherStepWait", None, C.c_int64, C.c_int32, C.POINTER(jni_exec.Longs))
    refs, blob, plans = np.zeros(len(want), e.ENTRY_REF), np.zeros(1 << 22, np.uint8), np.zeros(len(want_plans), abi.PLAN_REF)
    h = e._h if isinstance(e._h, int) else e._h.value
    begin(h, 0, C.byref(buf_of_array(refs)), len(refs), C.byref(buf_of_array(blob)), len(blob), C.byref(buf_of_array(plans)), len(plans))
    res = np.zeros(4, np.int64)
    wait(h, 0, C.byref(jni_exec.Longs(4, res.ctypes.data_as(C.POINTER(C.c_int64)))))
    assert L.fake_throws() == 0, L.fake_thrown_message()
    assert res[0] == len(want) and res[2] == len(want_plans)
    assert e._gathered(refs, blob) == want and np.array_equal(plans, want_plans)
