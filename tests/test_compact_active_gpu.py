"""Active lists on the compact host path (`-m gpu`): steps fed through rafting_step_begin_compact_active must equal the compact
model (tests/compact_active_model.py, the whole-shard model over the listed gids) bit for bit, decode to the oracle's dense
outbox, and leave every group of the shard, listed or not, in the oracle's state.  Tags follow the gid across active lists, whole-shard compact steps and dense steps;
bad lists are refused before anything is enqueued; the in-flight table survives rafting_state_save / load."""
import ctypes as C

import numpy as np
import pytest

from oracle import binding
from rafting_b200 import abi, compact, engine, workload
from tests import compact_active_model as active
from tests import compact_model as model
from tests import harness
from tests.compact_model import EL, PT, assert_step_reads_the_same, _sorted_esc

pytestmark = pytest.mark.gpu
U64 = np.uint64


def pick(G, n, seed):
    return np.sort(np.random.default_rng(seed).choice(G, n, replace=False)).astype(np.uint32)


def opened(G, R, rows, seed, storm=False):
    """The engine and the oracle at the same start: config #3 (storm) or elected leaders."""
    F = R - 1
    if storm:
        cfg, init, _ = model._storm_open(G, R, rows)
    else:
        cfg = abi.make_cfg(replicas=R, max_groups=G, max_rows=rows, entry_pool_cap=rows * G * 50)
        init = harness.init_array(G, terms=np.arange(G) % 7)
    e, o = engine.Engine(cfg), binding.Oracle(cfg)
    for s in (e, o):
        s.open_bulk(0, init)
    if not storm:
        w1 = workload.make_wl(seed, 1, G, F)
        harness.assert_outbox_equal(harness.elect_all(o, w1), harness.elect_all(e, w1), where="election (dense path)")
    return cfg, e, o


class Pump:
    """A compact pump around the engine and, beside it, the model, both checked against the oracle every step.  A step runs
    over an active list, the whole shard (None) or, for "dense", the dense host path over the whole shard."""

    def __init__(self, e, o, G, F, make, flags=0, empty_list=False):
        self.e, self.o, self.G, self.F, self.make, self.flags, self.empty_list = e, o, G, F, make, flags, empty_list
        self.st = model.InFlight(G, F)
        self.g_term = np.array([s.current_term for s in e.export_bulk(0, G)], np.int64)
        self.epoch = np.zeros(G, abi.I64X2)
        self.prev, self.nxt, self.frm, self.k = None, None, None, 0
        self.tagged_acks = 0

    def _epoch(self, gids):
        at = range(self.G) if gids is None else gids.tolist()
        for g in at:                                                    # pack reads the epoch of the listed groups only
            s = self.o.export(g)
            self.epoch[g] = (s.epoch_index, s.epoch_term)
        return self.epoch

    def step(self, gids, esc_cap=None, slot=0):
        G, F, k = self.G, self.F, self.k
        dense_step = isinstance(gids, str)
        to = None if dense_step else gids
        prev = None if self.prev is None else active.carry_outbox(self.prev, self.frm, to, G)
        ib = self.make(k, prev, to)
        want = self.o.step(ib, threads=8)
        self.k += 1
        if dense_step:                                                  # tags planned before stay taken (the reply came back dense)
            harness.assert_outbox_equal(want, self.e.step(ib), where=f"dense step {k}")
            self.g_term[:] = want.current_term
            self.prev, self.nxt, self.frm = want, None, None
            return want, None
        kept = None if self.nxt is None else active.carry(self.nxt, self.frm, gids, G)
        ci = model.encode(ib, kept, self.flags, empty_list=self.empty_list)
        assert_step_reads_the_same(ib, active.unpack(ci, self.g_term, self.st, self.flags, gids=gids), where=f"model unpack, step {k}")
        rows, n = ib.rows, ib.n
        cap = rows * n * F + 2 * rows * n if esc_cap is None else esc_cap
        mo = active.pack(want, self._epoch(gids), self.st, esc_cap=cap, flags=self.flags, replies=ci.reqs is not None, gids=gids)
        cout = compact.CompactOutbox(rows, n, F, esc_cap=cap, gids=gids)
        self.e.step_compact(ci, cout, slot=slot, reqs=ci.reqs, flags=self.flags)
        for name in compact.CompactOutbox.COLS:
            assert np.array_equal(getattr(cout, name), getattr(mo, name)), f"{name} differs from the model, step {k}"
        assert np.array_equal(cout.counts, mo.counts) and _sorted_esc(cout) == _sorted_esc(mo), f"escape records, step {k}"
        if kept is not None:                                            # an ack to a tagged plan never escapes
            ek = (ib.ev_meta & U64(0xF)).astype(np.int64) if ib.ev_meta is not None else np.zeros((rows, n, F), np.int64)
            tagged = ((ek == abi.EV_AE_ACK) | (ek == abi.EV_IS_ACK)) & (kept["tags"] < 32)
            assert np.array_equal((ci.ev_c[tagged] & np.uint32(0xF)).astype(np.int64), ek[tagged]), f"a tagged ack escaped, step {k}"
            self.tagged_acks += int(tagged.sum())
        if esc_cap is None:
            got = compact.decode_outbox(cout, elections=bool(self.flags & EL), prev_term=bool(self.flags & PT))
            harness.assert_outbox_equal(want, got, where=f"compact step {k}")
            self.prev = got
        else:
            self.prev = want
        self.g_term[np.arange(G) if gids is None else gids] = want.current_term[:n]
        self.nxt, self.frm = model.next_of(want, cout), gids
        return want, cout

    def assert_every_group_equal(self, e=None):
        got = (e or self.e).export_bulk(0, self.G)
        for g in range(self.G):
            assert harness.state_bytes(got[g], self.F) == harness.state_bytes(self.o.export(g), self.F), f"group {g}"


def leader_make(w):
    return lambda k, prev, gids: workload.leader_inbox_host(w, k, prev, gids=gids)


@pytest.mark.parametrize("n", [4096, 512])
def test_leader_stream_over_an_active_list(n):
    G, R, rows, seed = 65536, 3, 4, 0x5EED0002
    cfg, e, o = opened(G, R, rows, seed)
    p = Pump(e, o, G, R - 1, leader_make(workload.make_wl(seed, rows, G, R - 1)))
    A = pick(G, n, n)
    for _ in range(6):
        p.step(A)
    assert p.tagged_acks > n * rows
    p.assert_every_group_equal()


def test_config5_over_an_active_list_class_sorted():
    G, R, rows, seed = 16384, 3, 4, 0x5EED0005
    cfg, e, o = opened(G, R, rows, seed)
    w = workload.make_wl(seed, rows, G, R - 1)
    p = Pump(e, o, G, R - 1, lambda k, prev, gids: workload.mixed_inbox_host(w, k, prev, gids=gids), empty_list=True)
    A = pick(G, 4100, 6)
    for _ in range(8):
        p.step(A)
    p.assert_every_group_equal()


@pytest.mark.parametrize("flags", [EL, EL | PT])
def test_vote_storm_over_an_active_list(flags):
    G, R, rows = 16384, 5, 2
    cfg, e, o = opened(G, R, rows, 0, storm=True)
    _, _, w = model._storm_open(G, R, rows)
    p = Pump(e, o, G, R - 1, lambda k, prev, gids: workload.vote_inbox_host(w, k, prev, gids=gids), flags=flags)
    A = pick(G, 4000, 7)
    for _ in range(6):
        p.step(A)
    p.assert_every_group_equal()


def test_unsorted_launch_over_an_active_list():
    G, R, rows, seed = 1024, 5, 4, 0x5EED0005
    cfg, e, o = opened(G, R, rows, seed)
    w = workload.make_wl(seed, rows, G, R - 1)
    p = Pump(e, o, G, R - 1, lambda k, prev, gids: workload.mixed_inbox_host(w, k, prev, gids=gids), flags=EL | PT, empty_list=True)
    A = pick(G, 300, 8)
    for _ in range(8):
        p.step(A)
    p.assert_every_group_equal()


def test_active_whole_shard_and_dense_steps_mix_and_acks_follow_the_gid():
    G, R, rows, seed = 4096, 3, 2, 0x5EED0002
    cfg, e, o = opened(G, R, rows, seed)
    p = Pump(e, o, G, R - 1, leader_make(workload.make_wl(seed, rows, G, R - 1)))
    A = pick(G, 900, 9)
    B = np.union1d(A, pick(G, 700, 10)).astype(np.uint32)
    counts = []
    for k, gids in enumerate([A, B, None, A, "dense", B, A, None]):
        before = p.tagged_acks
        p.step(gids, slot=k % 4)
        counts.append(p.tagged_acks - before)
    assert min(counts[1:4]) > 500 and counts[6] > 500 and counts[7] > 500, counts
    p.assert_every_group_equal()


def test_escape_overflow_falls_back_to_the_compact_groups_dense_outbox():
    G, R, rows, seed = 4096, 3, 4, 0x5EED0002
    cfg, e, o = opened(G, R, rows, seed)
    w = workload.make_wl(seed, rows, G, R - 1)
    A = pick(G, 1000, 11)
    ib = workload.leader_inbox_host(w, 0, None, gids=A)                # the new leaders' first AppendEntries: older prevLogTerm
    want = o.step(ib)
    cin = compact.encode_inbox(ib, None, None)
    cout = compact.CompactOutbox(rows, len(A), R - 1, esc_cap=8, gids=A)
    e.step_compact(cin, cout)
    assert int(cout.counts[0]) > 8
    with pytest.raises(OverflowError):
        compact.decode_outbox(cout)
    dense = abi.Outbox(rows, len(A), R - 1, len(A))
    e.step_fetch_dense(0, dense.as_c())
    harness.assert_outbox_equal(want, dense, where="dense fallback")


def test_bad_active_lists_are_refused_and_leave_the_slot_free():
    G, R, rows, seed = 2048, 3, 2, 0x5EED0002
    cfg, e, o = opened(G, R, rows, seed)
    F = R - 1
    A = pick(G, 300, 12)
    ib = workload.leader_inbox_host(workload.make_wl(seed, rows, G, F), 0, None, gids=A)
    cin = compact.encode_inbox(ib, None, None)
    L = engine.lib()

    def begin(slot, n, gids):
        cout = compact.CompactOutbox(rows, max(n, 1), F, esc_cap=4096)
        ptr = None if gids is None else gids.ctypes.data
        return L.rafting_step_begin_compact_active(e._h, slot, n, ptr, C.byref(cin.as_c()), None, C.byref(cout.as_c()), 0)

    bad = A.copy(); bad[[10, 11]] = bad[[11, 10]]
    dup = A.copy(); dup[11] = dup[10]
    high = A.copy(); high[-1] = G
    cases = [(len(A), bad, -1), (len(A), dup, -1), (len(A), high, -1), (0, A, -1), (G + 1, np.arange(G + 1, dtype=np.uint32), -5),
             (len(A), None, -1)]
    for k, (n, gids, rc) in enumerate(cases):
        assert begin(k % 4, n, gids) == rc, k
    p = Pump(e, o, G, F, leader_make(workload.make_wl(seed, rows, G, F)))
    for slot in range(4):                                               # every slot is free, and the next steps are exact
        p.step(A, slot=slot)
    p.assert_every_group_equal()


def test_state_save_and_load_between_active_steps(tmp_path):
    G, R, rows, seed = 4096, 3, 4, 0x5EED0002
    cfg, e, o = opened(G, R, rows, seed)
    p = Pump(e, o, G, R - 1, leader_make(workload.make_wl(seed, rows, G, R - 1)))
    A = pick(G, 1500, 13)
    p.step(A); p.step(A)
    assert int(p.st.bits.astype(np.uint64).sum()) > 0                   # tags outstanding
    path = str(tmp_path / "shard.img")
    e.state_save(path)
    e2 = engine.Engine(cfg)
    e2.state_load(path)
    p.e = e2
    before = p.tagged_acks
    for _ in range(3):
        p.step(A)
    assert p.tagged_acks - before > 1500
    p.assert_every_group_equal()


def test_step_begin_compact_active_through_the_jni_glue(tmp_path):
    from tests import jni_exec
    from tests.jni_exec import Buf, buf_of_array, buf_of_struct, fn
    L = jni_exec.build(str(tmp_path))
    if L is None:
        pytest.skip("no gcc")
    G, R, rows, seed = 1024, 3, 2, 0x5EED0002
    F = R - 1
    cfg = abi.make_cfg(replicas=R, max_groups=G, max_rows=rows, entry_pool_cap=rows * G * 50)
    o = binding.Oracle(cfg)
    L.fake_reset()
    h = fn(L, "create", C.c_int64, C.POINTER(Buf))(C.byref(buf_of_struct(cfg)))
    assert h != 0 and L.fake_throws() == 0, L.fake_thrown_message()
    init = harness.init_array(G, terms=np.arange(G) % 7)
    o.open_bulk(0, init)
    fn(L, "groupOpenBulk", None, C.c_int64, C.c_int32, C.c_int32, C.POINTER(Buf))(h, 0, G, C.byref(buf_of_array(init)))
    begin = fn(L, "stepBeginCompactActive", None, C.c_int64, C.c_int32, C.c_int32, C.POINTER(Buf), C.POINTER(Buf), C.POINTER(Buf),
               C.POINTER(Buf), C.c_int32)
    wait = fn(L, "stepWaitCompact", None, C.c_int64, C.c_int32)
    A = pick(G, 200, 14)
    ib = workload.leader_inbox_host(workload.make_wl(seed, rows, G, F), 0, None, gids=A)
    want = o.step(ib)
    cin = compact.encode_inbox(ib, None, None)
    reqs = compact.CompactRequests()
    cout = compact.CompactOutbox(rows, len(A), F, esc_cap=rows * len(A) * F + 2 * rows * len(A), gids=A)
    begin(h, 1, len(A), C.byref(buf_of_array(A)), C.byref(buf_of_struct(cin.as_c())), C.byref(buf_of_struct(reqs.as_c())),
          C.byref(buf_of_struct(cout.as_c())), 0)
    wait(h, 1)
    assert L.fake_throws() == 0, L.fake_thrown_message()
    harness.assert_outbox_equal(want, compact.decode_outbox(cout), where="compact active step through the natives")
    fn(L, "destroy", None, C.c_int64)(h)
