"""Parity of the CUDA engine against the CPU oracle, through the C ABI (rafting_lease/rafting_step).

Bit-exact is the bar: every outbox column and every exported state byte must match on the same
seeded stream.  All tests here need an H100 (`-m gpu`)."""
import numpy as np
import pytest

from oracle import binding
from rafting_b200 import abi, workload
from tests import harness
from tests import test_oracle_kat as kat

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def engine_mod():
    from rafting_b200 import engine
    engine.lib()
    return engine


def _scenarios():
    return sorted(n for n in dir(kat) if n.startswith("test_") and callable(getattr(kat, n)))


SINGLE_GROUP = [n for n in _scenarios() if n not in (
    "test_major_position_table", "test_major_indices_random", "test_backoff_step_matches_double_math", "test_is_better",
    "test_upstream_golden_vectors", "test_upstream_replay_plumbing_on_the_source_comment_table")]


@pytest.mark.parametrize("name", SINGLE_GROUP)
def test_kat_scenarios_on_engine(engine_mod, monkeypatch, name):
    """Every hand-derived known-answer scenario of tests/test_oracle_kat.py, run on the GPU engine."""
    monkeypatch.setattr(kat, "SUT_FACTORY", engine_mod.Engine)
    getattr(kat, name)()


def _pair(engine_mod, G, R, rows, local_slot=0, pre_vote=True, ent=0, terms_mod=7, **cfgkw):
    cfg = abi.make_cfg(replicas=R, local_slot=local_slot, max_groups=G, max_rows=rows, pre_vote=pre_vote,
                       entry_pool_cap=ent, **cfgkw)
    o, e = binding.Oracle(cfg), engine_mod.Engine(cfg)
    init = harness.init_array(G, terms=np.arange(G) % terms_mod)
    o.open_bulk(0, init)
    e.open_bulk(0, init)
    return cfg, o, e


@pytest.mark.parametrize("R,G,rows", [(3, 4096, 8), (3, 777, 5), (5, 2048, 4), (2, 512, 3), (4, 777, 5), (7, 300, 2), (9, 130, 2),
                                       (33, 40, 2)])
def test_leader_stream_parity(engine_mod, R, G, rows):
    """configs #2/#4 shape at reduced size: election warm-up, then the leader steady-state stream."""
    cfg, o, e = _pair(engine_mod, G, R, rows)
    w1 = workload.make_wl(0x5EED0002, 1, G, R - 1)
    w = workload.make_wl(0x5EED0002, rows, G, R - 1, p_reject_ppm=60_000, p_error_ppm=20_000, p_cancel_ppm=20_000)
    oo, oe = harness.elect_all(o, w1), harness.elect_all(e, w1)
    harness.assert_outbox_equal(oo, oe, where="after election")
    assert ((oe.role_word & 3) == abi.ROLE_LEADER).all()
    last = harness.run_leader_workload([o, e], w, steps=14, drop_ab=(R == 5))
    harness.assert_states_equal(o, e, range(0, G, max(1, G // 257)), R - 1, where="end of stream")
    assert (last.commit_index > 0).mean() > 0.9      # progress is a property of the stream, not of parity
    # bulk digest path agrees with per-group export
    d = e.digest(0, G)
    assert len(set(d.tolist())) > 1


@pytest.mark.parametrize("R,local_slot,pre_vote,seed", [(3, 0, True, 1), (3, 2, False, 2), (5, 2, True, 3), (4, 1, True, 4), (7, 6, False, 5)])
def test_fuzz_parity_all_event_kinds(engine_mod, R, local_slot, pre_vote, seed):
    """Random mix of every op and lane-event kind (requests, votes, snapshots, flushes, acks, forged
    and stale replies), steered by the oracle's state so that every role and error path is reached."""
    G, rows = 48, 3
    cfg, o, e = _pair(engine_mod, G, R, rows, local_slot=local_slot, pre_vote=pre_vote, ent=rows * G * 8, terms_mod=3)
    fz = harness.Fuzzer(cfg, o, seed=seed, rows=rows)
    out = None
    roles, errs = set(), set()
    for k in range(60):
        ib = fz.make(out)
        out = o.step(ib)
        oe = e.step(ib)
        harness.assert_outbox_equal(out, oe, where=f"fuzz step {k}")
        roles |= set((out.role_word & 3).tolist())
        errs |= set(((out.rep_meta >> 8) & 0xFF).ravel().tolist())
        if k % 10 == 9:
            harness.assert_states_equal(o, e, range(G), R - 1, where=f"fuzz step {k}")
    assert roles == {0, 1, 2}
    assert len(errs) > 3


@pytest.mark.parametrize("R,seed", [(3, 11), (5, 12)])
def test_fuzz_parity_class_sorted_launch(engine_mod, R, seed):
    """The same fuzz over enough groups (>= 2048) that steps with requests take the class-sorted launch: followers,
    candidates and leaders are separated by classify_kernel and the slow classes run slow_group."""
    G, rows = 2304, 3
    cfg, o, e = _pair(engine_mod, G, R, rows, local_slot=1, pre_vote=True, ent=rows * G * 8, terms_mod=3)
    fz = harness.Fuzzer(cfg, o, seed=seed, rows=rows)
    out = None
    roles = set()
    for k in range(14):
        ib = fz.make(out)
        out = o.step(ib, threads=8)
        harness.assert_outbox_equal(out, e.step(ib), where=f"fuzz step {k}")
        roles |= set((out.role_word & 3).tolist())
    harness.assert_states_equal(o, e, range(0, G, 7), R - 1, where="class-sorted fuzz")
    assert roles == {0, 1, 2}


def test_active_list_and_sweep_parity(engine_mod):
    G, R, rows = 512, 3, 2
    cfg, o, e = _pair(engine_mod, G, R, rows)
    w1 = workload.make_wl(7, 1, G, R - 1)
    harness.elect_all(o, w1), harness.elect_all(e, w1)
    # compacted active list: only every third group takes part in this step
    gids = np.arange(0, G, 3, dtype=np.uint32)
    ib = abi.Inbox(rows, len(gids), R - 1, gids=gids)
    for r in range(rows):
        for i in range(len(gids)):
            ib.timeout(r, i, harness.T0 + r, rand=0)
    oo, oe = o.step(ib), e.step(ib)
    harness.assert_outbox_equal(oo, oe, gids=gids, where="active list")
    harness.assert_states_equal(o, e, range(G), R - 1, where="active list")
    # sweep rows: leaders whose keepAlive is due fire, others do not
    for now in (harness.T0 + 100, harness.T0 + 301, harness.T0 + 5000):
        ib = abi.Inbox(1, G, R - 1, sweep=True, with_ops=False)
        ib.row_now[0] = now
        oo, oe = o.step(ib), e.step(ib)
        harness.assert_outbox_equal(oo, oe, where=f"sweep {now}")
    harness.assert_states_equal(o, e, range(G), R - 1, where="sweep")


def test_compact_group_columns_parity(engine_mod):
    """RAFTING_INBOX_COMPACT_GROUPS: per-group outbox columns hold n_active entries indexed by position in
    gids[]; they must equal the gid-indexed columns of an identical engine at those gids, and the oracle's."""
    G, R, rows = 768, 3, 3
    cfg, o, e = _pair(engine_mod, G, R, rows)
    e2 = engine_mod.Engine(cfg)
    e2.open_bulk(0, harness.init_array(G, terms=np.arange(G) % 7))
    w1 = workload.make_wl(11, 1, G, R - 1)
    harness.elect_all(o, w1), harness.elect_all(e, w1), harness.elect_all(e2, w1)
    gids = np.arange(5, G, 7, dtype=np.uint32)
    for step in range(3):
        ib = abi.Inbox(rows, len(gids), R - 1, gids=gids)
        for r in range(rows):
            for i in range(len(gids)):
                if (i + step) % 2:
                    ib.submit(r, i, harness.T0 + 10 * step + r, 1 + (i % 3))
                else:
                    ib.timeout(r, i, harness.T0 + 10 * step + r, rand=0)
        wide = e2.step(ib)
        ib.flags |= abi.INBOX_COMPACT_GROUPS
        oo, oe = o.step(ib), e.step(ib)
        assert oe.commit_index.shape == (len(gids),) and oo.commit_index.shape == (len(gids),)
        harness.assert_outbox_equal(oo, oe, where=f"compact step {step}")
        for name, _ in abi.Outbox.GROUP_COLS:
            assert np.array_equal(getattr(oe, name), getattr(wide, name)[gids]), name
    harness.assert_states_equal(o, e, range(G), R - 1, where="compact")
    # a lease taken without the flag refuses a step that carries it
    L = e.lease(1, len(gids))
    L.gids[:] = gids
    L.use(ops=True, events=False, flags=abi.INBOX_COMPACT_GROUPS)
    L.op_meta[:] = 0
    with pytest.raises(engine_mod.RaftingError):
        L.begin()
    L.use(ops=True, events=False, flags=0)
    L.run()
    e2.close()


def test_closed_group_and_capacity_errors(engine_mod):
    cfg, o, e = _pair(engine_mod, 8, 3, 2)
    o.close_group(3), e.close_group(3)
    ib = abi.Inbox(1, 8, 2)
    for i in range(8):
        ib.timeout(0, i, harness.T0)
    harness.assert_outbox_equal(o.step(ib), e.step(ib))
    with pytest.raises(engine_mod.RaftingError):
        e.lease(3)                       # rows > max_rows
    with pytest.raises(engine_mod.RaftingError):
        engine_mod.Engine(abi.make_cfg(replicas=1))


def test_two_slot_host_pipeline_matches_oracle(engine_mod):
    """rafting_step_begin_host / rafting_step_wait_slot with caller-owned buffers, two steps in flight:
    the stream is pre-recorded (oracle run), then replayed through alternating slots without waiting for
    the previous step, and every outbox and the final state must still equal the serial oracle run."""
    G, R, rows, steps = 1024, 3, 4, 10
    cfg, o, e = _pair(engine_mod, G, R, rows)
    w1 = workload.make_wl(3, 1, G, R - 1)
    w = workload.make_wl(3, rows, G, R - 1)
    harness.elect_all(o, w1), harness.elect_all(e, w1)
    inboxes, want = [], []
    prev = None
    for k in range(steps):
        ib = workload.leader_inbox_host(w, k, prev)
        prev = o.step(ib)
        inboxes.append(ib); want.append(prev)
    got = [abi.Outbox(rows, G, R - 1, G) for _ in range(steps)]
    keep = []
    NSL = 3
    for k in range(steps):
        sl = k % NSL
        if k >= NSL:
            e.step_wait_slot(sl)
        ic, oc = inboxes[k].as_c(), got[k].as_c()
        keep.append((ic, oc))
        e.step_begin_host(sl, ic, oc)
    for sl in range(NSL):
        e.step_wait_slot(sl)
    for k in range(steps):
        harness.assert_outbox_equal(want[k], got[k], where=f"pipelined step {k}")
    harness.assert_states_equal(o, e, range(0, G, 13), R - 1, where="after the pipelined replay")
    # RAFTING_HOST_SLOTS (4) leases can be outstanding at once, one more is refused
    held = [e.lease(rows) for _ in range(4)]
    with pytest.raises(engine_mod.RaftingError):
        e.lease(rows)


@pytest.mark.parametrize("R,G", [(5, 3000), (3, 2000)])
def test_vote_storm_parity(engine_mod, R, G):
    """config #3 shape at reduced size through the generic (slow-path) handlers."""
    rows = 2
    cfg = abi.make_cfg(replicas=R, local_slot=1, max_groups=G, max_rows=rows, entry_pool_cap=workload.POOL_TERMS)
    o, e = binding.Oracle(cfg), engine_mod.Engine(cfg)
    init = harness.init_array(G, terms=1 + np.arange(G) % 5)
    init["last_index"] = 100 + np.arange(G) % 50
    init["last_term"] = 1 + np.arange(G) % 5
    o.open_bulk(0, init), e.open_bulk(0, init)
    w = workload.make_wl(0x5EED0003, rows, G, R - 1, local_slot=1)
    out = None
    for k in range(10):
        ib = workload.vote_inbox_host(w, k, out)
        out = o.step(ib)
        harness.assert_outbox_equal(out, e.step(ib), where=f"vote round {k}")
    harness.assert_states_equal(o, e, range(0, G, 7), R - 1, where="vote storm end")


def test_mixed_churn_parity(engine_mod):
    """config #5 shape at reduced size: fast path and slow path interleave inside one batch."""
    G, R, rows = 4096, 3, 4
    cfg = abi.make_cfg(replicas=R, max_groups=G, max_rows=rows, entry_pool_cap=workload.POOL_TERMS)
    o, e = binding.Oracle(cfg), engine_mod.Engine(cfg)
    init = harness.init_array(G, terms=np.arange(G) % 7)
    o.open_bulk(0, init), e.open_bulk(0, init)
    w1 = workload.make_wl(0x5EED0005, 1, G, R - 1)
    harness.elect_all(o, w1), harness.elect_all(e, w1)
    w = workload.make_wl(0x5EED0005, rows, G, R - 1)
    out = None
    for k in range(50):
        ib = workload.mixed_inbox_host(w, k, out)
        out = o.step(ib)
        harness.assert_outbox_equal(out, e.step(ib), where=f"mixed step {k}")
    harness.assert_states_equal(o, e, range(0, G, 5), R - 1, where="mixed end")


def test_shard_image_survives_the_process(engine_mod, tmp_path):
    """SURVEY §8(f)-4: rafting_state_save writes the whole shard (roles, timers, Leadership.State, run tables) as one
    checksummed file; a FRESH engine that loads it continues the stream exactly where the first one stopped — every
    outbox of the following steps equals the oracle's, which never stopped.  A corrupted image is refused untouched."""
    G, R, rows = 2048, 3, 4
    cfg = abi.make_cfg(replicas=R, max_groups=G, max_rows=rows)
    e, o = engine_mod.Engine(cfg), binding.Oracle(cfg)
    init = harness.init_array(G, terms=np.arange(G) % 7)
    e.open_bulk(0, init), o.open_bulk(0, init)
    w1 = workload.make_wl(41, 1, G, R - 1); w = workload.make_wl(41, rows, G, R - 1)
    harness.assert_outbox_equal(harness.elect_all(o, w1), harness.elect_all(e, w1), where="election")
    prev = harness.run_leader_workload([o, e], w, steps=5)
    path = str(tmp_path / "shard.img")
    e.state_save(path)
    e.close()                                                                  # the process "ends" here
    e2 = engine_mod.Engine(cfg)
    bad = str(tmp_path / "bad.img")
    blob = bytearray(open(path, "rb").read()); blob[len(blob) // 2] ^= 0x40
    open(bad, "wb").write(bytes(blob))
    with pytest.raises(engine_mod.RaftingError):
        e2.state_load(bad)                                                     # checksum mismatch: nothing loaded
    assert e2.export(5).alive == 0
    e2.state_load(path)
    harness.assert_states_equal(o, e2, range(0, G, 97), R - 1, where="after load")
    harness.run_leader_workload([o, e2], w, steps=4, first_step=5, prevs=prev)
    harness.assert_states_equal(o, e2, range(0, G, 97), R - 1, where="four steps after the restart")
    with pytest.raises(engine_mod.RaftingError):
        engine_mod.Engine(abi.make_cfg(replicas=R, max_groups=G // 2, max_rows=rows)).state_load(path)   # other shape
