"""The opt-in protocol fixes of cfg.flags on the default library (`-m gpu`): rafting_engine_create takes bits 1 and 2 and
refuses any other, and a flagged engine computes what the flagged oracle computes on every route of launch_step, on the
cluster runs the fixes exist for, on the benchmark's streams through the dense and compact host paths, through
rafting_step_device_seq and through the JNI glue, each on a stream that tests/test_cfg_fixes_cpu.py shows reaches
the fixed branches.  The leader stream, which carries no inbound request, still runs pair_kernel
and gives the unflagged engine's outboxes."""
import ctypes as C

import numpy as np
import pytest

from oracle import binding
from rafting_b200 import abi, compact, engine, workload
from tests import harness
from tests.test_cfg_fixes_cpu import (BOTH, FUZZ_IDS, HOST_PATHS, JEPSEN, LENIENT, SEQ_CASE, SEQ_LAUNCHES, SINGLE_BIT_IDS, STRICT,
                                      flagged, host_path_run, jepsen, record_fuzz)
from tests.test_cluster_gpu import Pair

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("flags", [4, 0x80000000, BOTH | 4])
def test_create_refuses_undefined_bits(flags):
    with pytest.raises(engine.RaftingError) as ex:
        engine.Engine(abi.make_cfg(replicas=3, max_groups=64, max_rows=2, flags=flags))
    assert "RAFTING_CFG_STRICT_CANDIDATE_VOTE" in str(ex.value)


@pytest.mark.parametrize("flags", [STRICT, LENIENT, BOTH])
def test_create_accepts_the_defined_bits(flags):
    e = engine.Engine(abi.make_cfg(replicas=3, max_groups=64, max_rows=2, flags=flags))
    e.close()


FUZZ = [(i, BOTH) for i in FUZZ_IDS] + [(i, b) for i in SINGLE_BIT_IDS for b in (STRICT, LENIENT)]


@pytest.mark.parametrize("case_id,flags", FUZZ)
def test_fuzz_flagged_engine_matches_flagged_oracle(case_id, flags):
    harness.run_fuzz_case(flagged(case_id, flags), harness.EngineSUT)


@pytest.mark.parametrize("R,pre_vote,seed", JEPSEN)
def test_unguarded_jepsen_runs_in_lock_step_converge(R, pre_vote, seed):
    c = jepsen(lambda cfg: Pair(engine, cfg), R, pre_vote, seed)
    assert c.counts["votes_granted_to_a_stale_log"] == 0 and c.counts["commit_rollback"] == 0
    for nd in c.nodes:
        harness.assert_states_equal(nd.sut.o, nd.sut.e, range(c.G), R - 1, where=f"node {nd.slot}")


def test_leader_stream_runs_pair_kernel_unchanged():
    G, R, rows, steps = 65536, 3, 4, 6
    F = R - 1
    cfgs = [abi.make_cfg(replicas=R, max_groups=G, max_rows=rows, flags=f) for f in (BOTH, 0)]
    o, ef, e0 = binding.Oracle(cfgs[0]), engine.Engine(cfgs[0]), engine.Engine(cfgs[1])
    init = harness.init_array(G, terms=np.arange(G) % 7)
    for s in (o, ef, e0):
        s.open_bulk(0, init)
    w1, w = workload.make_wl(0x5EED0002, 1, G, F), workload.make_wl(0x5EED0002, rows, G, F)
    want = harness.elect_all(o, w1)
    for s in (ef, e0):
        harness.assert_outbox_equal(want, harness.elect_all(s, w1), where="election")
    prev = want
    for k in range(steps):
        ib = workload.leader_inbox_host(w, k, prev)
        assert ib.flags & abi.INBOX_NO_REQUESTS
        prev = o.step(ib, threads=8)
        harness.assert_outbox_equal(prev, ef.step(ib), where=f"flagged engine, leader step {k}")
        harness.assert_outbox_equal(prev, e0.step(ib), where=f"unflagged engine, leader step {k}")
    harness.assert_states_equal(o, ef, range(0, G, 97), F, where="end of the leader stream")


@pytest.mark.parametrize("which,G", HOST_PATHS)
def test_bench_configs_through_the_host_paths(which, G):
    """The stream of test_cfg_fixes_cpu.host_path_run (which shows it reaches the fixed branches): dense host steps, compact
    steps with a request list over the whole shard, one over an active list and one due step, whose tail the device chooses.
    Every outbox equals the flagged oracle's, and so does every group's state at the end."""
    from tests.test_compact_due_gpu import _at
    cfg, init, steps = host_path_run(which, G)
    e = engine.Engine(cfg)
    e.open_bulk(0, init)
    F = e.F
    for k, (kind, ib, want, due) in enumerate(steps):
        where = f"{which} {kind} step {k}"
        if kind == "dense":
            harness.assert_outbox_equal(want, e.step(ib), where=where)
            continue
        if kind == "due":
            di, H, cap, tail, order = due
            cin = compact.encode_inbox(di, None, None, None, sweep=True)
            n = len(H) + cap
            cout = compact.CompactOutbox(ib.rows, n, F, esc_cap=ib.rows * n * F + 2 * ib.rows * n)
            got_tail = e.step_compact_due(cin, cout, cap, reqs=cin.reqs)
            assert np.array_equal(got_tail, tail), f"{where}: the tail"
            harness.assert_outbox_equal(want, _at(compact.decode_outbox(cout), order), where=where)
            continue
        n = ib.n
        cin = compact.encode_inbox(ib, None, None, None)
        cout = compact.CompactOutbox(ib.rows, n, F, esc_cap=ib.rows * n * F + 2 * ib.rows * n, gids=ib.gids)
        reqs = cin.reqs if cin.reqs is not None or ib.gids is not None else compact.CompactRequests()   # the whole shard: _req
        e.step_compact(cin, cout, reqs=reqs)
        harness.assert_outbox_equal(want, compact.decode_outbox(cout), where=where)
    o = binding.Oracle(cfg)
    o.open_bulk(0, init)
    for _, ib, _, _ in steps:
        o.step(ib, threads=8)
    got = e.export_bulk(0, G)
    for g in range(G):
        assert harness.state_bytes(got[g], F) == harness.state_bytes(o.export(g), F), f"{which}: group {g}"


def test_device_sequence_on_a_flagged_engine():
    """The first SEQ_LAUNCHES steps of a fuzz stream that reaches the fixed branches (test_cfg_fixes_cpu), enqueued with one
    rafting_step_device_seq call: launches with requests run the FIX step kernel, the NO_REQUESTS ones pair_kernel."""
    import torch
    from rafting_b200 import devbatch
    case = flagged(SEQ_CASE)
    cfg, F, G = case.cfg(), case.R - 1, case.G
    ibs, want = record_fuzz(case, SEQ_LAUNCHES)
    assert any(ib.flags & abi.INBOX_NO_REQUESTS for ib in ibs) and not all(ib.flags & abi.INBOX_NO_REQUESTS for ib in ibs)
    e = engine.Engine(cfg)
    e.open_bulk(0, case.init())
    dev = torch.device("cuda", 0)
    dins = [devbatch.DevInbox.from_host(ib, dev) for ib in ibs]
    douts = [devbatch.DevOutbox(ib.rows, ib.n, F, harness.gcols(ib, G), dev, fill=harness.POISON) for ib in ibs]
    torch.cuda.synchronize()
    n = len(ibs)
    e.step_device_seq((abi.InboxC * n)(*[d.as_c() for d in dins]), (abi.OutboxC * n)(*[d.as_c() for d in douts]), n)
    torch.cuda.synchronize()
    for k in range(n):
        harness.assert_outbox_equal(want[k], douts[k].to_host(), where=f"launch {k} of the sequence")
    o = harness.OracleSUT(cfg)
    o.open_bulk(0, case.init())
    for ib in ibs:
        o.step(ib)
    harness.assert_states_equal(o, e, range(G), F, where="end of the sequence")


def test_jni_glue_creates_a_flagged_engine(tmp_path):
    from tests import jni_exec
    from tests.test_jni_glue_gpu import GlueEngine
    L = jni_exec.build(str(tmp_path))
    if L is None:
        pytest.skip("no gcc")
    case = flagged("R3-G777")
    cfg = case.cfg()
    o, e = binding.Oracle(cfg), GlueEngine(L, cfg, case.G, case.R - 1)
    init = case.init()
    o.open_bulk(0, init), e.open_bulk(0, init)
    fz = harness.Fuzzer(cfg, o, seed=case.seed, rows=case.rows, sweep_every=case.sweep_every, stray_requests=case.stray)
    prev = None
    for k in range(20):
        ib = fz.make(prev)
        prev = o.step(ib)
        harness.assert_outbox_equal(prev, e.step(ib), where=f"step {k} through the natives")
    harness.assert_states_equal(o, e, range(case.G), case.R - 1, where="end of the stream")
    jni_exec.fn(L, "destroy", None, C.c_int64)(e.h)
