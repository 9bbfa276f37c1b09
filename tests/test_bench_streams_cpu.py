"""The CPU half of tests/test_bench_streams_gpu.py.

bench.py reuses device inboxes (its settle inbox across 8 launches, tools/bench_secondary.py one inbox for a whole run),
and the generators write a lane's payload (ev_tn / ev_el) only where they write an event: every other cell keeps what an
earlier launch left there.  A consumer must therefore never read a payload under a zero ev_meta.  The first tests hold the
oracle to that rule on the bench's streams; the GPU suite holds the engine to it.

The GPU suite also restates locals of bench.py's run_engine (SETTLE, the init recipe) to follow the bench launch by launch;
the last tests read run_engine's source so that a change to the bench the GPU suite would not follow fails here."""
import ast
import copy
import inspect
import sys

import numpy as np
import pytest

from oracle import binding
from rafting_b200 import abi, workload
from tests import harness
from tests.test_bench_streams_gpu import SETTLE, bench_init, state_digest


def reused(stale: abi.Inbox | None, fresh: abi.Inbox) -> abi.Inbox:
    """`fresh` as a reused inbox holds it: the generator's cells from `fresh`, every lane payload under a zero ev_meta kept
    from `stale` (the inbox's previous contents; None: never written, POISON)."""
    ib = copy.deepcopy(fresh)
    keep = fresh.ev_meta == 0
    for name in ("ev_tn", "ev_el"):
        cur = getattr(ib, name)
        if stale is None:
            cur.view(np.uint8).reshape(cur.shape + (-1,))[keep] = harness.POISON
        else:
            cur[keep] = getattr(stale, name)[keep]
    return ib


def run_twice(cfg, init, inboxes, where):
    """Steps two oracles side by side, one on fresh inboxes, one on the same inboxes as a reused buffer holds them; every
    outbox and the end states must be identical.  inboxes(k, prev) -> the fresh inbox of step k (None: the stream ended)."""
    a, b = binding.Oracle(cfg), binding.Oracle(cfg)
    a.open_bulk(0, init)
    b.open_bulk(0, init)
    prev, stale, k, stale_cells = None, None, 0, 0
    while (ib := inboxes(k, prev)) is not None:
        if stale is not None and (stale.rows, stale.n) != (ib.rows, ib.n):
            stale = None
        old = reused(stale, ib)
        stale_cells += int((ib.ev_meta == 0).sum())
        prev = a.step(ib, threads=4)
        harness.assert_outbox_equal(prev, b.step(old, threads=4), where=f"{where}: step {k}")
        stale, k = old, k + 1
    G = cfg.max_groups
    harness.assert_states_equal(a, b, range(G), cfg.replicas - 1, where=where)
    assert stale_cells > 0


def test_oracle_ignores_stale_payload_config2_stream():
    """config #2's stream (election through one reused single-row inbox, then the leader stream through another, op_ab
    absent) at a reduced size."""
    G, R, rows = 4096, 3, 16
    cfg = abi.make_cfg(replicas=R, max_groups=G, max_rows=rows)
    w1 = workload.make_wl(0x5EED0002, 1, G, R - 1)
    w = workload.make_wl(0x5EED0002, rows, G, R - 1)

    def inboxes(k, prev):
        if k < 3:
            return workload.election_inbox_host(w1, k, prev)
        if k == 3:
            prev = None                                  # the leader stream starts without a previous outbox, as the bench's
        if k >= 3 + SETTLE + 6:
            return None
        ib = workload.leader_inbox_host(w, k - 3, prev)
        ib.op_ab = None
        return ib
    run_twice(cfg, bench_init(G, 0), inboxes, "config #2")


def test_oracle_ignores_stale_payload_config5_stream():
    """config #5's stream for 144 ticks (both churn and catch-up cycles), one reused inbox, as bench_secondary drives it."""
    G, R, rows = 2048, 3, 4
    cfg = abi.make_cfg(replicas=R, max_groups=G, max_rows=rows, entry_pool_cap=workload.POOL_TERMS)
    w1 = workload.make_wl(0x5EED0005, 1, G, R - 1)
    w = workload.make_wl(0x5EED0005, rows, G, R - 1)
    ops = set()

    def inboxes(k, prev):
        if k < 3:
            return workload.election_inbox_host(w1, k, prev)
        if k == 3:
            prev = None
        if k >= 3 + 36:
            return None
        ib = workload.mixed_inbox_host(w, k - 3, prev)
        ops.update(np.unique(ib.op_meta & np.uint64(0xFF)).tolist())
        return ib
    run_twice(cfg, harness.init_array(G, terms=np.arange(G) % 7), inboxes, "config #5")
    assert {abi.OP_AE_REQUEST, abi.OP_FLUSH, abi.OP_TIMEOUT} <= ops


def test_oracle_ignores_stale_payload_config3_stream():
    """config #3's vote storm (R = 5, local_slot 2): vote replies only where a ballot was emitted."""
    G, R = 2048, 5
    cfg = abi.make_cfg(replicas=R, local_slot=2, max_groups=G, max_rows=1)
    init = harness.init_array(G, terms=1 + np.arange(G) % 5)
    init["last_index"] = 100 + np.arange(G) % 50
    init["last_term"] = 1 + np.arange(G) % 5
    w = workload.make_wl(0x5EED0003, 1, G, R - 1, local_slot=2)
    run_twice(cfg, init, lambda k, prev: workload.vote_inbox_host(w, k, prev) if k < 8 else None, "config #3")


# ---- the run_engine recipe the GPU suite restates ------------------------------------------------------------------------
@pytest.fixture(scope="module")
def run_engine_source():
    import bench
    tree = ast.parse(inspect.getsource(bench.run_engine))
    return tree, {ast.unparse(n) for n in ast.walk(tree) if isinstance(n, ast.stmt)}


def test_bench_recipe_statements(run_engine_source):
    """The statements of run_engine the GPU suite follows, as written in bench.py."""
    _, stmts = run_engine_source
    want = [
        f"SETTLE = {SETTLE}",
        "gid_base = rank * G",
        "seed = SEED2 if world == 1 else SEED4",
        "G = args.groups or (G_CONFIG2 if world == 1 else G_CONFIG4 // world)",
        "R, rows = (args.replicas, args.rows)",
        "cfg = abi.make_cfg(replicas=R, max_groups=G, max_rows=rows, device=local)",
        "e.open_bulk(0, init)",
        "e.comm_init(0, 1, None)",
        "w1 = workload.make_wl(seed, 1, G, F, gid_base=gid_base)",
        "w = workload.make_wl(seed, rows, G, F, gid_base=gid_base)",
        # the election: one single-row inbox and outbox, phases 0, 1, 2
        "in1, out1 = (devbatch.DevInbox(1, G, F, dev), devbatch.DevOutbox(1, G, F, G, dev))",
        "workload.election_step(w1, ph, prev_c, ic, on_device=True, stream=stream_ptr)",
        "outs = [devbatch.DevOutbox(rows, G, F, G, dev) for _ in range(2)]",
        # settle: one reused inbox without op_ab, the stream from step 0 without a previous outbox
        "settle = devbatch.DevInbox(rows, G, F, dev, unavail=False)",
        "ic = settle.as_c()",
        "workload.leader_step(w, k, None if prev_out is None else prev_out.as_c(), ic, on_device=True, stream=stream_ptr)",
        "prev_out = outs[k % 2]",
        "e.checkpoint()",
        # the recorded window: distinct inboxes without op_ab, steps SETTLE + k
        "probe = devbatch.DevInbox(rows, G, F, dev, unavail=False)",
        "inboxes = [probe] + [devbatch.DevInbox(rows, G, F, dev, unavail=False) for _ in range(L - 1)]",
        "L = window_launches(args, G)",
        "workload.leader_step(w, SETTLE + k, prev_out.as_c(), ic, on_device=True, stream=stream_ptr)",
        "prev_out = start_out",
        # the timed replay
        "ics = (abi.InboxC * L)(*[ib.as_c() for ib in inboxes])",
        "ocs = (abi.OutboxC * L)(*[outs[k % 2].as_c() for k in range(L)])",
        "e.restore(sync=False)",
        "e.step_device_seq(ics, ocs, L, gather=gather, stream=0)",
        "gather = world > 1",
        "dump_outputs(args.dump_outputs, outs[(L - 1) % 2], rows, G, F)",
    ]
    missing = [s for s in want if s not in stmts]
    assert not missing, f"bench.py's run_engine no longer holds {missing}: tests/test_bench_streams_gpu.py follows the old recipe"
    loops = {ast.unparse(n.iter) for n in ast.walk(run_engine_source[0]) if isinstance(n, ast.For)}
    assert {"(0, 1, 2)", "range(SETTLE)", "range(L)"} <= loops, loops


@pytest.mark.parametrize("gid_base", [0, 5 * 131072])
def test_bench_init_recipe(run_engine_source, gid_base):
    """run_engine's init statements, executed, give what bench_init restates."""
    import bench
    tree, _ = run_engine_source
    body = [n for n in ast.walk(tree) if isinstance(n, ast.Assign)
            and any((isinstance(t, ast.Name) and t.id == "init") or
                    (isinstance(t, ast.Subscript) and isinstance(t.value, ast.Name) and t.value.id == "init") for t in n.targets)]
    assert len(body) >= 2
    G = 1000
    ns = {"np": np, "abi": abi, "workload": workload, "G": G, "gid_base": gid_base}
    exec(compile(ast.Module(body=body, type_ignores=[]), bench.__file__, "exec"), ns)
    got = ns["init"]
    assert got.dtype == abi.GROUP_INIT_DTYPE
    assert got.tobytes() == bench_init(G, gid_base).tobytes()


def test_bench_window_shape(monkeypatch):
    """The default shape the GPU suite checks: 64 K groups, R = 3, 16 rows, 128 launches, the inbox bytes of a launch."""
    import bench
    monkeypatch.setattr(sys, "argv", ["bench.py"])
    args = bench.parse()
    assert (args.replicas, args.rows, args.groups, args.launches) == (3, 16, 0, 0)
    assert bench.window_launches(args, bench.G_CONFIG2) == 128
    assert bench.inbox_bytes_per_launch(bench.G_CONFIG2, 16, 2) == 16 * 65536 * (8 + 16 + 2 * (8 + 16 + 16))


def test_state_digest_restatement_is_fnv1a():
    """The GPU suite's restatement of rafting_state_digest is FNV-1a 64 (published test vectors)."""
    for text, want in ((b"", 0xCBF29CE484222325), (b"a", 0xAF63DC4C8601EC8C), (b"foobar", 0x85944171F73967E8)):
        got = state_digest(np.frombuffer(text, dtype=np.uint8).reshape(1, len(text)))
        assert int(got[0]) == want, text
