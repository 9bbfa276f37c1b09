"""The opt-in protocol fixes of cfg.flags without a GPU: the streams tests/test_cfg_fixes_gpu.py runs reach the fixed branches
(replayed into an oracle without the flags, some outbox differs), and the default library holds the kernels launch_step routes
a flagged engine to: a FIX instantiation of each step and slow kernel, and still exactly one pair_kernel."""
import copy
import os
import re
import shutil
import subprocess
from dataclasses import dataclass

import numpy as np
import pytest

from oracle import binding
from rafting_b200 import abi, compact, workload
from tests import harness
from tests.cluster_sim import Cluster

STRICT, LENIENT = abi.CFG_STRICT_CANDIDATE_VOTE, abi.CFG_LENIENT_FOLLOWER_COMMIT
BOTH = STRICT | LENIENT


@dataclass(frozen=True)
class FlaggedCase(harness.FuzzCase):
    """A fuzz case whose engine and oracle run with cfg.flags."""
    flags: int = BOTH

    def cfg(self) -> abi.Cfg:
        c = super().cfg()
        c.flags = self.flags
        return c


_CASES = {c.id: c for c in harness.FUZZ_UNSORTED + harness.FUZZ_SORTED}


def flagged(case_id: str, flags: int = BOTH) -> FlaggedCase:
    c = _CASES[case_id]
    return FlaggedCase(**{k: getattr(c, k) for k in c.__dataclass_fields__}, flags=flags)


# every route of launch_step (engine.cu): R = 2; R = 3 unsorted (rerouted from pair_kernel to the FIX step kernel) and
# class-sorted; R = 5; R = 9; R = 17 and 33 (looped); an active list with COMPACT_GROUPS
FUZZ_IDS = ["R2-G777", "R3-G777", "3-11", "5-12", "R9-G777", "R17-G300-wide", "R33-G300", "R3-active1500-compact"]
# the cases the GPU suite also runs with one bit alone
SINGLE_BIT_IDS = ["R3-G777", "5-12"]
# the stream tests/test_cfg_fixes_gpu.py enqueues with one rafting_step_device_seq call: R = 3, unsorted, every fourth launch
# flagged NO_REQUESTS (pair_kernel) and the others with requests (the FIX step kernel)
SEQ_CASE, SEQ_LAUNCHES = "R3-G777", 12
# the unguarded Jepsen runs of tests/test_cluster_cpu.py::test_opt_in_fixes_make_the_unguarded_runs_safe_and_live
JEPSEN = [(3, False, 102), (5, True, 1030), (3, False, 1007), (5, False, 1032), (5, False, 1031)]


class Recorder:
    """An oracle that records every call made on it, so that the same calls can be replayed into another oracle."""

    def __init__(self, cfg):
        self.o, self.calls = binding.Oracle(cfg), []

    def __getattr__(self, name):
        f = getattr(self.o, name)

        def call(*a, **kw):
            self.calls.append((name, copy.deepcopy(a), dict(kw)))
            return f(*a, **kw)
        return call


def unflagged(cfg: abi.Cfg) -> abi.Cfg:
    c = type(cfg).from_buffer_copy(cfg)
    c.flags = 0
    return c


def record_fuzz(case: FlaggedCase, steps: int) -> tuple[list, list]:
    """The first `steps` inboxes of `case` and the flagged oracle's outboxes (run on both sides, as the CPU fuzz rehearsal
    does)."""
    inboxes, outs = [], []

    class Rec(harness.OracleSUT):
        def step(self, ib):
            out = super().step(ib)
            inboxes.append(copy.deepcopy(ib))
            outs.append(out)
            return out
    harness.run_fuzz_case(case, harness.OracleSUT, steps=steps, ref_factory=Rec)
    return inboxes, outs


def fuzz_differs(case: FlaggedCase, steps: int) -> int:
    """Replays the recorded inboxes of `case` into an oracle without the flags from the same initial state; returns the number
    of steps whose outbox differs from the flagged oracle's."""
    inboxes, outs = record_fuzz(case, steps)
    o = harness.OracleSUT(unflagged(case.cfg()))
    o.open_bulk(0, case.init())
    return sum(bool(o.step(ib).equal(want)) for ib, want in zip(inboxes, outs))


@pytest.mark.parametrize("case_id", FUZZ_IDS)
def test_fuzz_streams_reach_the_fixed_branches(case_id):
    case = flagged(case_id)
    assert fuzz_differs(case, case.cpu_steps if case.leader_share else 2 * case.cpu_steps) > 0, case_id


@pytest.mark.parametrize("case_id", SINGLE_BIT_IDS)
@pytest.mark.parametrize("bit", [STRICT, LENIENT])
def test_fuzz_streams_reach_each_bit_alone(case_id, bit):
    case = flagged(case_id, bit)
    assert fuzz_differs(case, case.steps) > 0, (case_id, bit)


def test_device_sequence_stream_reaches_the_fixed_branches():
    assert fuzz_differs(flagged(SEQ_CASE), SEQ_LAUNCHES) > 0


def jepsen(make, R, pre_vote, seed, flags=BOTH):
    """The unguarded Jepsen run of tests/test_cluster_cpu.py with cfg.flags, every node built by make(cfg)."""
    rng = np.random.default_rng(seed)
    c = Cluster(make, G=4, R=R, seed=seed, drop_ppm=30_000, compact_every=30, pre_vote=pre_vote, guard_candidate_votes=False,
                cfg_flags=flags)
    c.run(80)
    for phase in range(10):
        k = int(rng.integers(0, (R - 1) // 2 + 1))
        c.cut = set(int(x) for x in rng.choice(R, size=k, replace=False))
        c.run(40)
    c.cut = set()
    c.run(250)
    c.drop_ppm = 0
    c.run(120, submit=False)
    c.check(converged=True)
    return c


@pytest.mark.parametrize("R,pre_vote,seed", [(3, False, 102), (5, True, 1030)])
def test_cluster_runs_reach_the_fixed_branches(R, pre_vote, seed):
    nodes = []

    def make(cfg):
        nodes.append((Recorder(cfg), cfg))
        return nodes[-1][0]
    jepsen(make, R, pre_vote, seed)
    differ = 0
    for rec, cfg in nodes:
        o = binding.Oracle(unflagged(cfg))
        mine = binding.Oracle(cfg)
        for name, a, kw in rec.calls:
            r0, r1 = getattr(o, name)(*a, **kw), getattr(mine, name)(*a, **kw)
            if name == "step":
                differ += bool(r0.equal(r1))
    assert differ > 0, (R, seed)


# the runs of tests/test_cfg_fixes_gpu.py::test_bench_configs_through_the_host_paths: config #5 class-sorted and unsorted (the
# R = 3 reroute), config #3 class-sorted
HOST_PATHS = [("config5", 16384), ("config5", 1024), ("config3", 16384)]


def host_path_run(which: str, G: int, flags: int = BOTH):
    """The bench stream `which` at G groups, closed loop on an oracle with `flags`, as the host-path test steps it: the election
    (config #5) and 6 steps as dense steps, 4 as compact steps over the whole shard, one over an active list of G / 4 groups
    and one due step.  Returns (cfg, init, steps), each step (kind, ib, want, due): ib the inbox the oracle stepped, want its
    outbox.  A due step's oracle inbox is the sweep step over the sorted list of the host's groups and the tail the device
    will choose (due_model.tail over the oracle's timers); `due` = (the due step's inbox, the host list, cap, tail, order),
    order mapping the sorted list back to the list's positions."""
    from tests import compact_active_model as active
    from tests import due_model as dm
    from tests import timers_model as tm
    if which == "config5":
        R, rows = 3, 4
        cfg = abi.make_cfg(replicas=R, max_groups=G, max_rows=rows, entry_pool_cap=rows * G * 50, flags=flags)
        init = harness.init_array(G, terms=np.arange(G) % 7)
        w1, w = workload.make_wl(0x5EED0005, 1, G, R - 1), workload.make_wl(0x5EED0005, rows, G, R - 1)
        make = lambda k, prev, gids=None: workload.mixed_inbox_host(w, k, prev, gids=gids)   # noqa: E731
    else:
        R, rows = 5, 1
        cfg = abi.make_cfg(replicas=R, local_slot=2, max_groups=G, max_rows=rows, entry_pool_cap=workload.POOL_TERMS, flags=flags)
        init = harness.init_array(G, terms=1 + np.arange(G) % 5)
        init["last_index"] = 100 + np.arange(G) % 50
        init["last_term"] = 1 + np.arange(G) % 5
        w1, w = None, workload.make_wl(0x5EED0003, rows, G, R - 1, local_slot=2)
        make = lambda k, prev, gids=None: workload.vote_inbox_host(w, k, prev, gids=gids)   # noqa: E731
    o = binding.Oracle(cfg)
    o.open_bulk(0, init)
    steps, prev = [], None

    def step(kind, ib, due=None):
        out = o.step(ib, threads=8)
        steps.append((kind, ib, out, due))
        return out
    if w1 is not None:
        for ph in ((0, 1, 2) if cfg.pre_vote else (0, 2)):
            prev = step("dense", workload.election_inbox_host(w1, ph, prev))
        prev = None
    for k in range(10):
        prev = step("dense" if k < 6 else "compact", make(k, prev))
    rng = np.random.default_rng(G)
    A = np.sort(rng.choice(G, G // 4, replace=False)).astype(np.uint32)
    prev = step("active", make(10, active.carry_outbox(prev, None, A, G), gids=A))
    # the due step: a host list with the stream's ops and events, its first row a sweep that fires the timers of every
    # group due by then (config #3 has one row: its due step fires timers only)
    H = np.sort(rng.choice(G, G // 8, replace=False)).astype(np.uint32)
    ib = make(11, active.carry_outbox(prev, A, H, G), gids=H)
    ib.row_now = np.zeros(rows, np.int64)
    ops = ib.op_meta != 0
    ib.row_now[0] = (int(ib.op_nr["x"][ops].min()) if ops.any() else workload.T0_MS) + 4000
    t = tm.table([o.export(g) for g in range(G)])
    n_due = int((tm.due(t, int(ib.row_now[0])) & ~np.isin(np.arange(G), H)).sum())
    cap = min(n_due + 50, G - len(H))
    tail, _ = dm.tail(t, H, cap, int(ib.row_now[0]))
    di = compact.due_inbox(ib, cap)
    L = np.concatenate([H, tail])
    order = np.argsort(L, kind="stable")
    si = abi.Inbox.__new__(abi.Inbox)                    # the same step over sorted(L), positional
    si.__dict__.update(di.__dict__)
    si.gids = np.ascontiguousarray(L[order], dtype=np.uint32)
    for name in ("op_meta", "op_nr", "op_ab", "op_cd", "op_e", "ev_meta", "ev_tn", "ev_el"):
        col = getattr(di, name)
        if col is not None:
            setattr(si, name, np.ascontiguousarray(col[:, order]))
    step("due", si, (di, H, cap, tail, order))
    return cfg, init, steps


@pytest.mark.parametrize("which,G", HOST_PATHS)
def test_host_path_streams_reach_the_fixed_branches(which, G):
    cfg, init, steps = host_path_run(which, G)
    p = binding.Oracle(unflagged(cfg))
    p.open_bulk(0, init)
    assert sum(bool(want.equal(p.step(ib, threads=8))) for _, ib, want, _ in steps) > 0, (which, G)


CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
FIX_KERNELS = ["unrolled11step_kernelILi1ELi3ELb1E", "unrolled11step_kernelILi2ELi3ELb1E", "unrolled11step_kernelILi4ELi3ELb1E",
               "unrolled11step_kernelILi8ELi2ELb1E", "looped11step_kernelILi32ELi0ELb1E", "unrolled11slow_kernelILi2ELi4ELb1E",
               "unrolled11slow_kernelILi4ELi4ELb1E"]


@pytest.mark.skipif(not os.path.exists(CUOBJDUMP), reason="cuobjdump not installed")
def test_library_has_the_fix_instantiations_and_one_pair_kernel():
    from rafting_b200 import _build
    out = subprocess.run([CUOBJDUMP, "-res-usage", _build.build()], capture_output=True, text=True, check=True).stdout
    names = re.findall(r"Function (\S+):", out)
    for k in FIX_KERNELS:
        assert sum(k in n for n in names) == 1, f"no FIX instantiation {k}"
    assert sum("pair_kernel" in n for n in names) == 1, [n for n in names if "pair_kernel" in n]
