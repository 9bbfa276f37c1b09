"""The host side of rafting_log_gather_step_begin, without a GPU: the rafting_plan_ref_t mirror, and compact.ae_ranges, the
pump's decoder of a compact outbox's AppendEntries ranges (what it passes to rafting_log_gather), against the ranges of the
dense plans the oracle produces on the leader stream, config #5's mixed stream and config #3's vote storm."""
import os
import shutil
import subprocess

import numpy as np
import pytest

from oracle import binding
from rafting_b200 import abi, compact, workload
from tests import compact_model as model
from tests import harness
from tests.compact_model import EL, PT

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.skipif(shutil.which("gcc") is None, reason="no gcc")
def test_plan_ref_mirror_matches_the_header(tmp_path):
    src, exe = tmp_path / "p.c", tmp_path / "p"
    names = abi.PLAN_REF.names
    src.write_text("#include <stdio.h>\n#include <stddef.h>\n#include \"rafting_b200.h\"\nint main(void) {\n"
                   '  printf("%zu\\n", sizeof(rafting_plan_ref_t));\n'
                   + "".join(f'  printf("%zu %zu\\n", offsetof(rafting_plan_ref_t, {n}), sizeof(((rafting_plan_ref_t*)0)->{n}));\n'
                             for n in names) + "  return 0;\n}\n")
    subprocess.run(["gcc", "-std=c11", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    out = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split("\n")
    assert int(out[0]) == abi.PLAN_REF.itemsize
    for n, line in zip(names, out[1:]):
        off, size = map(int, line.split())
        assert (off, size) == (abi.PLAN_REF.fields[n][1], abi.PLAN_REF.fields[n][0].itemsize), n


def dense_ranges(dense: abi.Outbox, F: int, n: int):
    m = dense.plan_meta.reshape(-1)
    c = np.where((m & 0xF) == abi.PLAN_AE, (m >> 16) & 0xFFFF, 0).astype(np.int64)
    t = np.flatnonzero(c)
    return t, (t // F) % n, dense.plan_pp.reshape(-1)["x"][t] + 1, c[t]


def _check(dense, co, F, G, where):
    got = compact.ae_ranges(co)
    want = dense_ranges(dense, F, G)
    for a, b, what in zip(got, want, ("lane slots", "gids", "first indices", "counts")):
        assert np.array_equal(a, b), f"{where}: {what}"
    return len(want[0]), int((co.plan_c.reshape(-1) >> 4 & 1).sum())


def _stream(G, R, rows, steps, flags, o, w, inbox):
    F = R - 1
    st, nxt, prev, plans, escaped = model.InFlight(G, F), None, None, 0, 0
    for k in range(steps):
        ib = inbox(w, k, prev)
        dense = o.step(ib)
        co = model.pack(dense, model.oracle_epoch(o, G), st, esc_cap=1 << 20, flags=flags, replies=True)
        p, e = _check(dense, co, F, G, f"flags {flags}, step {k}")
        plans, escaped = plans + p, escaped + e
        nxt, prev = model.next_of(dense, co), dense
    return plans, escaped


@pytest.mark.parametrize("flags", [0, EL, PT, EL | PT])
@pytest.mark.parametrize("R", [3, 5])
def test_decoded_ranges_equal_the_dense_plans_on_the_leader_and_mixed_streams(flags, R):
    G, rows = 256, 4
    for seed, inbox in ((0x5EED0002, workload.leader_inbox_host), (0x5EED0005, workload.mixed_inbox_host)):
        cfg = abi.make_cfg(replicas=R, max_groups=G, max_rows=rows, entry_pool_cap=workload.POOL_TERMS)
        o = binding.Oracle(cfg)
        o.open_bulk(0, harness.init_array(G, terms=np.arange(G) % 7))
        harness.elect_all(o, workload.make_wl(seed, 1, G, R - 1))
        plans, escaped = _stream(G, R, rows, 12, flags, o, workload.make_wl(seed, rows, G, R - 1), inbox)
        assert plans > 0 and (escaped > 0 or flags & PT)      # kind 1 escapes its prev-term plans; kind 7 carries them


@pytest.mark.parametrize("flags", [0, EL | PT])
def test_decoded_ranges_equal_the_dense_plans_on_the_vote_storm(flags):
    G, R, rows = 256, 3, 4
    o, w = model.storm(G, R, rows)
    # ballots (kinds 5 / 6 under EL) and the new leaders' heartbeats ask for nothing: no range may be decoded from them
    _stream(G, R, rows, 16, flags, o, w, workload.vote_inbox_host)


def test_decoded_ranges_of_an_active_list():
    G, R, rows = 256, 3, 4
    cfg = abi.make_cfg(replicas=R, max_groups=G, max_rows=rows, entry_pool_cap=workload.POOL_TERMS)
    o = binding.Oracle(cfg)
    o.open_bulk(0, harness.init_array(G, terms=np.arange(G) % 7))
    harness.elect_all(o, workload.make_wl(0x5EED0002, 1, G, R - 1))
    w, st, dense = workload.make_wl(0x5EED0002, rows, G, R - 1), model.InFlight(G, R - 1), None
    for k in range(4):
        dense = o.step(workload.leader_inbox_host(w, k, dense))
        co = model.pack(dense, model.oracle_epoch(o, G), st, esc_cap=1 << 20)
    L = np.arange(3, G, 5, dtype=np.uint32)
    sub = compact.CompactOutbox(rows, len(L), R - 1, esc_cap=1, gids=L)   # the same plans over a list: positions stand for L
    sub.plan_c[...] = co.plan_c[:, L]
    sub.last_entry[...] = co.last_entry[L]
    t, g, f, c = compact.ae_ranges(sub)
    wt, wg, wf, wc = dense_ranges(dense, R - 1, G)
    keep = np.isin(wg, L) & (co.plan_c.reshape(-1)[wt] >> 4 & 1 == 0)
    assert np.array_equal(g, wg[keep]) and np.array_equal(f, wf[keep]) and np.array_equal(c, wc[keep]) and len(t) > 0
