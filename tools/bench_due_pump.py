"""A heartbeat pump on the GPU: three ways to keep a 64 K x 3 node's timers going on a 10 ms tick (tests/timers_model.Peers:
followers kept by heartbeats, leaderless groups electing, a leader lost at tick 150 and a second election wave).

  dense   the dense whole-shard step with a sweep row (Engine.step: lease, fill, run, copy back)
  rule    compact sweep steps over the pipelining rule's list (include/rafting_b200.h), fed by due queries
  due     compact due steps (rafting_step_begin_compact_due) over each tick's event gids; the cap follows counts[3] of the
          steps waited for: max(cap0, 2 x the largest), so that a burst is caught before it overflows

at d = 0 and d = 3 steps in flight.  The stream is the dense pump's (every pump leaves the shard in the same state: the GPU
tests hold them to it), and each compact pump is checked against it by digest at the end.  Per tick it reports the time the
host spends inside the engine's calls (begin, wait, due query; the Python encoding is outside the window), the wire bytes up
and down (from the shapes of what crossed PCIe), and the groups listed.  One JSON line per (pump, d), with the device name and
power limit it was measured on.

    python tools/bench_due_pump.py [--ticks 320] [--cap0 4096]"""
import argparse
import json
import os
import subprocess
import sys
import time
from collections import deque

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from rafting_b200 import abi, compact, engine, workload  # noqa: E402
from tests import compact_active_model as active  # noqa: E402
from tests import harness  # noqa: E402
from tests import timers_model as tm  # noqa: E402


def device():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True).stdout.strip()
    except OSError:
        return "unknown"


G, R, ROWS = 65536, 3, 3
F = R - 1


def _open():
    cfg = abi.make_cfg(replicas=R, max_groups=G, max_rows=ROWS, entry_pool_cap=64, heartbeat_ms=100, election_ms=300)
    init = harness.init_array(G, terms=1 + np.arange(G) % 5)
    init["now_ms"] = workload.T0_MS
    e = engine.Engine(cfg)
    e.open_bulk(0, init)
    return e, init


def _stats(name, d, ts, up, down, listed, dev, **kw):
    ts = np.array(ts[1:]) * 1e6
    return dict(pump=name, d=d, groups=G, ticks=len(ts) + 1, tick_us_p50=round(float(np.median(ts)), 1),
                tick_us_p99=round(float(np.percentile(ts, 99)), 1), bytes_up_p50=int(np.median(up[1:])),
                bytes_down_p50=int(np.median(down[1:])), listed_p50=int(np.median(listed[1:])), listed_max=int(max(listed[1:])),
                device=dev, **kw)


def dense_pump(P, ticks, dev):
    e, init = _open()
    wants, terms, ts, up, down, inboxes = [], init["term"].astype(np.int64), [], [], [], []
    for k in range(ticks):
        ib = P.inbox(k, wants[k - P.DELAY] if k >= P.DELAY else None, terms)
        inboxes.append(ib)
        s = time.perf_counter()
        want = e.step(ib)
        ts.append(time.perf_counter() - s)
        wants.append(want)
        terms = want.current_term.copy()
        up.append(sum(getattr(ib, c).nbytes for c in ("row_now", "op_meta", "op_nr", "op_ab", "op_cd", "op_e", "ev_meta", "ev_tn", "ev_el")
                      if getattr(ib, c) is not None))
        down.append(sum(getattr(want, c).nbytes for c, _, _ in abi.Outbox.ROW_COLS) +
                    sum(getattr(want, c).nbytes for c, _ in abi.Outbox.GROUP_COLS))
    digest = e.digest(0, G)
    e.close()
    return inboxes, digest, _stats("dense", 0, ts, up, down, [G] * ticks, dev)   # synchronous: nothing in flight


def compact_pump(kind, P, inboxes, ticks, d, cap0, digest, dev):
    """kind "rule" or "due"; the inboxes are the dense pump's, so the acks' tags come from this pump's own outboxes"""
    import torch
    e, _ = _open()
    bufs = [torch.zeros(G, dtype=torch.int32).pin_memory() for _ in range(4)]
    events, steps, pending = {}, {}, deque()
    ts, up, down, listed, counts, overflows = [], [], [], [], [], 0
    clock = [0.0]

    def call(f, *a, **kw):
        s = time.perf_counter()
        r = f(*a, **kw)
        clock[0] += time.perf_counter() - s
        return r

    def finish(j):
        nonlocal overflows
        ci, cout, host, L = steps[j]
        if kind == "due":
            tail = call(e.step_wait_compact_due, j % 4)
            cout.gids = np.concatenate([host, tail])
            counts.append(int(cout.counts[3])); overflows += int(cout.counts[3]) > len(tail)
            down[j] += len(tail) * 4
        else:
            call(e.step_wait_compact, j % 4)
        down[j] += cout.nbytes() + int(min(cout.counts[0], cout.esc_cap)) * abi.CESC_OUT.itemsize
        steps[j] = (None, cout, host, cout.gids)

    if kind == "rule":
        for t in range(d + 1):
            call(e.timers_due_begin, t % 4, P.now(t), bufs[t % 4].data_ptr(), G)
    for k in range(ticks):
        ib = inboxes[k]
        clock[0] = 0.0
        up.append(0); down.append(0)
        while len(pending) > d:
            finish(pending.popleft())
        events[k] = tm.event_gids(ib)
        if kind == "rule":
            n_q, _ = call(e.timers_due_wait, k % 4)
            Q = bufs[k % 4].numpy()[:n_q].view(np.uint32).astype(np.int64)
            flight = [events[j] for j in pending]
            host = np.union1d(np.union1d(Q, events[k]), np.concatenate(flight) if flight else np.zeros(0, np.int64)).astype(np.uint32)
            cap = 0
        else:
            host = events[k].astype(np.uint32)
            cap = min(max(cap0, 2 * max(counts, default=0)), G - len(host))
        n = len(host) + cap
        ai = tm.slice_inbox(ib, host)
        if kind == "due":
            ai = compact.due_inbox(ai, cap)
        tags = np.full((ROWS, n, F), abi.CTAG_NONE, np.uint8)
        sent_term, sent_inc = np.zeros(n, np.int64), np.zeros(n, np.uint32)
        j = k - P.DELAY
        if j in steps and steps[j][0] is None:
            _, cj, _, Lj = steps[j]
            p = active.positions(Lj, host, G)
            has, q = p >= 0, np.maximum(p, 0)
            tp = cj.tags(rpc_only=True)
            nh = len(host)
            for r in range(2):
                tags[r + 1][:nh][has] = tp[r][q[has]]
            sent_term[:nh][has], sent_inc[:nh][has] = cj.current_term[q[has]], cj.incarnation[q[has]]
        ci = compact.encode_inbox(ai, tags, sent_term, sent_inc, sweep=True)
        cout = compact.CompactOutbox(ROWS, n, F, esc_cap=ROWS * n * F + 2 * ROWS * n, gids=host if kind == "rule" else None)
        reqs = None if ci.reqs is None else ci.reqs.as_c()
        up[k] += ci.nbytes() + (0 if ci.reqs is None else ci.reqs.nbytes()) + len(host) * 4 + ROWS * 8
        if kind == "due":
            call(e.step_begin_compact_due, k % 4, host, cap, ci.sweep, ci.as_c(), reqs, cout.as_c())
        else:
            call(e.step_begin_compact_sweep, k % 4, ci.sweep, ci.as_c(), reqs, cout.as_c(), gids=host)
        steps[k] = (ci, cout, host, host)
        pending.append(k)
        steps.pop(k - P.DELAY - 1, None)
        if kind == "rule":
            call(e.timers_due_begin, (k + d + 1) % 4, P.now(k + d + 1), bufs[(k + d + 1) % 4].data_ptr(), G)
        listed.append(n)
        ts.append(clock[0])
    clock[0] = 0.0
    while pending:
        finish(pending.popleft())
    if kind == "rule":
        for t in range(ticks, ticks + d + 1):
            e.timers_due_wait(t % 4)
    same = bool(np.array_equal(e.digest(0, G), digest))
    e.close()
    extra = dict(state_equals_dense=same)
    if kind == "due":
        extra.update(cap0=cap0, counts3_p50=int(np.median(counts)), counts3_max=int(max(counts)), overflows=overflows)
    return _stats(kind, d, ts, up, down, listed, dev, **extra)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ticks", type=int, default=320)
    ap.add_argument("--cap0", type=int, default=4096)
    a = ap.parse_args()
    dev = device()
    P = tm.Peers(G, rows=ROWS, lost_at=150, t0=workload.T0_MS)
    inboxes, digest, res = dense_pump(P, a.ticks, dev)
    print(json.dumps(res), flush=True)
    for d in (0, 3):
        for kind in ("rule", "due"):
            print(json.dumps(compact_pump(kind, P, inboxes, a.ticks, d, a.cap0, digest, dev)), flush=True)


if __name__ == "__main__":
    main()
