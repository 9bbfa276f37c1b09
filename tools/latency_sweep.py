#!/usr/bin/env python
"""p50 / p99 commitIndex latency as a function of the batch size (SURVEY.md §8d: "batch interval is a swept
parameter: 1 k ... 1 M events/step").  One synchronous host-path step per sample: acks are written into pinned
buffers, rafting_step_begin_host + rafting_step_wait_slot run, and the clock stops when the commit column is
readable on the host.  The stream is the closed-loop leader stream restricted to an active list of groups.
Prints one JSON line per (groups in the step, rows).

--compact: beside each dense line, the same traffic through the compact host path twice, each on a freshly elected engine:
  compact_whole_shard  rafting_step_begin_compact over all max_groups groups (the idle ones carry empty words)
  compact_active       rafting_step_begin_compact_active over the active list only
Every line then carries bytes up / down per launch (from the column sizes and rafting_compact_layout: what the copies move)
and escape records per launch (up and down).
--configs i,j,...: run only those entries of the sweep (0-based), e.g. to split it over several invocations."""
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from rafting_b200 import abi, compact, engine, workload  # noqa: E402

STEPS, WARM = 60, 10


def pinned(nbytes):
    import torch
    t = torch.zeros(max(int(nbytes), 1), dtype=torch.uint8).pin_memory()
    return t, t.numpy()


def caller_owned(e, w, rows, n, F, G, gids, lat):
    import torch
    # pinned host batch buffers owned by the caller
    def pinned(shape, dt):
        t = torch.zeros(int(np.prod(shape)) * np.dtype(dt).itemsize, dtype=torch.uint8).pin_memory()
        return t, np.frombuffer(t.numpy(), dtype=dt).reshape(shape)
    ib = abi.Inbox(rows, n, F, gids=gids); ib.flags = abi.INBOX_NO_REQUESTS
    ob = abi.Outbox(rows, n, F, G)
    keep = []
    for obj, names in ((ib, ("op_meta", "op_nr", "op_ab", "ev_meta", "ev_tn", "ev_el")),
                       (ob, [c[0] for c in abi.Outbox.ROW_COLS] + [c[0] for c in abi.Outbox.GROUP_COLS])):
        for name in names:
            a = getattr(obj, name)
            t, v = pinned(a.shape, a.dtype)
            keep.append(t); setattr(obj, name, v)
    ib.op_cd = None; ib.op_e = None
    prev_out = None
    for k in range(STEPS):
        ic = ib.as_c(); ic.op_cd = None; ic.op_e = None
        workload.leader_step(w, k, None if prev_out is None else prev_out.as_c(), ic)      # the peers (not timed)
        oc = ob.as_c()
        t0 = time.perf_counter()
        e.step_begin_host(0, ic, oc)
        e.step_wait_slot(0)
        _ = int(ob.commit_index[0])                                                      # commit column readable
        dt = time.perf_counter() - t0
        if k >= WARM:
            lat.append(dt * 1e3)
        prev_out = ob
    up = sum(getattr(ib, c).nbytes for c in ("op_meta", "op_nr", "op_ab", "ev_meta", "ev_tn", "ev_el")) + (0 if gids is None else gids.nbytes)
    down = sum(getattr(ob, c).nbytes for c in ("rep_meta", "plan_meta", "plan_pp", "plan_lc", "plan_epoch", "ballot_meta")) + \
        sum(getattr(ob, c[0]).nbytes for c in abi.Outbox.GROUP_COLS) + 16        # the sparse columns travel only when flagged
    return int(((ib.ev_meta & np.uint64(0xF)) != 0).sum()), dict(bytes_up=up, bytes_down=down)


def _listed(o: abi.Outbox, gids):
    """a whole-shard outbox seen from an active step over gids: its rows and group columns at the listed groups, by position"""
    a = abi.Outbox(o.rows, len(gids), o.F, len(gids))
    for name, _, _ in abi.Outbox.ROW_COLS:
        getattr(a, name)[...] = getattr(o, name)[:, gids]
    for name, _ in abi.Outbox.GROUP_COLS:
        getattr(a, name)[...] = getattr(o, name)[gids]
    return a


def compact_path(e, w, rows, F, G, gids, active, lat):
    """The leader stream over gids through the compact path: over the active list, or scattered into whole-shard steps.
    Both blocks are pinned and carved by rafting_compact_layout, so each launch is one copy up (two with a list) and one down."""
    n = len(gids) if active else G
    esc_cap = rows * n * F + 2 * rows * n
    _, out_off = engine.Engine.compact_layout(rows, n, F, 0, esc_cap)
    keep_out, ob = pinned(out_off[11])
    cout = compact.outbox_in_block(ob, out_off, rows, n, F, esc_cap, gids=gids if active else None)
    blk_in = None
    prev, tags, sent_term, sent_inc = None, None, None, None
    acks = up = down = esc_up = esc_down = 0
    for k in range(STEPS):
        ib = workload.leader_inbox_host(w, k, prev, gids=gids)                          # the peers (not timed)
        if not active:
            full = abi.Inbox(rows, G, F)
            full.flags = abi.INBOX_NO_REQUESTS
            full.op_cd = full.op_e = None
            for name in ("op_meta", "op_nr", "op_ab", "ev_meta", "ev_tn", "ev_el"):
                getattr(full, name)[:, gids] = getattr(ib, name)
            ib = full
        ci = compact.encode_inbox(ib, tags, sent_term, sent_inc)
        in_off, _ = engine.Engine.compact_layout(rows, n, F, len(ci.esc), esc_cap)
        if blk_in is None or blk_in[1].nbytes < in_off[5]:
            blk_in = pinned(in_off[5] * 2)
        cin = compact.inbox_in_block(blk_in[1], in_off, ci)
        t0 = time.perf_counter()
        e.step_compact(cin, cout)
        _ = int(cout.commit_index[0])                                                    # commit column readable
        dt = time.perf_counter() - t0
        nesc = int(cout.counts[0])
        got = compact.decode_outbox(cout)
        if k >= WARM:
            lat.append(dt * 1e3)
            acks += int(((ib.ev_meta & np.uint64(0xF)) != 0).sum())
            span_in = in_off[4] + len(ci.esc) * abi.CESC_IN.itemsize if len(ci.esc) else in_off[3] + rows * n * F * 4
            up += span_in + (n * 4 if active else 0)
            down += out_off[10] + max(min(nesc, esc_cap), min(esc_cap, 256)) * abi.CESC_OUT.itemsize
            esc_up += len(ci.esc)
            esc_down += nesc
        prev = got if active else _listed(got, gids)
        tags, sent_term, sent_inc = cout.tags(), cout.current_term.copy(), cout.incarnation.copy()
    m = STEPS - WARM
    return acks // m, dict(bytes_up=up // m, bytes_down=down // m, esc_records_up=esc_up / m, esc_records_down=esc_down / m)


COMPACT = "--compact" in sys.argv


LEASE = "--lease" in sys.argv


def main():
    G, R = 65536, 3
    F = R - 1
    out = []
    sweep = ((512, 1), (4096, 1), (65536, 1), (4096, 16), (65536, 4), (65536, 16))
    if "--configs" in sys.argv:
        sweep = [sweep[int(i)] for i in sys.argv[sys.argv.index("--configs") + 1].split(",")]
    for n_act, rows in sweep:
        cfg = abi.make_cfg(replicas=R, max_groups=G, max_rows=rows)
        gids = None if n_act == G else np.arange(0, G, G // n_act, dtype=np.uint32)[:n_act]
        n = G if gids is None else len(gids)

        def elected():
            e = engine.Engine(cfg)
            init = np.zeros(G, dtype=abi.GROUP_INIT_DTYPE)
            init["ballot"] = -1; init["first_index"] = 1; init["now_ms"] = workload.T0_MS - 2000
            init["term"] = np.arange(G) % 7
            e.open_bulk(0, init)
            w1 = workload.make_wl(0x5EED0002, 1, n, F)
            prev = None
            for ph in (0, 1, 2):                                   # election through the lease path
                ib = abi.Inbox(1, n, F, gids=gids); ib.flags = abi.INBOX_NO_REQUESTS
                ic = ib.as_c(); ic.op_cd = None; ic.op_e = None
                workload.election_step(w1, ph, None if prev is None else prev.as_c(), ic)
                ib.op_cd = None; ib.op_e = None
                prev = e.step(ib)
            return e
        e = elected()
        w = workload.make_wl(0x5EED0002, rows, n, F)
        lat = []
        extra = {}
        if LEASE:
            # engine-owned pinned columns: one contiguous block per direction, so the step is 1 (+1 for an active
            # list) copy up and 1 copy down; with an active list the group columns are compact (n entries, not G)
            prev_c = None
            ev_meta = None
            for k in range(60):
                fl = abi.INBOX_NO_REQUESTS | (0 if gids is None else abi.INBOX_COMPACT_GROUPS)
                L = e.lease(rows, 0 if gids is None else n, 0, fl)
                if gids is not None:
                    L.gids[:] = gids
                L.use(ops=True, events=True, flags=fl)
                ic = L.c.inbox; ic.op_cd = None; ic.op_e = None
                workload.leader_step(w, k, prev_c, ic)                                        # the peers (not timed)
                t0 = time.perf_counter()
                L.begin(); L.wait()
                _ = int(L.out.commit_index[0])
                dt = time.perf_counter() - t0
                if k >= 10:
                    lat.append(dt * 1e3)
                prev_keep = L.outbox_copy(); prev_c = prev_keep.as_c()
                ev_meta = L.ev_meta
            acks = int(((ev_meta & np.uint64(0xF)) != 0).sum())
        else:
            acks, extra = caller_owned(e, w, rows, n, F, G, gids, lat)
        rec = {"path": "dense", "buffers": "lease" if LEASE else "caller", "groups_in_step": n, "rows": rows, "acks_per_step": acks, "p50_ms": float(np.percentile(lat, 50)),
               "p99_ms": float(np.percentile(lat, 99)), "acks_per_s_at_p50": acks / (np.percentile(lat, 50) * 1e-3), **extra}
        print(json.dumps(rec), flush=True)
        out.append(rec)
        e.close()
        if not COMPACT:
            continue
        listed = np.arange(G, dtype=np.uint32) if gids is None else gids
        wl = workload.make_wl(0x5EED0002, rows, G, F)                  # keyed by gid: the same traffic as the dense line
        for active in (False, True):
            e, lat = elected(), []
            acks, extra = compact_path(e, wl, rows, F, G, listed, active, lat)
            rec = {"path": "compact_active" if active else "compact_whole_shard", "groups_in_step": n, "rows": rows, "acks_per_step": acks,
                   "p50_ms": float(np.percentile(lat, 50)), "p99_ms": float(np.percentile(lat, 99)),
                   "acks_per_s_at_p50": acks / (np.percentile(lat, 50) * 1e-3), **extra}
            print(json.dumps(rec), flush=True)
            out.append(rec)
            e.close()


if __name__ == "__main__":
    main()
