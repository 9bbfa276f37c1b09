#!/usr/bin/env python
"""Secondary rates of SURVEY.md §8(d), device-resident, at BASELINE.json's full sizes on one GPU:

  config #3  256 K groups x 5 replicas, PreVote on, RequestVote storm  -> vote replies + vote requests per second
  config #5  512 K groups x 3 replicas, leader churn + InstallSnapshot catch-up
                                                                        -> acks, follower-side AE requests, entries per second

The peers are the closed-loop generators of workload.cu running on the device (the same streams the full-size
parity tests replay against the oracle); every step is generator kernel -> step kernel on the engine's stream, and
only the step kernel is inside the CUDA-event pairs (second pass over the same stream after a rollback of the tables).  Algorithmic bytes per unit are SURVEY §8(d)'s:
B_vote = 64, B_ack(R) = 184 + 8(R-2), B_req(n) = 160 + 32 n.  Prints one JSON line per configuration.

--e2e instead runs config #5 end to end through the dense host path and the compact one with its request list (run_e2e)."""
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from rafting_b200 import abi, devbatch, engine, workload  # noqa: E402
from rafting_b200.workload import _bind  # noqa: E402
import ctypes as C  # noqa: E402


def peak_gbs():
    p = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "MEASURED_PEAKS.json")
    try:
        return float(json.load(open(p))["hbm_gbs"]), "measured (MEASURED_PEAKS.json hbm_gbs)"
    except Exception:
        return 3350.0, "data sheet (H100 SXM HBM3 3.35 TB/s, not measured)"


def init_array(G, **cols):
    a = np.zeros(G, dtype=abi.GROUP_INIT_DTYPE)
    a["ballot"] = -1; a["first_index"] = 1; a["now_ms"] = workload.T0_MS - 2000
    for k, v in cols.items():
        a[k] = v
    return a


def run(name, G, R, rows, steps, seed, gen, local_slot=0, elect=False, pool=False, quiet=False):
    import torch
    F = R - 1
    dev = torch.device("cuda:0")
    cfg = abi.make_cfg(replicas=R, local_slot=local_slot, max_groups=G, max_rows=rows, pre_vote=True,
                       entry_pool_cap=workload.POOL_TERMS if pool else 0)
    e = engine.Engine(cfg)
    if name == "config3":
        e.open_bulk(0, init_array(G, term=1 + np.arange(G) % 5, last_index=100 + np.arange(G) % 50,
                                  last_term=1 + np.arange(G) % 5))
    else:
        e.open_bulk(0, init_array(G, term=np.arange(G) % 7))
    st = torch.cuda.ExternalStream(e.stream(), device=dev)
    ob = [devbatch.DevOutbox(rows, G, F, G, dev) for _ in range(2)]
    ib = devbatch.DevInbox(rows, G, F, dev, requests=True)
    pool_t = None
    if pool:
        pool_t = torch.zeros(workload.POOL_TERMS, dtype=torch.int64, device=dev)
        _bind().rafting_wl_fill_term_pool(C.c_void_p(pool_t.data_ptr()), workload.POOL_TERMS, 1, C.c_void_p(e.stream()))
    prev = None
    if elect:
        w1 = workload.make_wl(seed, 1, G, F, local_slot=local_slot)
        ib1 = devbatch.DevInbox(1, G, F, dev, requests=False)
        ob1 = [devbatch.DevOutbox(1, G, F, G, dev) for _ in range(2)]
        for ph in (0, 1, 2):
            workload.election_step(w1, ph, prev, ib1.as_c(), on_device=True, stream=e.stream())
            oc = ob1[ph & 1].as_c()
            e.step_device(ib1.as_c(), oc, e.stream())
            prev = oc
        prev = None
    w = workload.make_wl(seed, rows, G, F, local_slot=local_slot)
    # pass 0 warms the kernels of this configuration up (module load, first-launch costs); the tables are then rolled back
    # (rafting_checkpoint / rafting_restore) and pass 1 — the identical stream, the generators are pure functions of the
    # previous outbox — is the timed one
    e.checkpoint()
    for timed in (False, True):
        if timed:
            e.restore()
        prev = None
        tot = dict(acks=0, votes=0, vote_requests=0, ae_requests=0, is_requests=0, entries=0, ops_other=0)
        ms = []
        with torch.cuda.stream(st):
            for k in range(steps):
                ic = ib.as_c()
                if pool:
                    ic.ent_terms = pool_t.data_ptr(); ic.ent_count = workload.POOL_TERMS
                rc = gen(C.byref(w), k, None if prev is None else C.byref(prev), C.byref(ic), 1, C.c_void_p(e.stream()))
                assert rc == 0, rc
                oc = ob[k & 1].as_c()
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record(st)
                e.step_device(ic, oc, e.stream())
                b.record(st)
                b.synchronize()
                ms.append(a.elapsed_time(b))
                prev = oc
                evk = ib.t["ev_meta"].view(torch.int64) & 0xF
                opm = ib.t["op_meta"].view(torch.int64)
                opk = opm & 0xFF
                tot["acks"] += int(((evk == abi.EV_AE_ACK) | (evk == abi.EV_IS_ACK)).sum())
                tot["votes"] += int(((evk == abi.EV_PV_REPLY) | (evk == abi.EV_RV_REPLY)).sum())
                tot["vote_requests"] += int(((opk == abi.OP_PREVOTE_REQ) | (opk == abi.OP_VOTE_REQ)).sum())
                ae = opk == abi.OP_AE_REQUEST
                tot["ae_requests"] += int(ae.sum())
                tot["entries"] += int((((opm >> 16) & 0xFFFF) * ae).sum())
                tot["is_requests"] += int((opk == abi.OP_IS_REQUEST).sum())
                tot["ops_other"] += int(((opk == abi.OP_SUBMIT) | (opk == abi.OP_TIMEOUT) | (opk == abi.OP_FLUSH)).sum())
    role = ob[(steps - 1) & 1].t["role_word"].view(torch.int32) & 3
    err = (ob[(steps - 1) & 1].t["err_word"].view(torch.int32) & 0xFFFF) != 0
    secs = sum(ms) * 1e-3
    peak, src = peak_gbs()
    b_ack = 184 + 8 * (R - 2)
    alg = tot["acks"] * b_ack + (tot["votes"] + tot["vote_requests"]) * 64 + \
        (tot["ae_requests"] + tot["is_requests"]) * 160 + tot["entries"] * 32
    rec = {
        "config": name, "groups": G, "replicas": R, "rows_per_step": rows, "steps": steps, "seed": hex(seed),
        "kernel_ms_total": sum(ms), "kernel_ms_per_step_median": float(np.median(ms)),
        "units": tot,
        "rates_per_s": {k: v / secs for k, v in tot.items() if v},
        "roofline": {"bound": "hbm", "algorithmic_bytes": alg, "achieved": alg / secs / 1e9, "peak": peak, "unit": "GB/s",
                     "frac": alg / secs / 1e9 / peak, "peak_source": src,
                     "bytes_per_unit": {"ack": b_ack, "vote": 64, "request": "160 + 32 n"}},
        "end_state": {"roles": torch.bincount(role.long(), minlength=3).tolist(), "groups_with_error": int(err.sum())},
    }
    if not quiet:
        print(json.dumps(rec), flush=True)
    e.close()
    return rec


def run_all(quiet=False, steps5=64):
    L = _bind()
    return [run("config3", 262144, 5, 1, 8, 0x5EED0003, L.rafting_wl_vote_step, local_slot=2, quiet=quiet),
            run("config5", 524288, 3, 4, steps5, 0x5EED0005, L.rafting_wl_mixed_step, elect=True, pool=True, quiet=quiet)]


def card():
    import subprocess
    import torch
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return {"name": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip().splitlines()[0] if q.returncode == 0 else None}


def run_e2e(G=524288, R=3, rows=4, settle=24, window=12, passes=3, seed=0x5EED0005):
    """config #5 end to end through two host paths.  A window of launches is recorded on the device path; each host path then
    replays it from pinned caller-owned buffers filled before the clock starts, four launches in flight:
      dense    rafting_step_begin_host: every inbox / outbox column, the sparse ones when the step produced any
      compact  rafting_step_begin_compact_req: ev_c / op_c words, AppendEntries as 32-byte records, every other request as an
               op escape, replies in rep_c
    Launch 0 of the window answers RPCs planned on the device path (no tags): it runs once, untimed, and the state after it
    is where every timed pass starts.  Both paths must end in the device path's state."""
    import time
    import torch
    from rafting_b200 import compact
    F, NSL = R - 1, 4
    dev = torch.device("cuda:0")
    L = _bind()
    inboxes, reqs, cins = [], [], []
    # ---- record the window on the device path ----
    e = engine.Engine(abi.make_cfg(replicas=R, max_groups=G, max_rows=rows, entry_pool_cap=rows * G * 50))
    e.open_bulk(0, init_array(G, term=np.arange(G) % 7))
    ib = devbatch.DevInbox(rows, G, F, dev, requests=True)
    ob = [devbatch.DevOutbox(rows, G, F, G, dev) for _ in range(2)]
    pool_t = torch.zeros(workload.POOL_TERMS, dtype=torch.int64, device=dev)
    L.rafting_wl_fill_term_pool(C.c_void_p(pool_t.data_ptr()), workload.POOL_TERMS, 1, C.c_void_p(e.stream()))
    w1 = workload.make_wl(seed, 1, G, F)
    ib1, ob1, prev = devbatch.DevInbox(1, G, F, dev), [devbatch.DevOutbox(1, G, F, G, dev) for _ in range(2)], None
    for ph in (0, 1, 2):
        workload.election_step(w1, ph, prev, ib1.as_c(), on_device=True, stream=e.stream())
        prev = ob1[ph & 1].as_c()
        e.step_device(ib1.as_c(), prev, e.stream())
    w = workload.make_wl(seed, rows, G, F)
    prev = None
    pool_h = pool_t.cpu().numpy()
    for k in range(settle + window):
        ic = ib.as_c()
        ic.ent_terms, ic.ent_count = pool_t.data_ptr(), workload.POOL_TERMS
        assert L.rafting_wl_mixed_step(C.byref(w), k, None if prev is None else C.byref(prev), C.byref(ic), 1, C.c_void_p(e.stream())) == 0
        if k == settle:
            torch.cuda.synchronize(); e.checkpoint()                      # the state at the start of the window
        if k >= settle:
            torch.cuda.synchronize()                                       # the generator ran on the engine's stream
            h = abi.Inbox(rows, G, F, with_ops=False, with_events=False)
            for name, dt, lane in (("op_meta", np.uint64, 0), ("op_nr", abi.I64X2, 0), ("op_ab", abi.I64X2, 0), ("op_cd", abi.I64X2, 0),
                                   ("op_e", np.int64, 0), ("ev_meta", np.uint64, 1), ("ev_tn", abi.I64X2, 1), ("ev_el", abi.I64X2, 1)):
                setattr(h, name, ib.t[name].cpu().numpy().view(dt).reshape((rows, G, F) if lane else (rows, G)))
            h.ent_terms, h.ent_count = pool_h, workload.POOL_TERMS
            inboxes.append(h)
        prev = ob[k & 1].as_c()
        e.step_device(ic, prev, e.stream())
    torch.cuda.synchronize()
    digest_dev = e.digest(0, G)
    del ib, ob, ib1, ob1
    e.restore()
    enc0 = compact.encode_inbox(inboxes[0], None, None, None)
    ESC_CAP = rows * G * F // 8
    cout0 = compact.CompactOutbox(rows, G, F, esc_cap=rows * G * (F + 2))
    e.step_compact(enc0, cout0, reqs=enc0.reqs if enc0.reqs is not None else compact.CompactRequests())   # launch 0, untimed
    e.checkpoint()
    tags, sent_term, sent_inc = cout0.tags(), cout0.current_term.copy(), cout0.incarnation.copy()
    _, out_off = engine.Engine.compact_layout(rows, G, F, 0, ESC_CAP)
    keep, couts = [], []
    for sl in range(NSL):
        t = torch.zeros(int(out_off[11]), dtype=torch.uint8).pin_memory(); keep.append(t)
        couts.append(compact.outbox_in_block(t.numpy(), out_off, rows, G, F, ESC_CAP))
    up_c, esc_in, esc_out, acks, ae, entries = [], [], [], 0, 0, 0
    for k in range(1, window):                                            # record pass (untimed): the tags the engine hands out
        ci = compact.encode_inbox(inboxes[k], tags, sent_term, sent_inc)
        q = ci.reqs if ci.reqs is not None else compact.CompactRequests()
        in_off, _ = engine.Engine.compact_layout(rows, G, F, len(ci.esc), ESC_CAP)
        t = torch.zeros(int(in_off[5]), dtype=torch.uint8).pin_memory(); keep.append(t)
        ci = compact.inbox_in_block(t.numpy(), in_off, ci)
        r_off = engine.Engine.compact_req_layout(len(q.req), len(q.op_esc), len(q.ent_terms))
        t = torch.zeros(max(1, int(r_off[3])), dtype=torch.uint8).pin_memory(); keep.append(t)
        blk = t.numpy()
        views = []
        for a, off in ((q.req, r_off[0]), (q.op_esc, r_off[1]), (q.ent_terms, r_off[2])):
            v = blk[int(off):int(off) + a.nbytes].view(a.dtype)
            v[...] = a
            views.append(v)
        q = compact.CompactRequests(*views)
        e.step_compact(ci, couts[0], reqs=q)
        if int(couts[0].counts[0]) > ESC_CAP:
            raise SystemExit(f"launch {k} produced {int(couts[0].counts[0])} escape records (> {ESC_CAP})")
        tags, sent_term, sent_inc = couts[0].tags(), couts[0].current_term.copy(), couts[0].incarnation.copy()
        cins.append(ci.as_c()); reqs.append(q.as_c())
        span = (in_off[4] + len(ci.esc) * abi.CESC_IN.itemsize) if len(ci.esc) else (in_off[3] + ci.ev_c.nbytes)
        up_c.append(span + (int(r_off[3]) if len(q.req) or len(q.op_esc) else 0))
        esc_in.append((len(ci.esc), len(q.op_esc))); esc_out.append(int(couts[0].counts[0]))
        h = inboxes[k]
        evk = (h.ev_meta & np.uint64(0xF)).astype(np.int64)
        opk = (h.op_meta & np.uint64(0xFF)).astype(np.int64)
        acks += int(((evk == abi.EV_AE_ACK) | (evk == abi.EV_IS_ACK)).sum())
        ae += int((opk == abi.OP_AE_REQUEST).sum())
        entries += int((((h.op_meta >> np.uint64(16)) & np.uint64(0xFFFF)).astype(np.int64) * (opk == abi.OP_AE_REQUEST)).sum())
    digest_rec = e.digest(0, G)
    cout_c = [co.as_c() for co in couts]
    n = window - 1

    def compact_pass():
        for j in range(n):
            sl = j % NSL
            if j >= NSL:
                e.step_wait_compact(sl)
            e.step_begin_compact_req(sl, cins[j], reqs[j], cout_c[sl])
        for sl in range(NSL):
            e.step_wait_compact(sl)

    # the dense host path: every launch's columns pinned
    host_in, host_out = [], []
    for k in range(1, window):
        h = inboxes[k]
        cols = {name: torch.from_numpy(np.ascontiguousarray(getattr(h, name)).view(np.uint8).reshape(-1)).pin_memory()
                for name in ("op_meta", "op_nr", "op_ab", "op_cd", "op_e", "ev_meta", "ev_tn", "ev_el")}
        cols["ent_terms"] = torch.from_numpy(pool_h.view(np.uint8).copy()).pin_memory()
        ic = abi.InboxC()
        ic.rows, ic.n_active, ic.flags, ic.ent_count = rows, 0, 0, workload.POOL_TERMS
        for name, t in cols.items():
            setattr(ic, name, t.data_ptr())
        host_in.append((cols, ic))
    for sl in range(NSL):
        o = devbatch.DevOutbox(rows, G, F, G, "cpu")
        cols = {name: t.pin_memory() for name, t in o.t.items()}
        oc = abi.OutboxC()
        for name, t in cols.items():
            setattr(oc, name, t.data_ptr())
        host_out.append((cols, oc))
    up_d = sum(t.numel() for t in host_in[0][0].values())
    down_d = sum(t.numel() for t in host_out[0][0].values()) + 16

    def dense_pass():
        for j in range(n):
            sl = j % NSL
            if j >= NSL:
                e.step_wait_slot(sl)
            e.step_begin_host(sl, host_in[j][1], host_out[sl][1])
        for sl in range(NSL):
            e.step_wait_slot(sl)

    res = {}
    for name, fn in (("dense", dense_pass), ("compact", compact_pass)):
        e.restore(); fn()                                                 # untimed: every slot's staging exists before the clock
        exact = bool((e.digest(0, G) == digest_dev).all())
        t0 = time.perf_counter()
        for _ in range(passes):
            e.restore(sync=False)
            fn()
        spent = time.perf_counter() - t0
        exact = exact and bool((e.digest(0, G) == digest_dev).all())
        res[name] = {"acks_per_s": acks * passes / spent, "ae_requests_per_s": ae * passes / spent, "entries_per_s": entries * passes / spent,
                     "launches": n * passes, "exact": exact}
    res["dense"].update({"path": "rafting_step_begin_host", "h2d_bytes_per_launch": int(up_d), "d2h_bytes_per_launch": int(down_d)})
    res["compact"].update({"path": "rafting_step_begin_compact_req", "h2d_bytes_per_launch": int(np.mean(up_c)),
                           "d2h_bytes_per_launch": int(out_off[10] + 256 * abi.CESC_OUT.itemsize + max(0, np.mean(esc_out) - 256) * abi.CESC_OUT.itemsize),
                           "escape_records_in_per_launch": {"events": float(np.mean([x[0] for x in esc_in])), "ops": float(np.mean([x[1] for x in esc_in]))}, "escape_records_out_per_launch": float(np.mean(esc_out))})
    rec = {"config": "config5_e2e", "groups": G, "replicas": R, "rows_per_launch": rows, "window_launches": n, "passes": passes,
           "launches_in_flight": NSL, "units_per_launch": {"acks": acks / n, "ae_requests": ae / n, "entries": entries / n},
           "record_pass_exact": bool((digest_rec == digest_dev).all()), "card": card(), **res}
    print(json.dumps(rec), flush=True)
    return rec


def main():
    if "--e2e" in sys.argv[1:]:
        run_e2e()
    else:
        run_all()


if __name__ == "__main__":
    main()
