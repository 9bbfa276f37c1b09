"""What getting a step's AppendEntries payloads costs a compact pump: config #2's leader stream (64 K groups x 3 replicas,
workload.leader_inbox_host) through compact whole-shard steps, each step's SUBMITs appended as 256-byte payloads after its
wait, then the payloads of the step's plans fetched two ways:

  host     decode the compact outbox's AE ranges on the host (compact.ae_ranges: plan_c words and escape records), then
           rafting_log_gather over them (per-entry lookups and requests built on one host core)
  device   rafting_log_gather_step_begin / _wait: the plans walked, probed and copied on the device

Both write into the same pinned buffers, and every step their refs and payloads are checked to agree.  Per path it reports
the wall time from the first call to the return of the last (p50 / p99 over the timed steps), entries/s and bytes/s at p50,
and the median device time of the path's kernels (CUDA events, rafting_log_stats), with the device name, power limit and
max SM clock read in the same run.  One JSON line.

    python tools/bench_step_gather.py [--steps 40] [--warmup 5] [--groups 65536] [--rows 4]"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from rafting_b200 import abi, compact, engine, workload  # noqa: E402
from tests import harness  # noqa: E402

PAYLOAD = 256


def device():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True).stdout.strip()
    except OSError:
        return "unknown"


def pinned(nbytes, dtype):
    import torch
    t = torch.zeros(nbytes, dtype=torch.uint8, pin_memory=True)
    a = t.numpy().view(dtype)
    return a, t


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=40)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--groups", type=int, default=65536)
    ap.add_argument("--rows", type=int, default=4)
    a = ap.parse_args()
    G, R, rows, F = a.groups, 3, a.rows, 2
    cfg = abi.make_cfg(replicas=R, max_groups=G, max_rows=rows)
    e = engine.Engine(cfg)
    e.open_bulk(0, harness.init_array(G, terms=np.arange(G) % 7))
    e.log_config(segment_bytes=1 << 24, hbm_segments=64, ring_slots=256)
    last = harness.elect_all(e, workload.make_wl(0x5EED0002, 1, G, F))
    w = workload.make_wl(0x5EED0002, rows, G, F)
    cap = G * F * 8                                 # refs the pinned buffers hold; grown between steps when a step needs more
    refs, _k1 = pinned(cap * 32, engine.Engine.ENTRY_REF)
    blob, _k2 = pinned(cap * PAYLOAD, np.uint8)
    plans, _k3 = pinned(rows * G * F * 16, abi.PLAN_REF)
    payload = np.random.default_rng(1).integers(0, 256, PAYLOAD * 4096, dtype=np.uint8)
    appended = np.zeros(G, np.int64)
    L = engine.lib()
    tags = sent_term = sent_inc = None
    host_ms, dev_ms, host_k, dev_k, n_ent, n_bytes = [], [], [], [], [], []
    for k in range(a.warmup + a.steps):
        ib = workload.leader_inbox_host(w, k, last)
        ci = compact.encode_inbox(ib, tags, sent_term, sent_inc)
        cout = compact.CompactOutbox(rows, G, F, esc_cap=rows * G * R)
        e.step_compact(ci, cout)
        last = compact.decode_outbox(cout)
        tags, sent_term, sent_inc = cout.tags(), cout.current_term.copy(), cout.incarnation.copy()
        # the payloads of the entries the step's SUBMITs created (the newest 64 of a longer run, after the election)
        hi = cout.last_entry["x"]
        lo = np.maximum(appended, hi - 64)
        cnt = np.maximum(hi - lo, 0)
        gids = np.repeat(np.arange(G), cnt)
        idx = np.repeat(lo, cnt) + 1 + (np.arange(cnt.sum()) - np.repeat(np.cumsum(cnt) - cnt, cnt))
        appended = np.maximum(appended, hi)
        if len(gids):
            ar = np.zeros(len(gids), engine.Engine.ENTRY_REF)
            ar["gid"], ar["len"], ar["index"] = gids, PAYLOAD, idx
            ar["term"] = cout.current_term[gids]
            ar["blob_off"] = (np.arange(len(gids)) % 4096) * PAYLOAD
            rc = L.rafting_log_append(e._h, ar.ctypes.data, len(ar), payload.ctypes.data, payload.nbytes)
            assert rc == 0, engine.lib().rafting_last_error()
        if int(compact.ae_ranges(cout)[3].sum()) > cap:
            cap = 2 * int(compact.ae_ranges(cout)[3].sum())
            refs, _k1 = pinned(cap * 32, engine.Engine.ENTRY_REF)
            blob, _k2 = pinned(cap * PAYLOAD, np.uint8)
        # host: decode, then rafting_log_gather
        t0 = time.perf_counter()
        _, g, f, c = compact.ae_ranges(cout)
        g32, c32 = g.astype(np.uint32), c.astype(np.uint32)
        n, nb = C.c_uint32(), C.c_size_t()
        rc = L.rafting_log_gather(e._h, len(g32), g32.ctypes.data, f.ctypes.data, c32.ctypes.data, refs.ctypes.data, cap,
                                  blob.ctypes.data, blob.nbytes, C.byref(n), C.byref(nb))
        t1 = time.perf_counter()
        assert rc == 0, engine.lib().rafting_last_error()
        want_refs = refs[:n.value][["gid", "len", "index", "term"]].copy()
        want_off = refs[:n.value]["blob_off"].copy()
        want_blob = blob[:nb.value].copy()
        hk = e.log_stats()["gather_kernel_ns"] / 1e6
        # device: rafting_log_gather_step_begin / _wait
        t2 = time.perf_counter()
        e.log_gather_step_begin(0, refs, blob, plans, refs_cap=cap)
        nr, nbytes, _, served = e.log_gather_step_wait(0)
        t3 = time.perf_counter()
        dk = e.log_stats()["gather_kernel_ns"] / 1e6
        got = refs[:nr]
        assert nr == n.value and np.array_equal(got[["gid", "len", "index", "term"]], want_refs), f"step {k}: refs differ"
        ok = got["len"] != 0xFFFFFFFF
        for r_off, w_off, ln in zip(got["blob_off"][ok][:64], want_off[ok][:64], got["len"][ok][:64]):
            assert np.array_equal(blob[r_off:r_off + ln], want_blob[w_off:w_off + ln]), f"step {k}: payload differs"
        if k >= a.warmup:
            host_ms.append((t1 - t0) * 1e3); dev_ms.append((t3 - t2) * 1e3)
            host_k.append(hk); dev_k.append(dk); n_ent.append(nr); n_bytes.append(nbytes)
    p = lambda v, q: float(np.percentile(v, q))  # noqa: E731
    ent, byt = float(np.median(n_ent)), float(np.median(n_bytes))
    print(json.dumps({
        "bench": "step_gather", "groups": G, "replicas": R, "rows": rows, "payload_bytes": PAYLOAD, "steps": a.steps,
        "entries_per_step": ent, "bytes_per_step": byt,
        "host_path_ms_p50": p(host_ms, 50), "host_path_ms_p99": p(host_ms, 99),
        "device_path_ms_p50": p(dev_ms, 50), "device_path_ms_p99": p(dev_ms, 99),
        "host_path_entries_per_s": ent / (p(host_ms, 50) / 1e3), "device_path_entries_per_s": ent / (p(dev_ms, 50) / 1e3),
        "host_path_bytes_per_s": byt / (p(host_ms, 50) / 1e3), "device_path_bytes_per_s": byt / (p(dev_ms, 50) / 1e3),
        "host_path_gather_kernel_ms_p50": float(np.median(host_k)), "device_path_kernels_ms_p50": float(np.median(dev_k)),
        "device": device()}))


if __name__ == "__main__":
    main()
