"""What getting a step's committed entries for RaftMachine.apply costs a compact pump, two ways, on the same ranges:

  host     rafting_log_gather: a host-index lookup and a request per entry, one kernel, and the calling thread blocked until
           the bytes are down
  device   rafting_log_gather_begin / _wait: one record per range from the host, then probe, layout and copy on the device;
           the host serves only what the ring does not hold

Streams: config #2 (64 K groups x 3, the leader stream) and config #5 (512 K groups x 3, the mixed stream with inbound
requests), through compact whole-shard steps.  After each step's wait the entries it created get payloads of 64-256 bytes
(rafting_log_append), rafting_outbox_apply_ranges turns its commit records into apply ranges, and after a warm-up the two
paths gather them alternately (which one goes first alternates too), into the same pinned buffers; every step their refs and
payloads are checked to agree.  Per path: wall time (p50 / p99 / min / max over the timed steps), host CPU time inside the
calls, the kernels' device time (rafting_log_stats), entries, bytes and host-served entries per step.  `--rounds` repeats
everything in one process; the device name, power limit and max SM clock are read in the same run.  One JSON line per
configuration and round.

    python tools/bench_apply_gather.py [--rounds 3] [--steps 16] [--warmup 4]"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from rafting_b200 import abi, compact, engine, ingest, workload  # noqa: E402
from tests import harness  # noqa: E402

CONFIGS = {2: (65536, 4, 0x5EED0002, workload.leader_inbox_host), 5: (524288, 4, 0x5EED0005, workload.mixed_inbox_host)}


def device():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True).stdout.strip()
    except OSError:
        return "unknown"


def pinned(nbytes, dtype):
    import torch
    t = torch.zeros(max(nbytes, 16), dtype=torch.uint8, pin_memory=True)
    return t.numpy()[:nbytes].view(dtype), t


def run(config: int, steps: int, warmup: int, seed: int):
    G, rows, wseed, inbox = CONFIGS[config]
    R, F = 3, 2
    cfg = abi.make_cfg(replicas=R, max_groups=G, max_rows=rows, entry_pool_cap=workload.POOL_TERMS)
    e = engine.Engine(cfg)
    e.open_bulk(0, harness.init_array(G, terms=np.arange(G) % 7))
    e.log_config(segment_bytes=1 << 24, hbm_segments=96, ring_slots=64)
    last = harness.elect_all(e, workload.make_wl(wseed, 1, G, F))
    w = workload.make_wl(wseed, rows, G, F)
    rng = np.random.default_rng(seed)
    pool = rng.integers(0, 256, 1 << 22, dtype=np.uint8)
    appended, applied = np.zeros(G, np.int64), np.zeros(G, np.int64)
    cap = 1 << 20
    refs, _k1 = pinned(cap * 32, engine.Engine.ENTRY_REF)
    blob, _k2 = pinned(cap * 272, np.uint8)
    L = engine.lib()
    res = {p: {"wall_ms": [], "cpu_ms": [], "kernel_ms": [], "served": []} for p in ("host", "device")}
    n_ent, n_bytes, n_ranges = [], [], []
    tags = sent_term = sent_inc = None
    for k in range(warmup + steps):
        ib = inbox(w, k, last)
        ci = compact.encode_inbox(ib, tags, sent_term, sent_inc)
        cout = compact.CompactOutbox(rows, G, F, esc_cap=rows * G * R)
        e.step_compact(ci, cout)
        last = compact.decode_outbox(cout)
        tags, sent_term, sent_inc = cout.tags(), cout.current_term.copy(), cout.incarnation.copy()
        # payloads of 64-256 bytes for the entries the step created (leaders' SUBMITs, followers' accepted entries)
        hi = cout.last_entry["x"]
        cnt = np.maximum(hi - appended, 0)
        if cnt.sum():
            gids = np.repeat(np.arange(G), cnt)
            idx = np.repeat(appended, cnt) + 1 + (np.arange(cnt.sum()) - np.repeat(np.cumsum(cnt) - cnt, cnt))
            ar = np.zeros(len(gids), engine.Engine.ENTRY_REF)
            ar["gid"], ar["index"], ar["term"] = gids, idx, cout.current_term[gids]
            ar["len"] = rng.integers(64, 257, len(gids))
            ar["blob_off"] = rng.integers(0, (len(pool) - 256) // 16, len(gids)) * 16
            assert L.rafting_log_append(e._h, ar.ctypes.data, len(ar), pool.ctypes.data, pool.nbytes) == 0, L.rafting_last_error()
        appended = np.maximum(appended, hi)
        ob = abi.Outbox(1, G, F, G)
        ob.commit_index[:], ob.role_word[:] = cout.commit_index, cout.role_word
        a = ingest.apply_ranges(ob, applied)
        g, f = a["gid"].astype(np.uint32), a["first"].astype(np.int64)
        c = (a["last"] - a["first"] + 1).astype(np.uint32)
        N = int(c.sum())
        if N > cap:
            cap = 2 * N
            refs, _k1 = pinned(cap * 32, engine.Engine.ENTRY_REF)
            blob, _k2 = pinned(cap * 272, np.uint8)
        if k < warmup or len(g) == 0:
            continue
        out = {}
        for path in (("host", "device") if k % 2 else ("device", "host")):
            w0, c0 = time.perf_counter(), time.thread_time()
            if path == "host":
                n, nb = C.c_uint32(), C.c_size_t()
                rc = L.rafting_log_gather(e._h, len(g), g.ctypes.data, f.ctypes.data, c.ctypes.data, refs.ctypes.data, cap,
                                          blob.ctypes.data, blob.nbytes, C.byref(n), C.byref(nb))
                assert rc == 0, L.rafting_last_error()
                got, served = (n.value, nb.value), -1
            else:
                e.log_gather_begin(0, (g, f, c), refs, blob, refs_cap=cap)
                nr, nbytes, served = e.log_gather_wait(0)
                got = (nr, nbytes)
            w1, c1 = time.perf_counter(), time.thread_time()
            r = res[path]
            r["wall_ms"].append((w1 - w0) * 1e3); r["cpu_ms"].append((c1 - c0) * 1e3)
            r["kernel_ms"].append(e.log_stats()["gather_kernel_ns"] / 1e6); r["served"].append(served)
            sample = rng.choice(got[0], min(got[0], 256), replace=False)
            out[path] = (got, refs[:got[0]].copy(), {int(i): blob[refs[i]["blob_off"]:refs[i]["blob_off"] + min(refs[i]["len"], 256)].tobytes()
                                                     for i in sample if refs[i]["len"] != 0xFFFFFFFF})
        (hg, hr, hs), (dg, dr, ds) = out["host"], out["device"]
        assert hg == dg and np.array_equal(hr, dr) and all(hs[i] == ds[i] for i in hs.keys() & ds.keys()), f"step {k}: paths differ"
        n_ent.append(dg[0]); n_bytes.append(dg[1]); n_ranges.append(len(g))
    e.close()
    return res, n_ent, n_bytes, n_ranges


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=16)
    ap.add_argument("--warmup", type=int, default=4)
    ap.add_argument("--configs", default="2,5")
    a = ap.parse_args()
    dev = device()
    for rnd in range(a.rounds):
        for config in [int(x) for x in a.configs.split(",")]:
            res, n_ent, n_bytes, n_ranges = run(config, a.steps, a.warmup, seed=rnd)
            q = lambda v, p: float(np.percentile(v, p)) if v else None  # noqa: E731
            row = {"bench": "apply_gather", "config": config, "round": rnd, "groups": CONFIGS[config][0], "steps": len(n_ent),
                   "ranges_per_step_p50": q(n_ranges, 50), "entries_per_step_p50": q(n_ent, 50),
                   "entries_per_step_range": [min(n_ent, default=0), max(n_ent, default=0)], "bytes_per_step_p50": q(n_bytes, 50)}
            for path, r in res.items():
                row[path] = {"wall_ms_p50": q(r["wall_ms"], 50), "wall_ms_p99": q(r["wall_ms"], 99),
                             "wall_ms_range": [min(r["wall_ms"], default=0), max(r["wall_ms"], default=0)],
                             "cpu_ms_p50": q(r["cpu_ms"], 50), "kernel_ms_p50": q(r["kernel_ms"], 50),
                             "host_served_max": max(r["served"], default=0)}
            row["gpu"] = dev
            print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
