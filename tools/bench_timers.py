"""Cost of the due query (rafting_timers_due_begin / _wait) on the GPU: begin -> wait wall time at 64 K and 1 M groups with
about 1 % and 10 % of the timers due, for a pinned output buffer (the device writes it) and a pageable one (staged, copied at
the wait).  Prints one JSON line per configuration, with the device name and power limit it was measured on.

    python tools/bench_timers.py [--iters 200]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from rafting_b200 import abi, engine  # noqa: E402
from tests import harness  # noqa: E402


def device():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True).stdout.strip()
    except OSError:
        return "unknown"


def main():
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=100)
    a = ap.parse_args()
    dev = device()
    for G in (65536, 1 << 20):
        cfg = abi.make_cfg(replicas=3, max_groups=G, max_rows=1, entry_pool_cap=16)
        e = engine.Engine(cfg)
        init = harness.init_array(G)
        init["rand_ms"] = 1 + np.random.default_rng(1).integers(0, 1000, G)     # followers' deadlines spread over 1 s
        e.open_bulk(0, init)
        t0 = int(init["now_ms"][0])
        pinned = torch.zeros(G, dtype=torch.int32).pin_memory()
        pageable = np.zeros(G, np.uint32)
        for frac in (0.01, 0.10):
            until = t0 + int(frac * 1000)
            for name, buf in (("pinned", pinned.data_ptr()), ("pageable", pageable)):
                ts = []
                for k in range(a.iters + 20):
                    s = time.perf_counter()
                    e.timers_due_begin(0, until, buf, G)
                    n, nxt = e.timers_due_wait(0)
                    ts.append(time.perf_counter() - s)
                ts = np.array(ts[20:]) * 1e6
                print(json.dumps(dict(groups=G, due=n, due_frac=round(n / G, 4), out=name, begin_to_wait_us_p50=round(float(np.median(ts)), 1),
                                      p99=round(float(np.percentile(ts, 99)), 1), device=dev)), flush=True)
        # device time of one query: CUDA events on the engine's stream around four queries enqueued back to back (no host wait
        # inside the window), the three launches each, at ~10 % due
        st = torch.cuda.ExternalStream(e.stream())
        ms = []
        for k in range(a.iters // 4 + 5):
            b, c = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            b.record(st)
            for s in range(4):
                e.timers_due_begin(s, t0 + 100, pinned.data_ptr(), G)
            c.record(st)
            for s in range(4):
                e.timers_due_wait(s)
            c.synchronize()
            ms.append(b.elapsed_time(c) / 4)
        ms = np.array(ms[5:]) * 1000
        # the alternative to mapped writes: a copy of cap = G entries down after the count is known
        src = torch.zeros(G, dtype=torch.int32, device="cuda")
        cp = []
        for k in range(a.iters + 10):
            b, c = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            b.record(); pinned.copy_(src, non_blocking=True); c.record(); c.synchronize()
            cp.append(b.elapsed_time(c) * 1000)
        print(json.dumps(dict(groups=G, device_us_per_query_p50=round(float(np.median(ms)), 2),
                              copy_of_cap_entries_us_p50=round(float(np.median(cp[10:])), 2), device=dev)), flush=True)
        e.close()


if __name__ == "__main__":
    main()
