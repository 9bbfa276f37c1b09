"""What a context coming or going costs a pipelined pump: the due pump of tools/bench_due_pump.py (64 K x 3, compact due
steps over each tick's event gids, d = 3 steps in flight) with k edits every 10 ticks (tests/edit_pump.py: closes, restarts
over multi-run logs and fresh opens), issued two ways:

  sync   drain every slot, then rafting_group_open / load_runs / close per record (the synchronous calls)
  edit   rafting_group_edit_begin: one call, enqueued behind the steps in flight

Per (mode, k) and run it reports the tick time p50 / p99 (the host's whole tick: edits, waits, encoding and begin), the
time of the edit itself on edit ticks (the call, or the drain and the calls), and for "edit" the device time of one call's
copy and kernel (CUDA events around the call on an idle stream, median of 20).  Each pump's end state is checked against the
dense reference's digest.  One JSON line per (mode, k, run), with the device name, power limit and max SM clock.

    python tools/bench_group_edits.py [--ticks 160] [--runs 3] [--k 16 256 4096]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tests import edit_pump as ep  # noqa: E402


def device():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True).stdout.strip()
    except OSError:
        return "unknown"


def edit_device_ms(e, recs, reps=20):
    import torch
    s = torch.cuda.ExternalStream(e.stream())
    t = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(s)
        e.group_edit_begin(recs)
        b.record(s)
        b.synchronize()
        t.append(a.elapsed_time(b))
    return float(np.median(t))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ticks", type=int, default=160)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--k", type=int, nargs="+", default=[16, 256, 4096])
    a = ap.parse_args()
    dev = device()
    for k in a.k:
        S = ep.Stream(k_edits=k)
        for t in range(a.ticks):
            S.advance(t)
        digest = S.ref.digest(0, ep.G)
        for run in range(a.runs):
            for mode in ("sync", "edit"):                               # alternating, so drift hits both alike
                P = ep.DuePump(S, d=3, mode=mode)
                P.run(a.ticks, timer=time.perf_counter)
                ts, es = np.array(P.ticks_s[1:]) * 1e3, np.array(P.edit_s) * 1e3
                res = dict(mode=mode, k=k, run=run, d=3, groups=ep.G, ticks=a.ticks, edit_ticks=len(es),
                           tick_ms_p50=round(float(np.median(ts)), 3), tick_ms_p99=round(float(np.percentile(ts, 99)), 3),
                           edit_ms_p50=round(float(np.median(es)), 3), edit_ms_max=round(float(es.max()), 3),
                           state_equals_reference=bool(np.array_equal(P.e.digest(0, ep.G), digest)), device=dev)
                if mode == "edit":
                    res["edit_device_ms_p50"] = round(edit_device_ms(P.e, S.edits[max(S.edits)]), 4)
                P.e.close()
                print(json.dumps(res), flush=True)
        S.ref.close()


if __name__ == "__main__":
    main()
