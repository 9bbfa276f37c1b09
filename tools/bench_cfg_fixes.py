#!/usr/bin/env python
"""What the opt-in protocol fixes of cfg.flags cost on the device: config #2 (64 K groups x 3, the leader stream, 16 rows),
config #3 (256 K x 5, vote storm) and config #5 (512 K x 3, leader churn + catch-up), device-resident and recorded as
tools/bench_secondary.py records them, each on an engine with flags 0 and on one with flags 3, alternating, in one process.
Only the step launch is inside the CUDA-event pairs.  Config #2 runs pair_kernel on both engines (its steps are flagged
RAFTING_INBOX_NO_REQUESTS, as bench.py's are); configs #3 and #5 run the FIX instantiations of the step and slow kernels on the flagged engine.
Prints one JSON line per window and a summary line with the card's name and power limit."""
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bench_secondary import card, run  # noqa: E402
from rafting_b200 import abi  # noqa: E402
from rafting_b200.workload import _bind  # noqa: E402

FLAGS = abi.CFG_STRICT_CANDIDATE_VOTE | abi.CFG_LENIENT_FOLLOWER_COMMIT


def windows():
    L = _bind()
    return {
        "config2": lambda f: run("config2", 65536, 3, 16, 32, 0x5EED0002, L.rafting_wl_leader_step, elect=True, quiet=True, flags=f,
                                 requests=False),
        "config3": lambda f: run("config3", 262144, 5, 1, 8, 0x5EED0003, L.rafting_wl_vote_step, local_slot=2, quiet=True, flags=f),
        "config5": lambda f: run("config5", 524288, 3, 4, 32, 0x5EED0005, L.rafting_wl_mixed_step, elect=True, pool=True,
                                 quiet=True, flags=f),
    }


def main():
    rounds = int(sys.argv[1]) if len(sys.argv) > 1 else 3
    ms = {}
    for r in range(rounds):
        for name, go in windows().items():
            for f in ((0, FLAGS) if r % 2 == 0 else (FLAGS, 0)):
                rec = go(f)
                ms.setdefault((name, f), []).append(rec["kernel_ms_total"])
                print(json.dumps({"round": r, "config": name, "flags": f, "kernel_ms_total": rec["kernel_ms_total"],
                                  "kernel_ms_per_step_median": rec["kernel_ms_per_step_median"], "units": rec["units"],
                                  "end_state": rec["end_state"]}), flush=True)
    summary = {"card": card(), "rounds": rounds, "configs": {}}
    for name in windows():
        a, b = np.array(ms[(name, 0)]), np.array(ms[(name, FLAGS)])
        summary["configs"][name] = {"flags0_ms": a.tolist(), "flags3_ms": b.tolist(),
                                    "median_ratio_flags3_over_flags0": float(np.median(b) / np.median(a))}
    print(json.dumps(summary), flush=True)


if __name__ == "__main__":
    main()
