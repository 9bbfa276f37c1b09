"""rafting_step_device_seq against the CPU oracle: one call enqueues a whole window of device-resident launches, and from
the second launch on pair_kernel is launched programmatically behind the previous one (it stages its first inbox rows
before the previous launch has finished).  Every launch steps into its own poisoned outbox (harness.POISON), so a cell it
should write and leaves alone differs from the oracle's; every outbox and the end state must be bit-exact.  Needs an H100
(`-m gpu`)."""
import numpy as np
import pytest

from oracle import binding
from rafting_b200 import abi, workload
from tests import harness

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("G,rows,launches", [(1024, 8, 12), (777, 5, 9)])
def test_device_sequence_matches_oracle(G, rows, launches):
    import torch
    from rafting_b200 import devbatch, engine
    R, F = 3, 2
    cfg = abi.make_cfg(replicas=R, max_groups=G, max_rows=rows)
    o, e = binding.Oracle(cfg), engine.Engine(cfg)
    init = harness.init_array(G, terms=np.arange(G) % 7)
    o.open_bulk(0, init)
    e.open_bulk(0, init)
    w1 = workload.make_wl(0x5EED0051, 1, G, F)
    w = workload.make_wl(0x5EED0051, rows, G, F, p_reject_ppm=60_000, p_error_ppm=20_000, p_cancel_ppm=20_000)
    prev = harness.elect_all(o, w1)
    harness.assert_outbox_equal(prev, harness.elect_all(e, w1), where="after election")
    # the oracle records the window closed-loop; the engine replays it in one call
    ibs, want = [], []
    for k in range(launches):
        ib = workload.leader_inbox_host(w, k, prev)
        prev = o.step(ib, out=harness.poisoned_outbox(ib, F, G))
        ibs.append(ib)
        want.append(prev)
    dev = torch.device("cuda", 0)
    dins = [devbatch.DevInbox.from_host(ib, dev) for ib in ibs]
    douts = [devbatch.DevOutbox(rows, G, F, G, dev, fill=harness.POISON) for _ in range(launches)]
    torch.cuda.synchronize()
    ics = (abi.InboxC * launches)(*[d.as_c() for d in dins])
    ocs = (abi.OutboxC * launches)(*[d.as_c() for d in douts])
    e.step_device_seq(ics, ocs, launches)
    torch.cuda.synchronize()
    for k in range(launches):
        harness.assert_outbox_equal(want[k], douts[k].to_host(), where=f"launch {k} of the sequence")
    harness.assert_states_equal(o, e, range(G), F, where="end of the sequence")
