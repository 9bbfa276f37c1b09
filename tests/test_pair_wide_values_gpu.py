"""Parity of pair_kernel (R = 3 leader stream) against the CPU oracle where values leave the 32-bit range.

Indices near 2^40, terms of 2^31 and more, a failure stamped more than 2^31 ms in the past, replies whose time or last
index jump by 2^31 in the middle of a launch, recovery_cool_down_ms > 0 with no failure yet, warps that mix such groups
with ordinary ones, and a partial last block.  Every outbox column and the exported state must stay bit-exact.  All tests
need an H100 (`-m gpu`)."""
import numpy as np
import pytest

from oracle import binding
from rafting_b200 import abi, workload
from tests import harness

pytestmark = pytest.mark.gpu

E40 = 1 << 40
T31 = 1 << 31


@pytest.fixture(scope="module")
def engine_mod():
    from rafting_b200 import engine
    engine.lib()
    return engine


def _init(G, big=()):
    """Groups in `big` open with a log that starts near 2^40 and a term of at least 2^31."""
    init = harness.init_array(G, terms=np.arange(G) % 7)
    big = np.asarray(list(big), dtype=np.int64)
    if len(big):
        t = T31 + (big % 5)
        init["term"][big] = t
        init["epoch_index"][big] = E40 + big
        init["epoch_term"][big] = t
        init["first_index"][big] = E40 + big + 1
        init["last_index"][big] = E40 + big + 2
        init["last_term"][big] = t
        init["commit_index"][big] = E40 + big
    return init


def _run(sut_factory, G, rows, steps=10, big=(), mutate=None, **cfgkw):
    cfg = abi.make_cfg(replicas=3, max_groups=G, max_rows=rows, **cfgkw)
    o, e = binding.Oracle(cfg), sut_factory(cfg)
    init = _init(G, big)
    o.open_bulk(0, init)
    e.open_bulk(0, init)
    w1 = workload.make_wl(0x5EED0032, 1, G, 2)
    w = workload.make_wl(0x5EED0032, rows, G, 2, p_reject_ppm=60_000, p_error_ppm=20_000, p_cancel_ppm=20_000)
    prev = harness.elect_all(o, w1)
    harness.assert_outbox_equal(prev, harness.elect_all(e, w1), where="after election")
    assert ((prev.role_word & 3) == abi.ROLE_LEADER).all()
    for k in range(steps):
        ib = workload.leader_inbox_host(w, k, prev)
        if mutate is not None:
            mutate(k, ib)
        out = o.step(ib)
        harness.assert_outbox_equal(out, e.step(ib), where=f"at step {k}")
        prev = out
    harness.assert_states_equal(o, e, range(G), 2, where="end of stream")
    return prev


def _acks(ib, r, lane, groups):
    """Positions (in `groups`) whose lane `lane` carries an AppendEntries ack in row r."""
    return [i for i in groups if (int(ib.ev_meta[r, i, lane]) & 0xF) == abi.EV_AE_ACK]


def test_large_indices_and_terms(engine_mod):
    """Every group opens with indices near 2^40 and terms >= 2^31."""
    G = 1024
    last = _run(engine_mod.Engine, G, 6, big=range(G))
    assert (last.commit_index > E40).mean() > 0.9


def test_warps_mixing_narrow_and_wide_groups(engine_mod):
    """One group in five opens near 2^40, so every warp mixes large and small values; 777 groups leave a partial last
    block."""
    G = 777
    last = _run(engine_mod.Engine, G, 5, big=range(0, G, 5))
    assert (last.commit_index > 0).mean() > 0.9


def test_partial_block(engine_mod):
    G = 777
    _run(engine_mod.Engine, G, 5)


def test_failure_far_in_the_past(engine_mod):
    """A failed reply stamped more than 2^31 ms before now: requestFailure lies that far in the past for the rest of the
    stream."""
    G = 1024

    def mutate(k, ib):
        if k == 3:
            sel = _acks(ib, 1, 0, range(0, G, 29))
            assert sel
            for i in sel:
                m = int(ib.ev_meta[1, i, 0])
                ib.ev_meta[1, i, 0] = (m & ~0x30) | (abi.OUT_ERROR << 4)
                ib.ev_tn[1, i, 0] = (0, harness.T0 - 2 * T31)
    _run(engine_mod.Engine, G, 6, mutate=mutate)


def test_recovery_cool_down_with_no_failure_yet(engine_mod):
    """recovery_cool_down_ms > 0: isReady compares now - requestFailure, and a follower that never failed has
    requestFailure == 0."""
    _run(engine_mod.Engine, 1024, 6, recovery_cool_down_ms=50)


def test_ack_leaving_the_windows_mid_launch(engine_mod):
    """Acks whose reply time lies 2^31 ms ahead, or whose last index lies 2^31 above, in the middle of a launch."""
    G = 1024

    def mutate(k, ib):
        if k == 4:
            sel = _acks(ib, 2, 1, range(3, G, 31))
            assert sel
            for i in sel:
                t = ib.ev_tn[2, i, 1]
                ib.ev_tn[2, i, 1] = (t["x"], t["y"] + T31)
        if k == 6:
            sel = _acks(ib, 1, 0, range(5, G, 37))
            assert sel
            for i in sel:
                el = ib.ev_el[1, i, 0]
                ib.ev_el[1, i, 0] = (el["x"], el["y"] + T31)
    _run(engine_mod.Engine, G, 6, mutate=mutate)
