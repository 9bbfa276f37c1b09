"""CPU checks of the fuzz matrix that tests/test_engine_gpu.py runs on the engine: it reaches every kernel and launch mode
launch_step can choose, each case steers the stream where it is meant to go, the poisoned-outbox driver catches a cell
left unwritten, and the knobs left at their defaults replay the streams the suite replayed before they existed."""
import hashlib

import numpy as np
import pytest

from rafting_b200 import abi
from tests import harness, launch_model

CASES = harness.FUZZ_UNSORTED + harness.FUZZ_SORTED


def test_launch_model_examples():
    assert launch_model.kernels(3, 2047) == (("pair_kernel",), "unsorted")
    assert launch_model.kernels(3, 2048) == (("classify_kernel", "slow_kernel<2,4>", "step_kernel<2,3>"), "class-sorted")
    assert launch_model.kernels(3, 4096, abi.INBOX_NO_REQUESTS) == (("pair_kernel",), "unsorted")
    assert launch_model.kernels(3, 4096, has_ops=False) == (("pair_kernel",), "unsorted")
    assert launch_model.kernels(2, 2048) == (("classify_kernel", "step_kernel<1,3>", "slow_group<1>"), "class-sorted")
    assert launch_model.kernels(9, 2048) == (("classify_kernel", "step_kernel<8,2>", "slow_group<8>"), "class-sorted")
    assert launch_model.kernels(10, 4096) == (("looped::step_kernel<32,0>",), "unsorted")


def test_matrix_reaches_every_launch():
    """Every (kernels, mode) launch_step can take for R = 2..33 has a case in the GPU matrix; a case's list says which
    mode its requests-carrying steps take."""
    covered = set()
    for case in CASES:
        mode = launch_model.kernels(case.R, case.n)[1]
        assert mode == ("class-sorted" if case in harness.FUZZ_SORTED else "unsorted"), case.id
        covered.add(launch_model.kernels(case.R, case.n))
        if case.stray:
            covered.add(launch_model.kernels(case.R, case.n, abi.INBOX_NO_REQUESTS))
    missing = launch_model.reachable() - covered
    assert not missing, missing


@pytest.mark.parametrize("case", [pytest.param(c, id=c.id) for c in CASES])
def test_matrix_case_on_the_oracle(case):
    """The case with the oracle on both sides, at a reduced step count: the driver runs, every outbox and state agrees,
    and the steering meets the case's coverage thresholds before any GPU time is spent on it."""
    cov = harness.run_fuzz_case(case, harness.OracleSUT, steps=case.cpu_steps)
    harness.check_coverage(case, cov)
    if case.stray:
        assert any(k[1] == "unsorted" for k in cov.launches)


class _ForgetsOneCell(harness.OracleSUT):
    """An SUT that leaves one cell unwritten whose right value is 0: plan_meta of a row that plans nothing."""

    def step(self, ib):
        out = super().step(ib)
        idle = np.argwhere(out.plan_meta == 0)
        if len(idle):
            r, i, f = idle[len(idle) // 2]
            out.plan_meta.view(np.uint8).reshape(out.plan_meta.shape + (8,))[r, i, f] = harness.POISON
        return out


def test_poisoned_driver_catches_an_unwritten_cell():
    case = harness.FUZZ_UNSORTED[0]
    with pytest.raises(AssertionError, match="plan_meta"):
        harness.run_fuzz_case(case, _ForgetsOneCell, steps=2)


# sha256 (first 16 hex digits) of every inbox the legacy cases feed, as the parent of the Fuzzer knobs generated them
LEGACY_DIGESTS = {
    "3-0-True-1": "335c1a701e7638ef", "3-2-False-2": "a76f67be8461ef77", "5-2-True-3": "a1ea37781651bc49",
    "4-1-True-4": "ff12490d75ca9120", "7-6-False-5": "046c5c0dacd9fb4c", "3-11": "28e05c32e2141787",
    "5-12": "f25a452ea245030a",
}


@pytest.mark.parametrize("case", [pytest.param(c, id=c.id) for c in CASES if c.legacy])
def test_legacy_streams_replay_unchanged(case):
    class Recording(harness.OracleSUT):
        h = hashlib.sha256()

        def step(self, ib):
            for a in (ib.op_meta, ib.op_nr, ib.op_ab, ib.op_cd, ib.op_e, ib.ent_terms[:ib.ent_count], ib.ev_meta, ib.ev_tn,
                      ib.ev_el):
                self.h.update(np.ascontiguousarray(a).tobytes())
            self.h.update(int(ib.flags).to_bytes(4, "little"))
            return super().step(ib)
    harness.run_fuzz_case(case, harness.OracleSUT, ref_factory=Recording)
    assert Recording.h.hexdigest()[:16] == LEGACY_DIGESTS[case.id]
