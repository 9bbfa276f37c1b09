"""The compact fuzz matrix (tests/compact_model.COMPACT_FUZZ) on the engine (`-m gpu`): every case's stream through the
case's compact entry point, checked every step against the oracle (the decoded outbox, or the dense fetch after an escape
overflow) and against the kernel model (the raw compact outbox word for word, and under COMPACT_PREV_TERM an unflagged twin
engine through prev_term_words); group state against the oracle on a spread of groups every few steps and on every group at
the end."""
import pytest

from tests import compact_model as model
from tests.compact_model import COMPACT_FUZZ

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("case", [pytest.param(c, id=c.id) for c in COMPACT_FUZZ])
def test_compact_fuzz_case_on_the_engine(case):
    cov = model.FuzzPump(case, engine=True).run(case.steps)
    assert cov.overflows == 1 and cov.roles == {0, 1, 2}, (cov.overflows, cov.roles)
