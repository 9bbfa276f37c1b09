"""Checkpoints, restores and shard images roll back every table, the compact path's in-flight table included (`-m gpu`).

The in-flight table (which tags of a (group, follower) lane are in flight, and the echo each one carries) is created by the
first compact call.  A restore to a checkpoint taken before that call must leave no tag handed out after it, and an image
saved before it must load as "nothing in flight": otherwise a replay of the same compact inboxes hands out other tags, and its
plan_c words and escape records differ from the first pass.  The compact steps are tests/compact_model.FuzzPump's, checked
against the oracle and the kernel model on the first pass; every recorded call is then run again on the rolled-back engine
and must give the first pass's compact outbox column for column."""
import dataclasses
import struct

import numpy as np
import pytest

from rafting_b200 import abi, compact
from tests import compact_model as model
from tests import harness

pytestmark = pytest.mark.gpu

_BY_ID = {c.id: c for c in model.COMPACT_FUZZ}
# whole-shard compact steps at R = 3 with elections carried compact, and sweep steps at R = 5 on a flagged engine; no step
# runs with a small escape list, so every pass decodes
IDS = ["R3-G777-whole-ELPT-wide", "R5-G777-sweep-EL-strict-lenient"]
K = 5


def _case(case_id):
    c = _BY_ID[case_id]
    return dataclasses.replace(c, cflags=c.cflags & ~model.PT, esc_step=-1)


class _Recorded:
    """The engine with every compact call it runs kept: (compact inbox, requests, flags, compact outbox)."""

    def __init__(self, e):
        self.e, self.calls = e, []

    def __getattr__(self, name):
        return getattr(self.e, name)

    def step_compact(self, cin, cout, slot=0, reqs=None, flags=0):
        self.e.step_compact(cin, cout, slot=slot, reqs=reqs, flags=flags)
        self.calls.append((cin, reqs, flags, cout))
        return cout


def _pump(case_id):
    p = model.FuzzPump(_case(case_id), engine=True)
    p.e = _Recorded(p.e)
    return p


def _again(e, call):
    cin, reqs, flags, cout = call
    out = compact.CompactOutbox(cout.rows, cout.n, cout.F, esc_cap=cout.esc_cap, gids=cout.gids)
    e.step_compact(cin, out, reqs=reqs, flags=flags)
    return out


def _assert_same_step(first, again, want, flags, where):
    for name in compact.CompactOutbox.COLS + ("counts",):
        a, b = getattr(first, name), getattr(again, name)
        assert np.array_equal(a, b), f"{name} differs from the first pass, {where}: first diffs at {np.argwhere(a != b)[:5].tolist()}"
    assert np.array_equal(first.tags(), again.tags()), f"tags differ, {where}"
    assert model._sorted_esc(first) == model._sorted_esc(again), f"escape records differ, {where}"
    harness.assert_outbox_equal(want, compact.decode_outbox(again, elections=bool(flags & model.EL)), where=where)


@pytest.mark.parametrize("sync", [True, False], ids=["restore", "restore-async"])
@pytest.mark.parametrize("when", ["before-the-table", "after-the-table"])
@pytest.mark.parametrize("case_id", IDS)
def test_restore_replays_compact_steps_bit_exact(case_id, when, sync):
    """Checkpoint (before the first compact call, or after one), K compact steps that leave tags unanswered, restore, the
    same K compact inboxes again: every compact column equals the first pass, and decodes to the oracle's outbox."""
    p = _pump(case_id)
    if when == "after-the-table":
        p.step()
    p.e.checkpoint()
    first = len(p.e.calls)
    wants = [p.step() for _ in range(K)]
    calls = p.e.calls[first:]
    assert len(calls) == K
    assert p.st.bits.any(), "no tag left in flight: the replay would not tell a stale table from a clean one"
    p.e.restore(sync=sync)
    for k, (call, want) in enumerate(zip(calls, wants)):
        _assert_same_step(call[3], _again(p.e.e, call), want, call[2], where=f"{case_id}: replayed compact step {k}")


@pytest.mark.parametrize("case_id", IDS)
def test_image_saved_before_the_compact_path_loads_without_tags(case_id, tmp_path):
    """An image saved before any compact call, loaded back into the engine after K compact steps: the engine goes on exactly
    as a fresh engine that loaded the same image, and as the first pass from that image did."""
    from rafting_b200 import engine
    p = _pump(case_id)
    path = str(tmp_path / "before.img")
    p.e.state_save(path)
    wants = [p.step() for _ in range(K)]
    assert p.st.bits.any()
    p.e.state_save(str(tmp_path / "after.img"))
    blocks = [struct.unpack_from("<I", open(f, "rb").read(), NBLOCKS_AT)[0] for f in (path, str(tmp_path / "after.img"))]
    assert blocks[1] == blocks[0] + 3, f"the first image already holds the in-flight table: {blocks}"
    p.e.state_load(path)
    fresh = engine.Engine(p.cfg)
    fresh.state_load(path)
    for k, (call, want) in enumerate(zip(p.e.calls, wants)):
        _assert_same_step(call[3], _again(p.e.e, call), want, call[2], where=f"{case_id}: step {k} after the load")
        _assert_same_step(call[3], _again(fresh, call), want, call[2], where=f"{case_id}: step {k} on a fresh engine")


NBLOCKS_AT = 20          # ImgHdr { magic, version, G, F, runs, nblocks (uint32 each), total (uint64) }


def _with_nblocks(path, out, n):
    blob = bytearray(open(path, "rb").read())
    blob[NBLOCKS_AT:NBLOCKS_AT + 4] = struct.pack("<I", n)
    open(out, "wb").write(bytes(blob))
    return out


def test_image_with_another_block_count_is_refused(tmp_path):
    """The tables of an image match the engine's one for one; the only difference accepted is an image without the in-flight
    table (saved before the compact path was used) into an engine that has one.  A refused image changes nothing."""
    from rafting_b200 import engine
    G, R, rows = 256, 3, 2
    cfg = abi.make_cfg(replicas=R, max_groups=G, max_rows=rows)
    init = harness.init_array(G, terms=np.arange(G) % 7)
    e = engine.Engine(cfg)
    e.open_bulk(0, init)
    pre = str(tmp_path / "pre.img")
    e.state_save(pre)
    nb = struct.unpack_from("<I", open(pre, "rb").read(), NBLOCKS_AT)[0]
    e.step_compact(compact.encode_inbox(abi.Inbox(rows, G, R - 1), None, None, None), compact.CompactOutbox(rows, G, R - 1))
    post = str(tmp_path / "post.img")
    e.state_save(post)
    assert struct.unpack_from("<I", open(post, "rb").read(), NBLOCKS_AT)[0] == nb + 3

    def refused(target, img):
        d = target.digest(0, G)
        with pytest.raises(engine.RaftingError):
            target.state_load(img)
        assert np.array_equal(target.digest(0, G), d)
    plain = engine.Engine(cfg)                     # no in-flight table
    plain.open_bulk(0, init)
    for n in (nb - 1, nb - 2, nb + 1, nb + 2):
        refused(plain, _with_nblocks(pre, str(tmp_path / f"plain{n}.img"), n))
    for n in (nb - 1, nb + 1, nb + 2, nb + 4):     # e has the in-flight table: nb + 3 blocks
        refused(e, _with_nblocks(post if n > nb else pre, str(tmp_path / f"compact{n}.img"), n))
    e.state_load(pre)                              # nb: the image saved before the compact call
    e.state_load(post)
    plain.state_load(pre)
