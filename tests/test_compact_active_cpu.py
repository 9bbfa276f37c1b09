"""Active lists on the compact host path, on CPU (rafting_step_begin_compact_active): a step over the busy groups gids[] carries
every compact column by position, while the in-flight table stays indexed by gid.  The numpy restatement of the compact
kernels (tests/compact_model.py) runs around the oracle: every dense inbox must survive encode -> unpack on every
column the step reads, every dense outbox pack -> decode, and a plan's tag must be found by its ack wherever its gid sits in
the next step's list.  The active kernels are modelled by tests/compact_active_model.py, the whole-shard model over the
listed gids' slice of the in-flight state."""
import numpy as np
import pytest

from oracle import binding
from rafting_b200 import abi, compact, workload
from tests import compact_active_model as active
from tests import compact_model as model
from tests import harness
from tests.compact_model import EL, PT, assert_step_reads_the_same

U64 = np.uint64


def pick(G, n, seed):
    return np.sort(np.random.default_rng(seed).choice(G, n, replace=False)).astype(np.uint32)


def leader_oracle(G, R, rows, seed=0x5EED0002):
    cfg = abi.make_cfg(replicas=R, max_groups=G, max_rows=rows, entry_pool_cap=rows * G * 50)
    o = binding.Oracle(cfg)
    o.open_bulk(0, harness.init_array(G, terms=np.arange(G) % 7))
    harness.elect_all(o, workload.make_wl(seed, 1, G, R - 1))
    return o, workload.make_wl(seed, rows, G, R - 1)


def pump(o, G, F, lists, make, flags=0, empty_list=False):
    """One step per entry of `lists` (an active list, or None for the whole shard) through the model around the oracle.
    Yields (k, gids, inbox, compact inbox, oracle outbox, compact outbox, what the pump carried into the step)."""
    st = model.InFlight(G, F)
    g_term = np.array([o.export(g).current_term for g in range(G)], np.int64)
    prev, nxt, frm = None, None, None
    for k, gids in enumerate(lists):
        ib = make(k, None if prev is None else active.carry_outbox(prev, frm, gids, G), gids)
        kept = None if nxt is None else active.carry(nxt, frm, gids, G)
        ci = model.encode(ib, kept, flags, empty_list=empty_list)
        assert (ci.gids is None) == (gids is None) and (gids is None or np.array_equal(ci.gids, gids))
        assert_step_reads_the_same(ib, active.unpack(ci, g_term, st, flags, gids=gids), where=f"encode -> unpack, step {k}")
        want = o.step(ib)
        n, rows = ib.n, ib.rows
        co = active.pack(want, model.oracle_epoch(o, G), st, esc_cap=rows * n * F + 2 * rows * n, flags=flags,
                        replies=ci.reqs is not None, gids=gids)
        got = compact.decode_outbox(co, elections=bool(flags & EL), prev_term=bool(flags & PT))
        harness.assert_outbox_equal(want, got, where=f"pack -> decode, step {k}")
        assert (got.gids is None) == (gids is None) and len(got.commit_index) == n
        yield k, gids, ib, ci, want, co, kept
        g_term[np.arange(G) if gids is None else gids] = want.current_term[:n]
        prev, nxt, frm = got, model.next_of(want, co), gids


def test_leader_stream_over_an_active_list_is_lossless():
    G, R, rows = 4096, 3, 4
    o, w = leader_oracle(G, R, rows)
    A = pick(G, 1500, 1)
    words = 0
    for k, gids, ib, ci, want, co, kept in pump(o, G, R - 1, [A] * 6, lambda k, prev, g: workload.leader_inbox_host(w, k, prev, gids=g)):
        assert ci.ev_c.shape == (rows, 1500, R - 1) and co.plan_c.shape == (rows, 1500, R - 1)
        words += int(((ci.ev_c & np.uint32(0xF)) == abi.EV_AE_ACK).sum())
    assert words > 10_000


@pytest.mark.parametrize("flags", [0, EL | PT])
def test_config5_over_an_active_list_with_a_request_list_is_lossless(flags):
    G, R, rows = 4096, 3, 4
    o, _ = leader_oracle(G, R, rows, seed=0x5EED0005)
    w = workload.make_wl(0x5EED0005, rows, G, R - 1)
    A = pick(G, 2100, 2)
    records = 0
    for k, gids, ib, ci, want, co, kept in pump(o, G, R - 1, [A] * 8, lambda k, prev, g: workload.mixed_inbox_host(w, k, prev, gids=g),
                                                flags=flags, empty_list=True):
        assert ci.reqs is not None
        records += len(ci.reqs.req)
        assert (ci.reqs.req["slot"] < rows * len(A)).all()                # positional slots
    assert records > 100


@pytest.mark.parametrize("flags", [EL, EL | PT])
def test_vote_storm_over_an_active_list_is_lossless(flags):
    G, R, rows = 4096, 5, 2
    o, w = model.storm(G, R, rows)
    A = pick(G, 1200, 3)
    ratios = model.Ratios()
    for k, gids, ib, ci, want, co, kept in pump(o, G, R - 1, [A] * 6, lambda k, prev, g: workload.vote_inbox_host(w, k, prev, gids=g),
                                                flags=flags):
        ratios.add(ib, ci, want, co)
    assert ratios.reply_words > 0.5 * ratios.replies and ratios.ballot_lanes > 0.5 * ratios.ballots, vars(ratios)


def test_tags_follow_the_gid_when_the_list_changes():
    """List A, then B (A with other gids interleaved, so A's gids move to other positions), then the whole shard, then A again:
    every ack to a tagged plan finds its tag by gid and travels as an ev_c word."""
    G, R, rows = 4096, 3, 2
    F = R - 1
    o, w = leader_oracle(G, R, rows)
    A = pick(G, 600, 4)
    B = np.union1d(A, pick(G, 400, 5)).astype(np.uint32)
    assert len(B) > len(A) and (active.positions(B, A, G) != np.arange(len(A))).sum() > 500        # A's gids sit elsewhere in B
    tagged_acks = []
    for k, gids, ib, ci, want, co, kept in pump(o, G, F, [A, B, None, A],
                                                lambda k, prev, g: workload.leader_inbox_host(w, k, prev, gids=g)):
        if kept is None:
            continue
        ek = (ib.ev_meta & U64(0xF)).astype(np.int64)
        ack = (ek == abi.EV_AE_ACK) | (ek == abi.EV_IS_ACK)
        tagged = ack & (kept["tags"] < 32)
        assert np.array_equal((ci.ev_c[tagged] & np.uint32(0xF)).astype(np.int64), ek[tagged]), f"an ack to a tagged plan escaped, step {k}"
        assert not ((ack & (kept["tags"] >= 32)).any()), f"an ack without a plan of the last step, step {k}"
        esc_slots = set(int(s) for s in ci.esc["slot"])
        assert not any(s in esc_slots for s in np.flatnonzero(tagged.reshape(-1))), f"step {k}"
        tagged_acks.append(int(tagged.sum()))
    assert len(tagged_acks) == 3 and min(tagged_acks) > 300, tagged_acks


def test_carry_maps_positions_by_gid():
    G = 16
    A, B = np.array([1, 4, 9], np.uint32), np.array([0, 1, 5, 9, 12], np.uint32)
    assert active.positions(A, B, G).tolist() == [-1, 0, -1, 2, -1]
    assert active.positions(None, A, G).tolist() == [1, 4, 9]
    assert active.positions(A, None, G)[[1, 4, 9]].tolist() == [0, 1, 2]
    nxt = dict(tags=np.arange(2 * 3 * 2, dtype=np.uint8).reshape(2, 3, 2), sent_term=np.array([7, 8, 9], np.int64))
    c = active.carry(nxt, A, B, G)
    assert c["tags"][:, 1].tolist() == nxt["tags"][:, 0].tolist() and (c["tags"][:, 0] == abi.CTAG_NONE).all()
    assert c["sent_term"].tolist() == [0, 7, 0, 9, 0]


def test_encode_and_decode_keep_the_list():
    rows, F = 1, 2
    gids = np.array([3, 10, 11], np.uint32)
    ib = abi.Inbox(rows, 3, F, gids=gids)
    ib.flags = abi.INBOX_NO_REQUESTS | abi.INBOX_COMPACT_GROUPS
    ci = compact.encode_inbox(ib, None, None)
    assert np.array_equal(ci.gids, gids) and ci.op_c.shape == (rows, 3)
    co = compact.CompactOutbox(rows, 3, F, gids=gids)
    o = compact.decode_outbox(co)
    assert np.array_equal(o.gids, gids) and len(o.commit_index) == 3
    with pytest.raises(ValueError):
        compact.decode_outbox(co, G=4096)
