"""Group edits without a GPU: the rafting_group_edit_t records Python builds, read back by C through the header, and the pump
contract of rafting_group_edit_begin at the model level — groups of one live node restarted mid-run from what survives on
disk, with that node's queued events and in-flight RPCs of those groups dropped, stay safe and converge."""
import os
import shutil
import subprocess

import numpy as np
import pytest

from oracle import binding
from rafting_b200 import abi, durable
from rafting_b200.engine import edit_close, edit_open
from tests.cluster_sim import T0, TICK_MS, Cluster

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.skipif(shutil.which("gcc") is None, reason="no gcc")
def test_records_round_trip_through_the_header(tmp_path):
    recs = np.array([edit_open(3, runs=[(1, 1), (4, 2), (9, 5)], term=7, ballot=2, last_index=12, last_term=5, commit_index=4,
                               now_ms=123, rand_ms=0),
                     edit_close(9),
                     edit_open(1 << 20, term=1, epoch_index=6, epoch_term=2, first_index=7, last_index=8, last_term=2, rand_ms=55)],
                    dtype=abi.GROUP_EDIT)
    path = tmp_path / "recs.bin"
    recs.tofile(path)
    src = tmp_path / "p.c"
    src.write_text(r'''#include <stdio.h>
#include "rafting_b200.h"
int main(int argc, char** argv) {
    rafting_group_edit_t r[3];
    FILE* f = fopen(argv[1], "rb");
    if (fread(r, sizeof(r[0]), 3, f) != 3) return 1;
    for (int k = 0; k < 3; k++) {
        printf("%u %u %lld %d %lld %lld %lld %lld %lld %lld %lld %u", r[k].gid, r[k].kind, (long long)r[k].init.term, r[k].init.ballot,
               (long long)r[k].init.epoch_index, (long long)r[k].init.epoch_term, (long long)r[k].init.first_index,
               (long long)r[k].init.last_index, (long long)r[k].init.last_term, (long long)r[k].init.commit_index,
               (long long)r[k].init.rand_ms, r[k].n_runs);
        for (unsigned j = 0; j < r[k].n_runs; j++) printf(" %lld:%lld", (long long)r[k].runs[j].x, (long long)r[k].runs[j].y);
        printf("\n");
    }
    return RAFTING_EDIT_OPEN == 1 && RAFTING_EDIT_CLOSE == 2 ? 0 : 2;
}''')
    exe = tmp_path / "p"
    res = subprocess.run(["gcc", "-std=c11", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], capture_output=True, text=True)
    assert res.returncode == 0, res.stderr[-3000:]
    out = subprocess.run([str(exe), str(path)], capture_output=True, text=True, check=True).stdout.splitlines()
    assert out == ["3 1 7 2 0 0 1 12 5 4 0 3 1:1 4:2 9:5",
                   "9 2 0 0 0 0 0 0 0 0 0 0",
                   f"{1 << 20} 1 1 -1 6 2 7 8 2 0 55 0"]
    with pytest.raises(ValueError):
        edit_open(0, runs=[(i + 1, i) for i in range(abi.TERM_RUNS + 1)])


class GroupRestartCluster(Cluster):
    """Cluster with per-group restarts inside a live node: the node's engine keeps running, and the chosen groups are reopened
    from the StableLock record and the payload store, as a pump that rebuilds some of its contexts does.  Nothing of the old
    life reaches the new one: the node's queued events for those groups and every in-flight message addressed to it for
    them are dropped, and so are the old life's requests still on their way to a peer or queued there, so that no reply to
    them is ever produced.  To the peers that is message loss, which the protocol tolerates.  With an engine that has
    group_edit_begin the reopen is one call of it (an OPEN of an alive gid replaces it); otherwise a close and the
    synchronous calls."""

    def restart_groups(self, slot, gids, restore):
        nd = self.nodes[slot]
        now = T0 + TICK_MS * (self.tick + 1)
        recs = []
        for g in sorted(gids):
            st = restore(g)
            ms = nd.snapshot[g]
            keys = sorted(nd.store[g])
            runs = []
            for i in keys:
                t = nd.store[g][i][0]
                if not runs or runs[-1][1] != t:
                    runs.append((i, t))
            recs.append(edit_open(g, runs=runs if len(runs) > 1 else None, term=st.term, ballot=st.ballot, now_ms=now,
                                  epoch_index=ms[0] if ms else 0, epoch_term=ms[1] if ms else 0,
                                  first_index=keys[0] if keys else 1, last_index=keys[-1] if keys else 0,
                                  last_term=nd.store[g][keys[-1]][0] if keys else 0, rand_ms=0))
            nd.queue[g].clear()
            nd.install[g] = None
            nd.inc_term[g] = dict()
        recs = np.array(recs, dtype=abi.GROUP_EDIT)
        if hasattr(nd.sut, "group_edit_begin"):
            nd.sut.group_edit_begin(recs)
        else:
            for r in recs:
                g = int(r["gid"])
                nd.sut.close_group(g)
                kw = {k: int(r["init"][k]) for k in abi.GROUP_INIT_DTYPE.names if k != "_pad"}
                nd.sut.open_group(g, **kw)
                if r["n_runs"]:
                    nd.sut.load_runs(g, [(int(x), int(y)) for x, y in r["runs"][:r["n_runs"]].tolist()])
        gs = set(int(g) for g in recs["gid"])

        def old_request(item):
            return item[0] == "op" and item[1].get("src") == slot

        self.inflight = [m for m in self.inflight if not (m[3] in gs and (m[2] == slot or old_request(m[4])))]
        for peer in self.nodes:
            if peer is not nd:
                for g in gs:
                    kept = [it for it in peer.queue[g] if not old_request(it)]
                    peer.queue[g].clear()
                    peer.queue[g].extend(kept)
        self.counts["group_restarts"] += len(gs)


def group_restarts(make, R, seed, tmp_path):
    G = 8
    journals = [durable.Journal(os.path.join(str(tmp_path), f"n{k}"), G) for k in range(R)]
    c = GroupRestartCluster(make, G=G, R=R, seed=seed, drop_ppm=20_000, compact_every=30, guard_candidate_votes=True)
    c.on_outbox = lambda nd, ob: journals[nd.slot].commit_step(ob.role_word, ob.current_term)
    rng = np.random.default_rng(seed)
    c.run(120)
    for phase in range(6):
        slot = c.leader_of(int(rng.integers(0, G))) if phase % 2 == 0 else int(rng.integers(0, R))
        slot = int(rng.integers(0, R)) if slot is None else slot
        gids = rng.choice(G, size=int(rng.integers(1, G // 2 + 1)), replace=False)
        c.restart_groups(slot, gids, lambda g, s=slot: journals[s].restore(g))
        k = int(rng.integers(0, (R - 1) // 2 + 1))
        c.cut = set(int(x) for x in rng.choice(R, size=k, replace=False))
        c.run(40)
    c.cut = set()
    c.run(250)
    c.drop_ppm = 0
    c.run(120, submit=False)
    c.check(converged=True)
    for j in journals:
        j.close()
    assert c.counts["group_restarts"] >= 6
    return c


@pytest.mark.parametrize("R,seed", [(3, 41), (5, 43)])
def test_per_group_restarts_in_a_live_node_stay_safe_and_converge(R, seed, tmp_path):
    group_restarts(binding.Oracle, R, seed, tmp_path)
