#!/usr/bin/env python
"""The packed pre-filtered solve of a range-sharded group (yd_shard_filter_and_wait_for_starting_new_tasks_packed,
include/ydshard.h) on ONE GPU: W rank handles in W threads of one process over the test-only NCCL stand-in, or with
--real-nccl one rank over PyTorch's NCCL.  Built on tests/shard_filter_check.py's Group and Workload (same arguments).

Every call is checked exactly against ONE CPU checker handle's packed call on the concatenated queue (the checker's
packed call is its definition: the unpacked call with the hex keys, the grants packed): every rank's verdicts, hits,
offered count, packed grants and ids; the ranks' grants unpacked with their ids equal the checker's unpacked grants;
after every call every servant's running_tasks and every replica's next task id.  Each call is followed by the staged
offered queue decided again (24-byte records, as the unpacked call leaves them), a plain sharded solve and a free.
  --fuzz N   N seeded calls per stage set (none, cache, dedupe, both): random cuts with empty ranges, a range filtered out
             entirely, everything filtered out, batches with requestors behind servant IPs (the sequential fallback);
             then a cluster with a capacity above 8192, which every rank refuses with nothing changed.

Prints one JSON line per case and a final {"shard_filter_packed": ...} line; exit code 0 iff everything matched.
"""
import json
import sys

import shard_filter_check as B  # (parses this script's arguments, loads the NCCL stand-in)

np = B.np
from yadcc_b200 import _abi, binary_digests, pack_requests, unpack_grants  # noqa: E402
from yadcc_b200._abi import FILTER_CACHE_HIT, FILTER_JOINED, FILTER_OFFERED  # noqa: E402
from yadcc_b200.dispatcher import Servant  # noqa: E402


class PackedGroup(B.Group):
    def packed(self, now, full, cuts, cd, td):
        """One group packed call on the queue `full` (REQ_DTYPE) cut at `cuts`, with binary digests cd / td (or None),
        checked against the checker.  Returns each rank's offered count."""
        W = self.W
        f16 = pack_requests(np.ascontiguousarray(full))
        parts = [np.ascontiguousarray(f16[cuts[r]:cuts[r + 1]]) for r in range(W)]
        counts = [len(p) for p in parts]
        sl = lambda m, r: None if m is None else np.ascontiguousarray(m[cuts[r]:cuts[r + 1]])  # noqa: E731
        got = B.par([lambda r=r: self.ranks[r]._filter_packed_with(
            self.lib.yd_shard_filter_and_wait_for_starting_new_tasks_packed, parts[r], sl(cd, r), sl(td, r), now, True,
            None, None) for r in range(W)])
        v1, h1, g1, ids1 = self.oracle.filter_and_wait_for_starting_new_tasks_packed(f16, cd, td, now, True)
        lo, first, offered = 0, 0, []
        for r in range(W):
            v, h, g, ids = got[r]
            hi = lo + counts[r]
            mine = int((v1[lo:hi] == FILTER_OFFERED).sum())
            if v.tolist() != v1[lo:hi].tolist():
                self.fail("verdicts differ", rank=r)
            if h.tolist() != h1[lo:hi].tolist():
                self.fail("hits differ", rank=r)
            if len(g) != mine:
                self.fail("offered counts differ", rank=r, group=len(g), single=mine)
            if g.tolist() != g1[first:first + mine].tolist():
                self.fail("packed grants differ", rank=r)
            if ids.tolist() != ids1.tolist():
                self.fail("ids differ", rank=r, group=ids.tolist(), single=ids1.tolist())
            if unpack_grants(g, ids).tolist() != unpack_grants(g1, ids1)[first:first + mine].tolist():
                self.fail("unpacked grants differ", rank=r)
            self.counts["empty_ranges"] += int(counts[r] == 0)
            self.counts["filtered_ranges"] += int(counts[r] > 0 and mine == 0)
            offered.append(mine)
            lo, first = hi, first + mine
        self.counts["all_filtered"] += int(len(full) > 0 and sum(offered) == 0)
        self.counts["calls"] += 1
        self.counts["offered"] += sum(offered)
        self.counts["cache_hits"] += int((v1 == FILTER_CACHE_HIT).sum())
        self.counts["joined"] += int((v1 == FILTER_JOINED).sum())
        self.record(unpack_grants(g1, ids1), np.repeat(np.arange(W), offered))
        self.compare()
        return offered


def run_fuzz(world: int, calls: int, case_seed: int) -> bool:
    g = PackedGroup("fuzz-packed", world, case_seed)
    w = B.Workload(g)
    ok = True
    try:
        for sv in B.servants(np.random.default_rng(3)):
            for d in g.handles:
                d.keep_servant_alive(sv, 3600.0, now=0.0)
        rng = g.rng
        combos = sorted({(int(t), int(e)) for t, e in zip(rng.integers(0, B.N_TU, 600), rng.integers(0, 4, 600))})
        km, _ = w.keys(combos)
        for d in g.handles:
            d.bloom_reset(1 << 16, 4)
            d.bloom_add(km[0::3])
        w.cached = set(combos[0::3])
        running = combos[1::3]
        now = 1.0
        for stages in (0, 1, 2, 3):
            for k in range(calls):
                now += 0.25
                g.ev = f"packed stages {stages} call {k}"
                if k % 5 == 0:
                    sub = [running[int(i)] for i in rng.integers(0, len(running), 60)]
                    gr = g.solve(now, w.queue(sub))
                    B.index_from(g, w.keys(sub)[1], gr)
                    now += 0.05
                n = int(rng.choice([1, 3, 40, 150, 400])) if k % 6 else 0
                special = k % 7
                cs = w.combos(n, w.cached if special == 1 and stages & 1 else None)
                cuts = g.cut(n)
                if special == 2 and world > 1:
                    cuts = sorted([0, 0] + cuts[1:])[:world + 1]
                    cuts[-1] = n
                if special == 3 and stages & 1 and world > 1 and n:
                    cached = sorted(w.cached)
                    for j in range(cuts[-2], n):
                        cs[j] = cached[int(rng.integers(0, len(cached)))]
                q = w.queue(cs, 0.3 if special == 4 else 0.0)
                km, dm = w.keys(cs) if n else (np.zeros((0, 81), np.uint8), np.zeros((0, 64), np.uint8))
                offered = g.packed(now, q, cuts, binary_digests(km) if stages & 1 else None,
                                   binary_digests(dm) if stages & 2 else None)
                g.redecide(now + 0.02, offered)
                g.solve(now + 0.03, w.queue(w.combos(int(rng.integers(0, 30)))))
                g.free()
    except B.Mismatch:
        ok = False
    print(json.dumps({"case": "fuzz-packed", "world": world, "ok": ok, **g.counts}), flush=True)
    g.close()
    return ok


def run_refusal(world: int, case_seed: int) -> bool:
    """A servant with a capacity above 8192 (replicated state): every rank returns (size_t)-1, nothing changes."""
    g = PackedGroup("refusal", world, case_seed)
    w = B.Workload(g)
    ok, refused = True, False
    try:
        for sv in B.servants(np.random.default_rng(3)) + [Servant("10.9.0.1:8000", None, [B.DIGESTS[0]], 0, 10000, 0,
                                                                  64 << 30, 48 << 30, 10000)]:
            for d in g.handles:
                d.keep_servant_alive(sv, 3600.0, now=0.0)
        q = pack_requests(w.queue(w.combos(40)))
        cuts = g.cut(40)
        before = [(d.next_task_id(), d.servant_state()["running_tasks"].tolist()) for d in g.ranks]
        raw = []
        for r in range(world):
            part = np.ascontiguousarray(q[cuts[r]:cuts[r + 1]])
            raw.append((part, np.zeros(max(len(part), 1), np.uint8), np.zeros(max(len(part), 1), _abi.GRANT8_DTYPE)))
        f = _abi.yd_prefilter_packed(None, None)
        rets = B.par([lambda r=r: int(g.lib.yd_shard_filter_and_wait_for_starting_new_tasks_packed(
            g.ranks[r]._h, B.ns(1.0), raw[r][0].ctypes.data, len(raw[r][0]), B.C.byref(f), raw[r][1].ctypes.data, None,
            raw[r][2].ctypes.data, None)) for r in range(world)])
        refused = all(x == B.REFUSED for x in rets)
        after = [(d.next_task_id(), d.servant_state()["running_tasks"].tolist()) for d in g.ranks]
        ok = refused and before == after
    except B.Mismatch:
        ok = False
    print(json.dumps({"case": "refusal", "world": world, "ok": ok, "refused_everywhere": refused}), flush=True)
    g.close()
    return ok


def main():
    a = B.ARGS
    ok = run_fuzz(a.world, a.fuzz, a.seed * 1000 + 7)
    ok = run_refusal(a.world, a.seed * 1000 + 8) and ok
    line = {"shard_filter_packed": ok, "world": a.world, "nccl": "real" if B.FAKE is None else "fake_nccl",
            "torch_loaded": "torch" in sys.modules}
    print(json.dumps(line), flush=True)
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
