#!/usr/bin/env python
"""The packed RPC window of a range-sharded group (yd_shard_wait_for_starting_task_rpcs_packed, include/ydshard.h) on ONE
GPU: W rank handles in W threads of one process over the test-only NCCL stand-in.  Built on tests/shard_rpcs_check.py's
Group (imported: it takes the same arguments and loads the stand-in before anything else).

Two groups run in lock-step, fed the same servants, windows, frees, keep-alives and ticks:
  packed group    every window through the packed group call; every rank's results, grants and ids must equal ONE CPU
                  checker handle's packed call on the window (its definition: the unpacked call, the grants packed),
                  grants_out[k] must have ordinal k, and after every event the harness compares servant state and next
                  task id with the checker's
  unpacked twin   every window through the unpacked group call; its results must equal the packed group's, and its
                  grants the packed group's unpacked with its ids
  --rpcs N        N seeded windows (counts up to 0xFFFFFFFF, the limits on both sides, a digest nobody holds, fewer
                  decisions than ranks); every fifth one also with cap one short, which every rank refuses
Then a cluster with a capacity above 8192, whose window every rank refuses with nothing changed.

Prints one JSON line per case and a final {"shard_rpcs_packed": ...} line; exit code 0 iff everything matched.
"""
import json
import sys

import shard_rpcs_check as B  # (parses this script's arguments, loads the NCCL stand-in)

np = B.np
from rpc_packed_cases import ordinals_are_positions  # noqa: E402
from yadcc_b200 import _abi, unpack_grants  # noqa: E402
from yadcc_b200.dispatcher import Servant  # noqa: E402

REFUSED = (1 << 64) - 1
DIGESTS = [f"{i:02x}" * 32 for i in range(5)]


def servants(rng):
    out = []
    for i in range(24):
        host = f"10.3.0.{i % 16}"  # 8 hosts with two servants: a requestor there needs the sequential solver
        envs = [DIGESTS[i % 4]] + ([DIGESTS[4]] if i % 5 == 0 else [])
        out.append(Servant(f"{host}:{8000 + i}", None, envs, 8, 8, int(rng.integers(0, 3)), 64 << 30, 48 << 30,
                           int(rng.choice([2, 4, 8])), _abi.PRIORITY_USER if i % 3 else _abi.PRIORITY_DEDICATED))
    return out


def window(rng, bound, w):
    rows = []
    for _ in range(int(rng.choice([1, 2, 3, 7, 20, 60, 300]))):
        dg = DIGESTS[int(rng.integers(0, 5))] if rng.random() < 0.85 else "ee" * 32
        ip = f"10.3.0.{int(rng.integers(0, 16))}" if rng.random() < 0.3 else f"172.20.0.{int(rng.integers(0, 9))}"
        imm = int(rng.choice([0, 1, 1, 2, 4, bound + 5, 0xFFFFFFFF], p=[0.1, 0.3, 0.2, 0.15, 0.15, 0.05, 0.05]))
        pre = int(rng.choice([0, 0, 1, 3, bound * 2]))
        rows.append((dg, int(rng.integers(0, 10)), ip, imm, pre, int(rng.choice([0, 100, 10000, 10001])),
                     int(rng.choice([1, 10, 30, 31])) * 1_000_000_000))
    if w % 7 == 3:  # fewer decisions than ranks
        rows = [(DIGESTS[0], 0, "172.20.0.1", 1, 0, 0, 10_000_000_000)]
    return rows


def arr(d, rows):
    r = np.zeros(len(rows), dtype=_abi.RPC_WAIT_DTYPE)
    for i, (dg, mv, ip, imm, pre, ms, ka) in enumerate(rows):
        r[i] = (d.intern_env(dg), mv, d.intern_ip(ip), imm, pre, ms, ka)
    return r


def packed_call(g, rpcs, now, cap=None):
    """The packed group call on every rank: [(return, results, grants8, ids)]."""
    out = []
    for r in range(g.W):
        total = int(g.lib.yd_rpc_expanded_requests(g.ranks[r]._h, rpcs[r].ctypes.data, len(rpcs[r])))
        out.append((np.zeros(len(rpcs[r]), _abi.RPC_RESULT_DTYPE), np.zeros(max(total, 1), _abi.GRANT8_DTYPE),
                    np.zeros(1, _abi.PACKED_IDS_DTYPE), total if cap is None else cap(total)))
    rets = B.par([lambda r=r: int(g.lib.yd_shard_wait_for_starting_task_rpcs_packed(
        g.ranks[r]._h, B.ns(now), rpcs[r].ctypes.data, len(rpcs[r]), out[r][0].ctypes.data, out[r][1].ctypes.data,
        out[r][3], out[r][2].ctypes.data)) for r in range(g.W)])
    return [(k, res, g8[:k] if k != REFUSED else g8[:0], ids[0]) for k, (res, g8, ids, _) in zip(rets, out)]


def run_windows(n_windows: int, world: int, case_seed: int) -> bool:
    g = B.Group("rpc-windows-packed", world, case_seed)
    t = B.Group("rpc-windows-unpacked", world, case_seed)
    g.counts.update(device_windows=0, granted=0)
    rng = np.random.default_rng(case_seed)
    ok = True
    try:
        svs = servants(rng)
        for grp in (g, t):
            grp.every(lambda d: [d.keep_servant_alive(sv, 3600.0, now=0.0) for sv in svs])
        bound = int(g.lib.yd_grant_capacity_bound(g.ranks[0]._h))
        for w in range(n_windows):
            g.ev = t.ev = f"window {w}"
            now = 1.0 + w
            rows = window(rng, bound, w)
            want_res, want_g8, want_ids = g.oracle.wait_for_starting_task_rpcs_packed(arr(g.oracle, rows), now)
            want = (want_res.tolist(), want_g8.tolist(), want_ids.tolist())
            got = packed_call(g, [arr(d, rows) for d in g.ranks], now)
            g.same("packed results, grants and ids", [(x[1].tolist(), x[2].tolist(), x[3].tolist()) for x in got], want)
            if not ordinals_are_positions(want_g8):
                g.fail("an ordinal is not its grant's place")
            t.oracle.wait_for_starting_task_rpcs(arr(t.oracle, rows), now)
            twin = B.par([lambda r=r: t.ranks[r]._rpcs_with(t.lib.yd_shard_wait_for_starting_task_rpcs, arr(t.ranks[r], rows),
                                                            now) for r in range(world)])
            unpacked = unpack_grants(want_g8, want_ids)
            t.same("unpacked twin's results and grants", [(x[0].tolist(), x[1].tolist()) for x in twin],
                   (want_res.tolist(), unpacked.tolist()))
            total = int(g.lib.yd_rpc_expanded_requests(g.ranks[0]._h, arr(g.ranks[0], rows).ctypes.data, len(rows)))
            g.counts["device_windows"] += int(total > 0)
            g.counts["granted"] += len(want_g8)
            for tid, sidx in zip(unpacked["task_id"].tolist(), unpacked["servant_index"].tolist()):
                g.outstanding[tid] = t.outstanding[tid] = sidx
            g.counts["rpc_windows"] += 1
            g.compare()
            t.compare()
            if w % 5 == 4 and total:  # cap one short: every rank refuses, nothing is decided
                before = g.oracle.next_task_id()
                rets = packed_call(g, [arr(d, rows) for d in g.ranks], now, cap=lambda n: n - 1)
                if [x[0] for x in rets] != [REFUSED] * world:
                    g.fail("a window larger than cap was not refused", rcs=[x[0] for x in rets])
                if any(d.next_task_id() != before for d in g.ranks):
                    g.fail("a refused window decided something")
                g.counts["refusals"] += 1
            if g.outstanding and rng.random() < 0.5:
                ids = sorted(g.outstanding)
                ids = [ids[i] for i in rng.choice(len(ids), size=len(ids) // 2, replace=False)]
                g.free(ids)
                t.free(ids)
                g.compare()
                t.compare()
            if w % 4 == 1:
                for grp in (g, t):
                    grp.keepalive(now + 0.5, sorted(g.outstanding)[:50] + [10**9], 5.0)
            if w % 6 == 5:
                for grp in (g, t):
                    grp.every(lambda d: d.on_expiration_timer(now=now + 0.6))
                    grp.compare()
    except B.Mismatch:
        ok = False
    print(json.dumps({"case": "rpc-windows-packed", "world": world, "ok": ok, **g.counts}), flush=True)
    g.close()
    t.close()
    return ok


def run_refusal(world: int, case_seed: int) -> bool:
    """A servant with a capacity above 8192 (replicated state): every rank returns (size_t)-1, nothing changes."""
    g = B.Group("refusal", world, case_seed)
    ok, refused = True, False
    try:
        svs = servants(np.random.default_rng(3)) + [Servant("10.9.0.1:8000", None, [DIGESTS[0]], 0, 10000, 0, 64 << 30,
                                                            48 << 30, 10000)]
        for d in g.ranks:
            [d.keep_servant_alive(sv, 3600.0, now=0.0) for sv in svs]
        rows = [(DIGESTS[0], 0, "172.20.0.1", 3, 1, 0, 10_000_000_000)] * 40
        before = [(d.next_task_id(), d.servant_state()["running_tasks"].tolist()) for d in g.ranks]
        rets = packed_call(g, [arr(d, rows) for d in g.ranks], 1.0)
        refused = all(x[0] == REFUSED for x in rets)
        ok = refused and before == [(d.next_task_id(), d.servant_state()["running_tasks"].tolist()) for d in g.ranks]
    except B.Mismatch:
        ok = False
    print(json.dumps({"case": "refusal", "world": world, "ok": ok, "refused_everywhere": refused}), flush=True)
    g.close()
    return ok


def main():
    a = B.ARGS
    ok = run_windows(a.rpcs, a.world, a.seed * 1000 + 501)
    ok = run_refusal(a.world, a.seed * 1000 + 502) and ok
    line = {"shard_rpcs_packed": ok, "world": a.world, "nccl": "real" if B.FAKE is None else "fake_nccl",
            "torch_loaded": "torch" in sys.modules}
    print(json.dumps(line), flush=True)
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
