#!/usr/bin/env python
"""The merge solver's record window on a range-sharded group (kRqMargin, parallel.cuh), on ONE GPU: W rank handles in
W threads of one process over the test-only NCCL stand-in, driven by shard_threads_check.py's harness (imported first:
it loads tests/fake_nccl/libnccl.so.2 with RTLD_GLOBAL; this process must not import torch).

Each case of merge_cases.SHARDED is one batch, cut into W equal ranges so that the class's records lie on every rank,
and checked after every event against one CPU checker fed the whole queue.  Prints one JSON line per case (its
`handbacks`: 1 when the group decided the whole queue instead) and a final {"shard_parity": ...} line; exit code 0 iff
everything matched.
"""
import argparse
import json
import sys

_argv, sys.argv = sys.argv, sys.argv[:1]
import shard_threads_check as T  # noqa: E402  (loads the NCCL stand-in before anything else)
sys.argv = _argv

import merge_cases as M  # noqa: E402


class EvenCuts(T.Harness):
    def cut_points(self, n: int):
        return [n * g // self.W for g in range(self.W + 1)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--world", type=int, default=2)
    ap.add_argument("--cases", default=",".join(M.SHARDED))
    a = ap.parse_args()
    ok = True
    for k, name in enumerate(x for x in a.cases.split(",") if x):
        h = EvenCuts(name, a.world, k)
        try:
            h.run(T.make_handles_streams(h, lambda d, name=name: M.stream(d, M.SHARDED[name])))
            good = True
        except T.Mismatch:
            good = False
        print(json.dumps({"case": name, "world": a.world, "ok": good, **h.counts}), flush=True)
        h.close()
        ok = ok and good
    a4 = (T.C.c_ulonglong * 4)()
    T.FAKE.yd_fake_nccl_stats(0, a4)
    print(json.dumps({"shard_parity": ok, "world": a.world, "fake_nccl_collectives": int(a4[0]),
                      "torch_loaded": "torch" in sys.modules}), flush=True)
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
