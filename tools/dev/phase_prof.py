#!/usr/bin/env python
"""Phase stamps of the fused kernel (YDSCHED_FUSED_PROF=1), L2 flushed / warm: python tools/dev/phase_prof.py cfg2-mod

For every speculative solve (variant 4) it also prints each block's stamps as min / median / max over the blocks: its
start, each item of phase A by kind (request tile, slot tile, class), the barrier arrival and wait, phase B and its end
-- in us from the first block's start --, the links of phase B and the servant counters (from the barrier departure
of the blocks that count them) and the CUDA-event time of the same solve, whose excess over the kernel's span
(first block's start to the last block's end) is the launch and the drain."""
import os, sys, tempfile, time
from pathlib import Path
sys.path.insert(0, str(Path(__file__).resolve().parent.parent.parent))
import numpy as np
import torch
from bench import build_workload
from yadcc_b200 import STATUS_GRANTED, TaskDispatcher, pack_requests, unpack_grants

KINDS = {1: "request tile", 2: "slot tile", 3: "class item"}
WORDS = 12  # fused.cuh: kProfBlockWords


def captured(fn):
    """fn()'s return value and what the library printed to stderr meanwhile."""
    sys.stderr.flush()
    saved = os.dup(2)
    with tempfile.TemporaryFile() as f:
        os.dup2(f.fileno(), 2)
        try:
            r = fn()
        finally:
            os.dup2(saved, 2)
            os.close(saved)
        f.seek(0)
        return r, f.read().decode()


def block_stamps(line):
    """(per-block stamps as a G x WORDS array, the last block's end) of one `ydsched: fused blocks` line."""
    tok = line.split()
    G, last_end = int(tok[3]), int(tok[5])
    return np.array([int(x) for x in tok[7:]], dtype=np.int64).reshape(G, WORDS), last_end


def kernel_span(b, last_end):
    """us from the first block's start to the last block done (report and clean-up included)."""
    return (max(b[:, 6].max(), last_end) - b[:, 0].min()) / 1e3


def block_table(line, event_us):
    """The per-block stamps of one `ydsched: fused blocks` line, as rows of (label, values in us)."""
    b, last_end = block_stamps(line)
    G = len(b)
    t0 = b[:, 0].min()
    rows = [("start", (b[:, 0] - t0) / 1e3)]
    per_kind = {}
    for i in range(G):
        kinds, count = int(b[i, 7]) & 0xFFFF, int(b[i, 7]) >> 16
        prev = b[i, 0]
        for k in range(min(count, 3)):
            kind = (kinds >> (4 * k)) & 15
            label = f"{KINDS.get(kind, kind)}{' (2nd item)' if k else ''}"
            per_kind.setdefault(label, []).append((b[i, 1 + k] - prev) / 1e3)
            prev = b[i, 1 + k]
    for label in sorted(per_kind):
        rows.append((f"{label}, n={len(per_kind[label])}", np.array(per_kind[label])))
    rows += [
        ("barrier arrival", (b[:, 4] - t0) / 1e3),
        ("barrier wait", (b[:, 5] - b[:, 4]) / 1e3),
        ("phase B", (b[:, 6] - b[:, 5]) / 1e3),
        ("end of B", (b[:, 6] - t0) / 1e3),
    ]
    # phase B of the block's first request tile, link by link (blocks without a request tile leave words 8..10 at 0)
    tiled = b[b[:, 10] != 0]
    if len(tiled):
        rows += [
            (f"B: tables, n={len(tiled)}", (tiled[:, 8] - tiled[:, 5]) / 1e3),
            ("B: selection", (tiled[:, 9] - tiled[:, 8]) / 1e3),
            ("B: final_tile", (tiled[:, 10] - tiled[:, 9]) / 1e3),
        ]
    # the blocks that counted the servants' grants (word 11), from their barrier departure
    counting = b[b[:, 11] != 0]
    if len(counting):
        rows.append((f"B: servant counters, n={len(counting)}", (counting[:, 11] - counting[:, 5]) / 1e3))
    span = kernel_span(b, last_end)
    head = (f"    {G} blocks; kernel span {span:.1f} us (first start .. last block done, report and clean-up included), "
            f"event {event_us:.1f} us, launch + drain {event_us - span:.1f} us")
    return head, rows


if __name__ == "__main__":
    os.environ["YDSCHED_FUSED_PROF"] = "1"
    for name in sys.argv[1:] or ["cfg2-mod"]:
        w = build_workload(name)
        d = TaskDispatcher()
        w.register(d, now=0.0, expires_in=3600.0)
        src = w.build_requests(d)
        reqs = d.alloc_requests(len(src)); reqs[...] = src
        out = d.alloc_grants(len(src))
        r16 = pack_requests(src, d.alloc_requests16(len(src)))
        o8 = d.alloc_grants8(len(src))
        flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
        for it in range(14):
            mode = "staged" if it < 10 else "e2e-packed"
            cold = it >= 3
            if mode == "staged":
                d.stage_requests(reqs)
            if cold:
                flush.fill_(it); torch.cuda.synchronize()
            print(f"{name} {mode} {'cold' if cold else 'warm'}:", file=sys.stderr, end=" ", flush=True)
            t0 = time.perf_counter()
            if mode == "staged":
                (g, text) = captured(lambda: d.wait_for_staged_tasks(len(src), 1.0 + it, out=out))
            else:
                ((g8, ids), text) = captured(lambda: d.wait_for_starting_new_tasks_packed(r16, 1.0 + it, out8=o8, unpack=False))
            t1 = time.perf_counter()
            if mode != "staged":
                g = unpack_grants(g8, ids)
            st = d.last_solve_stats()
            event_us = 1e3 * (st['prep_ms'] + st['solve_ms'] + st['final_ms'])
            print(f"   device {event_us:.1f} us total {st['total_ms']*1e3:.1f} host {1e6*(t1-t0):.1f} us launches {st['kernel_launches']}", file=sys.stderr, flush=True)
            for line in text.splitlines():
                if not line.startswith("ydsched: fused blocks"):
                    print("   " + line, file=sys.stderr)
                elif mode == "staged":
                    head, rows = block_table(line, event_us)
                    print(head, file=sys.stderr)
                    print(f"    {'us':34s} {'min':>6s} {'median':>6s} {'max':>6s}", file=sys.stderr)
                    for label, v in rows:
                        print(f"    {label:34s} {v.min():6.1f} {np.median(v):6.1f} {v.max():6.1f}", file=sys.stderr)
            d.free_tasks(g["task_id"][g["status"] == STATUS_GRANTED].copy())
            d.on_expiration_timer(now=1.5 + it)
        d.close()
