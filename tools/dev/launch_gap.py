#!/usr/bin/env python
"""Where the time of a staged solo solve goes outside its kernel: python tools/dev/launch_gap.py [--solves 60] [--out f.json]

bench.py's `value` for cfg2-mod is the CUDA-event time around a staged solve, L2 flushed before each.  This probe makes
bench.py's staged calls (free the previous grants, tick, flush L2 with a 256 MiB write, synchronise, stage, solve) and
prints the median and range over the solves, each quantity in a pass of its own so that no measurement disturbs another:

  event      ev[1] -> ev[4] on the solve stream, as bench.py computes it (prep_ms + solve_ms + final_ms)
  span       the kernel's %globaltimer span, first block's start to the last block's end (YDSCHED_FUSED_PROF,
             phase_prof.py's parsing)
  kernel     k_fused_front's device duration from torch.profiler (CUDA activities)
  host       YDSCHED_HOST_PROF's "launch" (host time from ev[1]'s record to ev[4]'s, inside the window) and the
             field before it (upload and preparation, before the window)
  floors     an empty kernel of the same launch shape (launch_floor.cu) on an idle stream after the same flush:
             a patched one-node graph, the same graph behind an external event-wait node, and a direct launch

It also counts the YDSCHED_DEBUG `variant` / `graph` fields of the timed solves.  Nothing here changes a device
setting; the floor kernel is compiled with nvcc into a temporary directory."""
import argparse, ctypes, json, os, re, subprocess, sys, tempfile
from pathlib import Path

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE.parent.parent))
sys.path.insert(0, str(HERE))
import numpy as np
import torch
from bench import build_workload
from phase_prof import block_stamps, captured, kernel_span
from yadcc_b200 import STATUS_GRANTED, TaskDispatcher

ENVS = ("YDSCHED_HOST_PROF", "YDSCHED_FUSED_PROF", "YDSCHED_DEBUG")


def staged_solves(w, flush, n, env=(), hook=None):
    """bench.py's staged steps on a fresh handle (created with the given switches): 5 warm-up solves, then n timed.
    hook(stats, stderr text) per timed solve."""
    for k in ENVS:
        os.environ.pop(k, None)
    for k in env:
        os.environ[k] = "1"
    d = TaskDispatcher()
    for k in env:
        os.environ.pop(k)
    try:
        w.register(d, now=0.0, expires_in=3600.0)
        src = w.build_requests(d)
        reqs = d.alloc_requests(len(src))
        reqs[...] = src
        out = d.alloc_grants(len(src))
        prev = None
        for it in range(5 + n):
            now = 2.0 + it
            if prev is not None:
                d.free_tasks(prev)
            d.on_expiration_timer(now=now)
            flush.fill_(~it & 0xFF)
            torch.cuda.synchronize()
            d.stage_requests(reqs)
            g, text = captured(lambda: d.wait_for_staged_tasks(len(src), now, out=out))
            prev = g["task_id"][g["status"] == STATUS_GRANTED].copy()
            if it >= 5 and hook is not None:
                hook(d.last_solve_stats(), text)
        d.free_tasks(prev)
    finally:
        d.close()


def build_floor(tmp):
    so = Path(tmp) / "liblaunch_floor.so"
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    subprocess.check_call([nvcc, "-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-Xcompiler", "-fPIC",
                           "-shared", "-o", str(so), str(HERE / "launch_floor.cu")])
    lib = ctypes.CDLL(str(so))
    lib.floor_init.argtypes = [ctypes.c_uint, ctypes.c_size_t]
    lib.floor_once.argtypes = [ctypes.c_int]
    lib.floor_once.restype = ctypes.c_float
    lib.floor_error.restype = ctypes.c_char_p
    return lib


def stat(v):
    v = np.asarray(v, dtype=np.float64)
    return {"median": round(float(np.median(v)), 2), "min": round(float(v.min()), 2), "max": round(float(v.max()), 2),
            "n": int(len(v))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="cfg2-mod")
    ap.add_argument("--solves", type=int, default=60)
    ap.add_argument("--out", default=None, help="also write the result as JSON here")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "launch_gap.py measures on a GPU"
    w = build_workload(a.workload)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    res, debug = {}, {"variant": {}, "graph": {}}

    event = []
    staged_solves(w, flush, a.solves, hook=lambda st, t: event.append(1e3 * (st["prep_ms"] + st["solve_ms"] + st["final_ms"])))
    res["event_us"] = stat(event)

    host_launch, host_before, shape = [], [], {}

    def on_host(st, text):
        m = re.search(r"host us: .*\) (\S+) ([\d.]+) launch ([\d.]+)", text)
        host_before.append(float(m.group(2)))
        host_launch.append(float(m.group(3)))
        m = re.search(r"ydsched: solve n .* variant (\d+) .* slot_b (\d+) cls_bound (\d+) .* graph (\d+) ", text)
        for k, v in (("variant", m.group(1)), ("graph", m.group(4))):
            debug[k][v] = debug[k].get(v, 0) + 1
        shape["slot_b"], shape["cls_bound"] = int(m.group(2)), int(m.group(3))
    staged_solves(w, flush, a.solves, env=("YDSCHED_HOST_PROF", "YDSCHED_DEBUG"), hook=on_host)
    res["host_launch_us"] = stat(host_launch)
    res["host_before_window_us"] = stat(host_before)

    span, span_event = [], []

    def on_span(st, text):
        line = next((x for x in text.splitlines() if x.startswith("ydsched: fused blocks")), None)
        if line is not None:
            span.append(kernel_span(*block_stamps(line)))
            span_event.append(1e3 * (st["prep_ms"] + st["solve_ms"] + st["final_ms"]))
    staged_solves(w, flush, a.solves, env=("YDSCHED_FUSED_PROF",), hook=on_span)
    res["span_us"] = stat(span) if span else None
    res["event_us_profiled"] = stat(span_event) if span_event else None

    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        staged_solves(w, flush, a.solves)
    kern = [e.time_range.elapsed_us() for e in prof.events()
            if e.device_type == DeviceType.CUDA and "k_fused_front" in e.name]
    res["kernel_us"] = stat(kern[-a.solves:]) if kern else None

    # the floors, with the solo kernel's dynamic shared memory (ydsched.cu FusedLoffWords)
    words = shape["cls_bound"] * ((shape["slot_b"] + 1023) // 1024 + 1) + 1
    dyn = 4 * words if words <= 16384 else 0
    grid = torch.cuda.get_device_properties(0).multi_processor_count
    with tempfile.TemporaryDirectory() as tmp:
        lib = build_floor(tmp)
        assert lib.floor_init(grid, dyn) == 0, ("floor_init", lib.floor_error())
        floors = {0: [], 1: [], 2: []}
        for it in range(5 + a.solves):
            for mode in (0, 1, 2):
                flush.fill_(it & 0xFF)
                torch.cuda.synchronize()
                ms = lib.floor_once(mode)
                assert ms >= 0, ("floor_once", mode, lib.floor_error())
                if it >= 5:
                    floors[mode].append(1e3 * ms)
        lib.floor_close()
    res["floor_graph_patched_us"] = stat(floors[0])
    res["floor_graph_wait_node_us"] = stat(floors[1])
    res["floor_direct_us"] = stat(floors[2])
    res["floor_shape"] = {"grid": grid, "block": 1024, "static_smem": 43744, "dyn_smem": dyn, "arg_bytes": 832}
    res["debug"] = debug
    res["gpu"] = torch.cuda.get_device_name(0)
    try:
        res["power_limit"] = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"],
                                            capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        res["power_limit"] = None

    for k, v in res.items():
        if isinstance(v, dict) and "median" in v:
            print(f"{k:28s} median {v['median']:7.2f}  min {v['min']:7.2f}  max {v['max']:7.2f}  (n {v['n']})")
    print(json.dumps(res))
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        Path(a.out).write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
