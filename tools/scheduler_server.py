#!/usr/bin/env python
"""A minimal yadcc scheduler endpoint: TCP in, FlareStd frames through include/ydwire.h, TCP out.

    python tools/scheduler_server.py --port 8336 --user-tokens some_fancy_token \\
        --servant-tokens some_fancy_token [--library <any library speaking the ydsched C ABI>]

An unmodified yadcc daemon pointed at flare://host:8336 heartbeats, asks for grants, renews and
frees them against it.  All frames that arrive within one batching window (--window-ms) are
handed to ONE yd_wire_handle_frames call, so concurrent WaitForStartingTask RPCs become one
batched GPU solve; answers are what serving the frames one by one in arrival order would give.
The 1 Hz expiration sweep (task_dispatcher.cc:81-82) runs from the same loop.  This is glue for
demos and tests, not a production server: one thread, no TLS, no back-pressure.

With --state FILE a restart keeps the scheduler's servants, leases and task ids: the state is
imported from FILE at start if it exists, and exported to it (a temporary file, then a rename) when
the process gets SIGINT or SIGTERM.  Nothing else goes into the file: the import rebases every time
onto the new process's clock (include/ydstate.h), so the two processes need no common clock."""
from __future__ import annotations

import argparse
import asyncio
import os
import signal
import struct
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
from yadcc_b200 import TaskDispatcher  # noqa: E402
from yadcc_b200.service import SchedulerService  # noqa: E402


class Endpoint:
    def __init__(self, svc: SchedulerService, window_ms: float):
        self.svc = svc
        self.window = window_ms / 1e3
        self.pending: list[tuple[bytes, str, bool, asyncio.StreamWriter]] = []
        self.wake = asyncio.Event()
        self.t0 = time.monotonic()

    def now(self) -> float:
        return time.monotonic() - self.t0

    async def client(self, reader: asyncio.StreamReader, writer: asyncio.StreamWriter):
        peer = writer.get_extra_info("peername")
        ip, v6 = peer[0], ":" in peer[0]
        buf = b""
        try:
            while True:
                while len(buf) < 16 or len(buf) < 16 + sum(struct.unpack("<III", buf[4:16])):
                    if len(buf) >= 4 and buf[:4] != b"CPRF":  # 'FRPC' little endian
                        return
                    chunk = await reader.read(65536)
                    if not chunk:
                        return
                    buf += chunk
                n = 16 + sum(struct.unpack("<III", buf[4:16]))
                self.pending.append((buf[:n], ip, v6, writer))
                buf = buf[n:]
                self.wake.set()
        finally:
            writer.close()

    async def pump(self):
        last_tick = self.now()
        while True:
            try:
                await asyncio.wait_for(self.wake.wait(), timeout=0.25)
            except asyncio.TimeoutError:
                pass
            self.wake.clear()
            if self.pending:
                await asyncio.sleep(self.window)  # let the batch fill
                batch, self.pending = self.pending, []
                outs = self.svc.handle_frames([(f, ip, v6) for f, ip, v6, _ in batch], now=self.now())
                for (verdict, _consumed, _status, frame), (_, _, _, w) in zip(outs, batch):
                    if verdict == 1 and frame:
                        w.write(frame)
                    elif verdict == -1:
                        w.close()
            if self.now() - last_tick >= 1.0:
                last_tick = self.now()
                self.svc.dispatcher.on_expiration_timer(now=last_tick)


def save_state(d: TaskDispatcher, path: str, now: float) -> None:
    """Export the dispatcher's state to `path` atomically: a reader sees the old file or the new one."""
    tmp = f"{path}.tmp.{os.getpid()}"
    with open(tmp, "wb") as f:
        f.write(d.export_state(now=now))
        f.flush()
        os.fsync(f.fileno())
    os.replace(tmp, path)


async def serve(args, ready: asyncio.Event | None = None):
    d = TaskDispatcher(args.library) if args.library else TaskDispatcher()
    if args.state and os.path.exists(args.state):
        with open(args.state, "rb") as f:
            d.import_state(f.read(), now=0.0)  # now = 0 on the endpoint's clock, which starts below
    svc = SchedulerService(d, acceptable_user_tokens=args.user_tokens, acceptable_servant_tokens=args.servant_tokens,
                           min_daemon_version=args.min_daemon_version)
    ep = Endpoint(svc, args.window_ms)
    server = await asyncio.start_server(ep.client, args.host, args.port)
    work = asyncio.gather(server.serve_forever(), ep.pump())
    stopped = []
    if args.state:
        def stop():
            save_state(d, args.state, ep.now())
            stopped.append(True)
            work.cancel()

        loop = asyncio.get_running_loop()
        for sig in (signal.SIGINT, signal.SIGTERM):
            loop.add_signal_handler(sig, stop)
    if ready is not None:
        ready.set()
    async with server:
        try:
            await work
        except asyncio.CancelledError:
            if not stopped:
                raise


def parse_args(argv=None):
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--host", default="127.0.0.1")
    ap.add_argument("--port", type=int, default=8336)
    ap.add_argument("--user-tokens", required=True)
    ap.add_argument("--servant-tokens", required=True)
    ap.add_argument("--min-daemon-version", type=int, default=0)
    ap.add_argument("--window-ms", type=float, default=1.0)
    ap.add_argument("--library", default=None, help="ydsched C-ABI library (default: the CUDA build)")
    ap.add_argument("--state", default=None,
                    help="state file: imported at start if it exists, exported on SIGINT / SIGTERM (include/ydstate.h)")
    return ap.parse_args(argv)


if __name__ == "__main__":
    asyncio.run(serve(parse_args()))
