"""Fingerprints of the reference's results (oracle/_ref/libydref.so, the original sources
compiled verbatim) for the tests that compare the CPU restatement with it, so that the
comparison runs where the reference is not built.

check_reference(key, run, mine) asserts that `mine` equals what the reference produced for
`key`: a SHA-256 over every array's dtype, shape and bytes and every other value, stored in
tests/golden/reference_results.json.  Where the reference is built, `run()` -- the same work on
the reference -- is also called and compared in full; YD_WRITE_REFERENCE_RESULTS=1 then stores
its fingerprint instead of checking it.
"""
import hashlib
import json
import os
from pathlib import Path

import numpy as np

from conftest import REF_LIB

STORE = Path(__file__).parent / "golden" / "reference_results.json"


def _feed(h, x) -> None:
    if isinstance(x, np.ndarray):
        a = np.ascontiguousarray(x)
        h.update(f"nd{a.dtype.str}{a.shape}".encode())
        h.update(a.tobytes())
    elif isinstance(x, (list, tuple)):
        h.update(f"seq{len(x)}[".encode())
        for v in x:
            _feed(h, v)
        h.update(b"]")
    elif isinstance(x, dict):
        h.update(f"map{len(x)}{{".encode())
        for k in sorted(x, key=repr):
            _feed(h, k)
            _feed(h, x[k])
        h.update(b"}")
    else:
        h.update(f"{type(x).__name__}:{x!r};".encode())


def fingerprint(x) -> str:
    h = hashlib.sha256()
    _feed(h, x)
    return h.hexdigest()


def _same(a, b) -> bool:
    if isinstance(a, np.ndarray) or isinstance(b, np.ndarray):
        a, b = np.asarray(a), np.asarray(b)
        return a.shape == b.shape and a.dtype == b.dtype and bool((a == b).all())
    if isinstance(a, (list, tuple)):
        return isinstance(b, (list, tuple)) and len(a) == len(b) and all(_same(x, y) for x, y in zip(a, b))
    if isinstance(a, dict):
        return isinstance(b, dict) and a.keys() == b.keys() and all(_same(a[k], b[k]) for k in a)
    return a == b


def check_reference(key: str, run, mine) -> None:
    stored = json.loads(STORE.read_text()) if STORE.exists() else {}
    if REF_LIB.exists():
        live = run()
        assert _same(live, mine), f"{key}: differs from the reference"
        if os.environ.get("YD_WRITE_REFERENCE_RESULTS"):
            stored[key] = fingerprint(live)
            STORE.write_text(json.dumps(stored, indent=1, sort_keys=True) + "\n")
    assert key in stored, f"{key}: no stored reference result (build the reference, set YD_WRITE_REFERENCE_RESULTS=1)"
    assert fingerprint(mine) == stored[key], f"{key}: differs from the reference's stored result"
