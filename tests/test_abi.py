"""CPU-side checks of the drop-in boundary: every library exports exactly the
symbols include/ydsched.h declares, and the CUDA library refuses to run without a
GPU instead of silently computing on the CPU."""
import ctypes
import re
from pathlib import Path

import pytest

from conftest import CUDA_LIB, PORT_LIB, REF_LIB, ROOT, have_gpu
from yadcc_b200 import _abi


def header_symbols(header="ydsched.h"):
    text = (ROOT / "include" / header).read_text()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    inline = set(re.findall(r"static inline \w+ (yd_[a-z_0-9]+)\s*\(", text))  # header-only helpers, not exports
    return sorted(set(re.findall(r"\b(yd_[a-z_]+)\s*\(", text)) - inline)


def test_prototypes_cover_header():
    assert header_symbols() == sorted(name for name, _, _ in _abi.PROTOTYPES)
    assert header_symbols("ydservice.h") == sorted(name for name, _, _ in _abi.SERVICE_PROTOTYPES)
    assert header_symbols("ydwire.h") == sorted(name for name, _, _ in _abi.WIRE_PROTOTYPES)


@pytest.mark.parametrize("lib", [CUDA_LIB, PORT_LIB, REF_LIB], ids=["cuda", "port", "ref"])
def test_library_exports_every_symbol(lib, port_lib):
    if not Path(lib).exists():
        if lib == REF_LIB:
            pytest.skip("reference build not present")
        pytest.fail(f"{lib} missing: run make / __graft_entry__.build()")
    h = ctypes.CDLL(str(lib))
    for name in header_symbols() + header_symbols("ydservice.h") + header_symbols("ydwire.h"):
        assert hasattr(h, name), f"{lib} does not export {name}"


def test_struct_sizes_match_header():
    assert _abi.REQ_DTYPE.itemsize == 24  # struct yd_task_req
    assert _abi.GRANT_DTYPE.itemsize == 16  # struct yd_grant
    assert _abi.REQ16_DTYPE.itemsize == 16  # struct yd_task_req16
    assert _abi.GRANT8_DTYPE.itemsize == 8  # struct yd_grant8
    assert _abi.PACKED_IDS_DTYPE.itemsize == 16  # struct yd_packed_ids
    assert ctypes.sizeof(_abi.yd_prefilter) == 48  # struct yd_prefilter
    assert _abi.SERVANT_STATE_DTYPE.itemsize == 32
    assert ctypes.sizeof(_abi.yd_servant) == 72
    assert ctypes.sizeof(_abi.yd_running_task) == 32


def test_cuda_backend_fails_loudly_without_gpu():
    """No CPU fallback on the product path."""
    if have_gpu():
        pytest.skip("a GPU is present")
    from yadcc_b200 import TaskDispatcher

    lib = _abi.load_library(CUDA_LIB)
    assert lib.yd_backend_name() == b"cuda-sm90a"
    with pytest.raises(RuntimeError):
        TaskDispatcher(lib)


def test_missing_library_is_an_error(tmp_path, monkeypatch):
    monkeypatch.setenv("YDSCHED_LIBRARY", str(tmp_path / "nope.so"))
    with pytest.raises(FileNotFoundError):
        _abi.load_library()


def test_product_package_never_references_oracle():
    for p in (ROOT / "yadcc_b200").rglob("*"):
        if p.suffix in {".py", ".cu", ".cuh", ".h", ".cc"}:
            text = p.read_text()
            assert "libydoracle" not in text and "libydref" not in text and "oracle/" not in text.replace(
                "never touches `oracle/`", ""
            ), p
