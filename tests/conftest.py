"""Shared fixtures.  Backends:

  port  oracle/libydoracle.so      CPU restatement (always buildable: g++ only)
  ref   oracle/_ref/libydref.so    reference sources compiled verbatim (present
                                   when built in the dev container; travels to
                                   the GPU box as a prebuilt file)
  cuda  yadcc_b200/libydsched.so   the product; needs an H100 -> @pytest.mark.gpu
"""
import os
import subprocess
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

PORT_LIB = ROOT / "oracle" / "libydoracle.so"
REF_LIB = ROOT / "oracle" / "_ref" / "libydref.so"
CUDA_LIB = ROOT / "yadcc_b200" / "libydsched.so"


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a real H100 (run with -m gpu)")


def _ensure_port():
    if not PORT_LIB.exists():
        subprocess.check_call(["make", "-C", str(ROOT / "oracle"), "libydoracle.so"])
    return PORT_LIB


def have_gpu() -> bool:
    if os.environ.get("YD_FORCE_NO_GPU"):
        return False
    try:
        import torch

        return torch.cuda.is_available()
    except Exception:
        return False


@pytest.fixture(scope="session")
def port_lib():
    return str(_ensure_port())


@pytest.fixture(scope="session")
def ref_lib():
    if not REF_LIB.exists():
        pytest.skip("oracle/_ref/libydref.so not built (needs /root/reference)")
    return str(REF_LIB)


@pytest.fixture(scope="session")
def cuda_lib():
    assert CUDA_LIB.exists(), "yadcc_b200/libydsched.so missing: run `make` / __graft_entry__.build()"
    return str(CUDA_LIB)


def cpu_backends():
    out = [pytest.param("port", id="port")]
    out.append(pytest.param("ref", id="ref"))
    return out


@pytest.fixture
def make_dispatcher(request):
    """Factory: make_dispatcher('port'|'ref'|'cuda', **kw) -> TaskDispatcher."""
    from yadcc_b200 import TaskDispatcher

    made = []

    def factory(kind: str, **kw):
        if kind == "port":
            lib = str(_ensure_port())
        elif kind == "ref":
            if not REF_LIB.exists():
                pytest.skip("oracle/_ref/libydref.so not built (needs /root/reference)")
            lib = str(REF_LIB)
        elif kind == "cuda":
            assert CUDA_LIB.exists(), "yadcc_b200/libydsched.so missing"
            lib = str(CUDA_LIB)
        else:
            raise ValueError(kind)
        d = TaskDispatcher(lib, **kw)
        made.append(d)
        return d

    yield factory
    for d in made:
        d.close()
