"""CPU: the C-ABI shared library builds, loads and exports every symbol include/fear_b200.h declares."""
import os
import re

import pytest

from feartracker_b200 import _lib, build

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    build.build()  # cross-compiles for sm_90a without a GPU
    return _lib.load()


def _declared_symbols():
    with open(os.path.join(ROOT, "include", "fear_b200.h")) as f:
        text = re.sub(r"/\*.*?\*/", "", f.read(), flags=re.S)
    return sorted(set(re.findall(r"\b(fear_[a-z0-9_]+)\s*\(", text)))


def test_every_declared_symbol_is_exported_and_bound(lib):
    declared = _declared_symbols()
    assert len(declared) >= 20
    for name in declared:
        assert hasattr(lib, name), f"libfear_b200.so does not export {name}"
    assert declared == _lib.exported_symbols(), "ctypes signature table out of sync with the header"


def test_weight_table_and_stage_names(lib):
    assert lib.fear_abi_version() == 1
    table = _lib.weight_table()
    names = [n for n, _ in table]
    assert len(names) == len(set(names)) == 124
    assert names[0] == "stem.w" and names[-1] == "cls_pred.pw.b"
    assert dict(table)["xif4_5.pw.w"] == 672 * 112 and dict(table)["reg_dw.pw.w"] == 256 * 320
    assert "corr" in _lib.stage_names()


def test_calls_fail_loudly_without_device(lib):
    import torch

    if torch.cuda.is_available():
        pytest.skip("GPU present")
    assert lib.fear_init(0) != 0
    assert "CUDA" in _lib.last_error() or "device" in _lib.last_error()
    with pytest.raises(RuntimeError):
        _lib.init(0)
