"""The C-ABI library loads on a CPU-only box and exports every symbol include/lcd_b200.h declares;
the ctypes table in rtabmap_b200/capi.py covers exactly the same set; and the product fails
loudly (no CPU fallback) when no CUDA device exists."""
import re
from pathlib import Path

import pytest

import rtabmap_b200
from rtabmap_b200 import capi

HEADER = (Path(__file__).resolve().parent.parent / "include" / "lcd_b200.h").read_text()


def declared_symbols():
    text = re.sub(r"/\*.*?\*/", "", HEADER, flags=re.S)
    return sorted(set(re.findall(r"\b(lcd_[a-z0-9_]+)\s*\(", text)))


def test_header_declares_something():
    syms = declared_symbols()
    assert "lcd_create" in syms and "lcd_localize_batch" in syms and len(syms) >= 30


def test_library_exports_every_declared_symbol():
    lib = rtabmap_b200.load_library()
    for s in declared_symbols():
        assert hasattr(lib, s), f"liblcd_b200.so does not export {s}"
    assert lib.lcd_abi_version() == 2
    assert lib.lcd_build_arch() == b"sm_90a"


def test_ctypes_table_matches_header():
    assert sorted(capi.SIGNATURES) == declared_symbols()


def test_product_never_imports_the_oracle():
    pkg = Path(rtabmap_b200.__file__).parent
    for f in list(pkg.rglob("*.py")) + list(pkg.rglob("*.cu")) + list(pkg.rglob("*.cuh")):
        src = f.read_text()
        assert "oracle" not in src.replace("oracle/", "").lower() or "import oracle" not in src
        assert "from oracle" not in src and "import oracle" not in src and "liboracle" not in src


def test_engine_fails_loudly_without_gpu(has_gpu):
    if has_gpu:
        pytest.skip("a GPU is present")
    with pytest.raises(rtabmap_b200.LcdError):
        rtabmap_b200.Engine()


def test_verify_result_records_round_trip_through_a_byte_buffer():
    """lcd_process_fetch_async writes lcd_verify_result records into caller memory; the binding reads them back from a byte buffer.
    The record is 400 bytes (4 ints, 2 x 3 doubles, 12 floats, 36 doubles), the size the library's static_assert pins."""
    import ctypes

    import numpy as np

    n = 3
    assert ctypes.sizeof(capi.VerifyResult) == 400
    arr = (capi.VerifyResult * n)()
    for i in range(n):
        arr[i].ok, arr[i].n_matches, arr[i].n_inliers, arr[i].iterations_run = i % 2, 10 + i, 5 + i, 7
        for k in range(3):
            arr[i].rvec[k], arr[i].tvec[k] = 0.1 * k + i, 1.0 * k - i
        for k in range(36):
            arr[i].covariance[k] = 0.5 * k
    res = rtabmap_b200.Engine.results_from_buffer(np.frombuffer(bytes(arr), dtype=np.uint8), n)
    assert [r["ok"] for r in res] == [False, True, False] and res[2]["n_matches"] == 12 and res[1]["n_inliers"] == 6
    assert np.allclose(res[2]["tvec"], [-2, -1, 0]) and res[0]["covariance"].shape == (6, 6) and res[0]["covariance"][1, 0] == 3.0
