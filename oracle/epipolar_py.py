"""ctypes binding of oracle/liboracle_epipolar.so, the CPU restatement of EpipolarGeometry::check (oracle_epipolar.cpp), and the
epipolar outcome of Rtabmap::process's decision on top of oracle/decide_py.py — TEST INFRASTRUCTURE ONLY (tests/, tools/).

Rtabmap.cpp:2193 runs the check between the single-hypothesis rejection and the ratio rejections, so a frame reaches it exactly when
decide_py gives it RATIO, LAST_NULL or ACCEPTED; a failed check makes it EPIPOLAR_REJECTED with no loop id, and the highest hypothesis
stays as the decision left it.
"""
from __future__ import annotations

import ctypes as C
import subprocess
from pathlib import Path

import numpy as np

from oracle import decide_py as dp

HERE = Path(__file__).resolve().parent
LIB = HERE / "liboracle_epipolar.so"
SRCS = [HERE / "oracle_epipolar.cpp", HERE / "oracle.cpp", HERE / "oracle_verify.cpp", HERE / "pnp_math.h",
        HERE.parent / "rtabmap_b200" / "csrc" / "fm_solver.h"]

METHOD_NONE, METHOD_7POINT, METHOD_LMEDS, METHOD_RANSAC = range(4)
EPIPOLAR_REJECTED = 11
_lib = None


def build() -> None:
    """Compile liboracle_epipolar.so when it is missing or older than its sources, with the flags of oracle/Makefile.  It includes
    oracle_verify.cpp, whose PnP oracle calls into oracle.cpp."""
    if LIB.exists() and LIB.stat().st_mtime >= max(s.stat().st_mtime for s in SRCS):
        return
    tmp = LIB.with_name(f".{LIB.name}.tmp")
    subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-w", "-ffp-contract=off", "-shared", "-o", str(tmp),
                    str(SRCS[0]), str(SRCS[1])], check=True, capture_output=True, cwd=str(HERE))
    tmp.replace(LIB)


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        build()
        L = C.CDLL(str(LIB))
        P, I, D = C.c_void_p, C.c_int, C.c_double
        L.epo_find_pairs_unique.argtypes = [P, I, P, I, P, P, P]
        L.epo_find_pairs_unique.restype = I
        L.epo_find_fundamental.argtypes = [P, P, I, D, D, I, P, P, P]
        L.epo_find_fundamental.restype = I
        L.epo_run_7point.argtypes = [P, P, P]
        L.epo_run_7point.restype = I
        _lib = L
    return _lib


def _p(a: np.ndarray):
    return a.ctypes.data_as(C.c_void_p)


def find_pairs_unique(ids_a, ids_b):
    """EpipolarGeometry::findPairsUnique: (word ids, rows in A, rows in B) of the ids >= 0 found exactly once on each side, ascending."""
    a = np.ascontiguousarray(ids_a, np.int32)
    b = np.ascontiguousarray(ids_b, np.int32)
    m = max(min(len(a), len(b)), 1)
    ra, rb, ids = np.zeros(m, np.int32), np.zeros(m, np.int32), np.zeros(m, np.int32)
    n = lib().epo_find_pairs_unique(_p(a), len(a), _p(b), len(b), _p(ra), _p(rb), _p(ids))
    return ids[:n], ra[:n], rb[:n]


def find_fundamental(p1, p2, param1: float = 3.0, param2: float = 0.99, check_subset: bool = True) -> dict:
    """cv2.findFundamentalMat(p1, p2, cv2.FM_RANSAC, param1, param2) as OpenCV 4.13 runs it on float32 points."""
    a = np.ascontiguousarray(p1, np.float32).reshape(-1, 2)
    b = np.ascontiguousarray(p2, np.float32).reshape(-1, 2)
    n = len(a)
    mask = np.zeros(max(n, 1), np.uint8)
    F = np.zeros(9, np.float64)
    info = np.zeros(4, np.int32)
    inl = lib().epo_find_fundamental(_p(a), _p(b), n, float(param1), float(param2), int(check_subset), _p(mask), _p(F), _p(info))
    return {"mask": mask[:n], "F": F.reshape(3, 3) if info[1] else None, "n_inliers": int(inl), "method": int(info[0]),
            "found": int(info[1]), "iterations": int(info[2]), "raises": int(info[3])}


def run_7point(p1, p2):
    """The 7-point kernel alone: its models as a (k, 3, 3) array (k = -1 when the determinant polynomial vanishes identically)."""
    a = np.ascontiguousarray(p1, np.float32).reshape(7, 2)
    b = np.ascontiguousarray(p2, np.float32).reshape(7, 2)
    F = np.zeros(27, np.float64)
    k = lib().epo_run_7point(_p(a), _p(b), _p(F))
    return k, F.reshape(3, 3, 3)[:max(k, 0)]


def check(ids_a, uv_a, ids_b, uv_b, match_count_min: int = 8, param1: float = 3.0, param2: float = 0.99) -> dict:
    """EpipolarGeometry::check(A = new frame, B = hypothesis) over word ids and their keypoints (row i = word i).  Where the reference
    fails (no matrix returned, or OpenCV raises) the check is a rejection."""
    ids, ra, rb = find_pairs_unique(ids_a, ids_b)
    out = {"n_pairs": len(ids), "ok": 0, "n_inliers": 0, "method": METHOD_NONE, "found": 0, "iterations": 0, "raises": 0,
           "F": None, "mask": np.zeros(len(ids), np.uint8)}
    if len(ids) < match_count_min or len(ids) < 7:
        return out
    r = find_fundamental(np.asarray(uv_a, np.float32)[ra], np.asarray(uv_b, np.float32)[rb], param1, param2)
    out.update(r)
    out["ok"] = int(r["found"] and r["n_inliers"] >= match_count_min)
    if not r["found"]:
        out["n_inliers"] = 0
    return out


def decide_epipolar(decision, epipolar_ok: bool | None):
    """A decide_py decision after the epipolar check of its highest hypothesis (None: the frame was not checked)."""
    hid, hval, loop_id, status = decision
    if epipolar_ok is None or status not in (dp.RATIO, dp.LAST_NULL, dp.ACCEPTED) or epipolar_ok:
        return decision
    return hid, hval, 0, EPIPOLAR_REJECTED
