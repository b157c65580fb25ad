"""CPU oracle of the GPS filter of Rtabmap::process's place list (Rtabmap/LoopGPS) and of the decision over the filtered list, for
localisation clients — TEST INFRASTRUCTURE ONLY (tests/, tools/).

Restates, statement by statement, in double with float where the reference uses float:
  GeodeticCoords::toGeocentric_WGS84           GeodeticCoords.cpp:75-102    (math: glibc's libm, as the compiled reference)
  GeodeticCoords::Geocentric_WGS84ToENU_WGS84  GeodeticCoords.cpp:119-149
  the construction of signaturesToCompare     Rtabmap.cpp:2046-2115, localisation mode (originOffsetENU = identity)
Both geodetic functions are pinned bit for bit to the reference's own GeodeticCoords.cpp, compiled into oracle/_ref/libref_geodetic.so
by oracle/geodetic.mk (tests/test_oracle_gps.py).

The decision over the filtered list (`GpsClient`) composes the restatements that already exist: adjustLikelihood (oracle_py),
the Bayes filter over the compared ids (bayes_py's sparse restatement, or the reference's compiled BayesFilter.cpp, which takes any key
set) and the hypothesis selection (decide_py).
"""
from __future__ import annotations

import ctypes as C
import math
import subprocess
from pathlib import Path

import numpy as np

from oracle import decide_py as dc
from oracle import oracle_py as orc
from oracle.bayes_py import _repeated_float_add, prediction_columns

HERE = Path(__file__).resolve().parent
REF_GEO_LIB = HERE / "_ref" / "libref_geodetic.so"
_ref_geo = None

f32 = np.float32
_A = 6378137.0           # semi-major axis (m)
_B = 6356752.3142        # semi-minor axis
_AE = math.acos(_B / _A)
_COS2 = math.cos(_AE) * math.cos(_AE)
_SIN2 = math.sin(_AE) * math.sin(_AE)


def build() -> None:
    """Compile _ref/libref_geodetic.so from the reference's GeodeticCoords.cpp when it is missing and the reference is present."""
    if not REF_GEO_LIB.exists() and orc._reference_present():
        subprocess.run(["make", "-C", str(HERE), "-f", "geodetic.mk"], check=True, capture_output=True)


def ref_geo_lib():
    """The reference's compiled GeodeticCoords, or None when it has not been built."""
    global _ref_geo
    if _ref_geo is None:
        build()
        if not REF_GEO_LIB.exists():
            return None
        R = C.CDLL(str(REF_GEO_LIB))
        D, P = C.c_double, C.c_void_p
        R.ref_geo_geocentric.argtypes = [D, D, D, P]
        R.ref_geo_enu.argtypes = [P, P, D, D, D, P]
        _ref_geo = R
    return _ref_geo


def ref_geocentric(lat, lon, alt):
    out = np.zeros(3, np.float64)
    ref_geo_lib().ref_geo_geocentric(float(lat), float(lon), float(alt), out.ctypes.data_as(C.c_void_p))
    return out


def ref_enu(point, origin_point, lat, lon, alt=0.0):
    p = np.ascontiguousarray(point, np.float64)
    o = np.ascontiguousarray(origin_point, np.float64)
    out = np.zeros(3, np.float64)
    ref_geo_lib().ref_geo_enu(p.ctypes.data_as(C.c_void_p), o.ctypes.data_as(C.c_void_p), float(lat), float(lon), float(alt),
                              out.ctypes.data_as(C.c_void_p))
    return out


def geocentric(lat: float, lon: float, alt: float):
    """GeodeticCoords(lat, lon, alt).toGeocentric_WGS84() -> (x, y, z)."""
    lon_r = lon * math.pi / 180.0
    lat_r = lat * math.pi / 180.0
    s = math.sin(lat_r)
    N = _A / math.sqrt(1.0 - _SIN2 * (s * s))
    return ((N + alt) * math.cos(lat_r) * math.cos(lon_r), (N + alt) * math.cos(lat_r) * math.sin(lon_r), (_COS2 * N + alt) * s)


def enu(points, origin_point, lat: float, lon: float):
    """Geocentric_WGS84ToENU_WGS84 of points [k, 3] (float64, element-wise IEEE operations) around origin_point at (lat, lon)."""
    clat, slat = math.cos(lat * math.pi / 180.0), math.sin(lat * math.pi / 180.0)
    clon, slon = math.cos(lon * math.pi / 180.0), math.sin(lon * math.pi / 180.0)
    p = np.asarray(points, np.float64).reshape(-1, 3)
    rx, ry, rz = p[:, 0] - origin_point[0], p[:, 1] - origin_point[1], p[:, 2] - origin_point[2]
    x = -slon * rx + clon * ry
    y = -clon * slat * rx - slon * slat * ry + clat * rz
    z = clon * clat * rx + slon * clat * ry + slat * rz
    return np.stack([x, y, z], 1)


class GpsMap:
    """The GPS of a map's real places (rows of (stamp, longitude, latitude, altitude, error)) and their offsetENU x, y, z (float32),
    with every place's geocentric point computed once, as _gpsGeocentricCache holds it."""

    def __init__(self, gps, offsets=None):
        self.gps = np.asarray(gps, np.float64).reshape(-1, 5)
        n = len(self.gps)
        self.offsets = np.zeros((n, 3), np.float32) if offsets is None else np.asarray(offsets, np.float32).reshape(n, 3)
        self.fix = self.gps[:, 0] > 0
        self.geo = np.zeros((n, 3), np.float64)
        for i in np.nonzero(self.fix)[0]:
            _, lon, lat, alt, _ = self.gps[i]
            self.geo[i] = geocentric(lat, lon, alt)


def gate(gmap: GpsMap, frame_gps, local_radius: float) -> np.ndarray:
    """Rtabmap.cpp:2046-2115 for one frame that computes: which real places are compared (bool [n]).  frame_gps: (stamp, longitude,
    latitude, altitude, error); local_radius: RGBD/LocalRadius (a float)."""
    stamp, lon, lat, alt, error = (float(v) for v in frame_gps)
    n = len(gmap.gps)
    if not stamp > 0.0:
        return np.ones(n, bool)
    origin = geocentric(lat, lon, alt)
    rel = enu(gmap.geo, origin, lat, lon)
    # relativePose += offsetENU - originOffsetENU: a float difference (the origin's offset is the identity), added to a double
    off = (gmap.offsets - f32(0)).astype(np.float32).astype(np.float64)
    x, y, z = rel[:, 0] + off[:, 0], rel[:, 1] + off[:, 1], rel[:, 2] + off[:, 2]
    z = np.where(z > error, z - error, np.where(z < -error, z + error, 0.0))
    r = f32(local_radius)
    accept = (x * x + y * y) + z * z < float(f32(r * r))
    return np.where(gmap.fix, accept, True)


def sparse_columns(bf, ids, neighbors, stm=()):
    """BayesFilterOracle.sparse_columns with normalize's renormalisation test made in double, as BayesFilter.cpp:469 makes it
    (`addedProbabilitiesSum < maxNorm - 0.0001`: a float against a double).  Under NumPy 2's promotion rules bayes_py compares the float32 sums with the
    bound rounded to float32, which decides differently when a column's sum falls between the two; a cut place list (a few hundred
    places, Bayes/PredictionLC with a uniform fill) reaches such sums."""
    f = np.float32
    n = len(ids)
    first = 1 if ids[0] < 0 else 0
    col_ptr, rows, levels = prediction_columns(ids, neighbors, stm)
    vals = np.array([f(v) for v in bf.lc], np.float32)[levels + 1]
    counts = np.diff(col_ptr)
    real = np.array([i > 0 for i in ids])
    s = np.zeros(n, np.float32)
    for k in range(int(counts.max(initial=0))):
        c = np.nonzero(counts > k)[0]
        s[c] = (s[c] + vals[col_ptr[c] + k]).astype(np.float32)
    entry_col = np.repeat(np.arange(n), counts)
    diag = np.nonzero(rows == entry_col)[0]
    lc0 = bf.lc[0]
    need = s.astype(np.float64) < float(bf.total) - lc0
    delta = np.zeros(n, np.float32)
    delta[need] = (float(bf.total) - lc0 - s[need].astype(np.float64)).astype(np.float32)
    dcol = entry_col[diag]
    vals[diag] = np.where(need[dcol], (vals[diag] + delta[dcol]).astype(np.float32), vals[diag])
    s = np.where(need, (s + delta).astype(np.float32), s)
    other = f(f(1.0) - bf.total) if bf.total < 1 else f(0)
    value = f(0)
    if other > 0 and n > 1:
        value = f(other / f(n - 1))
        nonzero = np.bincount(entry_col[(vals != 0) & (rows >= first)], minlength=n)
        s = _repeated_float_add(s, value, np.where(real, (n - first) - nonzero, 0))
    max_norm = f(1 - (lc0 if first else 0))
    s64 = s.astype(np.float64)
    renorm = real & ((s64 < float(max_norm) - 0.0001) | (s64 > float(max_norm) + 0.0001))
    scale = np.where(renorm, (max_norm / np.where(renorm, s, f(1))).astype(np.float32), f(1)).astype(np.float32)
    u = np.where(real, value, f(0)).astype(np.float32)
    vals = np.where(vals == 0, u[entry_col], vals)
    scaled_u = (u * scale).astype(np.float32)
    u = np.where(renorm, np.where(scaled_u < bf.eps, f(0), scaled_u), u).astype(np.float32)
    sv = (vals * scale[entry_col]).astype(np.float32)
    vals = np.where(renorm[entry_col], np.where(sv < bf.eps, f(0), sv), vals).astype(np.float32)
    return col_ptr, rows, vals, u


class GpsClient:
    """One localisation client deciding over GPS-filtered place lists: the sparse restatement of its Bayes filter (bayes_py), optionally
    the reference's compiled BayesFilter.cpp, and the restated decision on each."""

    def __init__(self, sparse, decide: dc.DecideClient, ref=None, decide_ref: dc.DecideClient | None = None):
        self.sparse, self.decide, self.ref, self.decide_ref = sparse, decide, ref, decide_ref

    @staticmethod
    def adjusted(raw_row, compared, virtual_place_ratio=0):
        """adjustLikelihood over the virtual place and the compared places (in id order): [1 + compared count]."""
        lik = np.concatenate([[f32(0)], np.asarray(raw_row, np.float32)[compared]]).astype(np.float32)
        return orc.adjust_likelihood(lik, virtual_place_ratio)

    def posterior(self, ids, adj, tables, stm=()):
        """(sparse restatement, reference or None) of computePosterior over ids (the virtual place and the compared places)."""
        cols = sparse_columns(self.sparse, ids, tables.__getitem__, stm)
        ps = self.sparse._update(ids, adj, lambda last: self.sparse._prior(ids, last, *cols))
        pr = None
        if self.ref is not None:
            self.ref.set_graph(tables, stm)
            pr = self.ref.compute_posterior(ids, adj)
        return ps, pr
