"""Inputs shared by the GPS filter tests (tests/test_oracle_gps.py on the CPU, tests/test_gpu_decide_gps.py on the GPU): places and
frames with GPS fixes along a trajectory, and hand cases at the edges of Rtabmap.cpp:2046-2115."""
import math

import numpy as np

LAT0, LON0 = 46.78, -71.27          # an origin for the synthetic trajectories
M_PER_DEG_LAT = 111320.0


def to_geodetic(east, north, up=0.0, lat0=LAT0, lon0=LON0):
    """(latitude, longitude, altitude) a local east / north / up offset in metres away from (lat0, lon0), on a sphere (inputs only)."""
    lat = lat0 + north / M_PER_DEG_LAT
    lon = lon0 + east / (M_PER_DEG_LAT * math.cos(math.radians(lat0)))
    return lat, lon, up


def gps_row(east, north, up=0.0, error=0.0, stamp=1.0):
    lat, lon, alt = to_geodetic(east, north, up)
    return (stamp, lon, lat, alt, error)


def trajectory_gps(n, rng, spacing=4.0, no_fix=0.0, offsets=0.0):
    """GPS rows [n, 5] of places along a wandering path with `spacing` metres between places, a share `no_fix` of places without a fix,
    and offsetENU [n, 3] float32 (a share `offsets` of places with a non-zero one); and the places' (east, north) positions."""
    heading = np.cumsum(rng.normal(0, 0.15, n))
    e = np.cumsum(spacing * np.cos(heading))
    nn = np.cumsum(spacing * np.sin(heading))
    up = rng.normal(0, 3.0, n)
    gps = np.array([gps_row(e[i], nn[i], up[i], stamp=1000.0 + i) for i in range(n)], np.float64)
    gps[rng.random(n) < no_fix, 0] = 0.0
    off = np.zeros((n, 3), np.float32)
    k = rng.random(n) < offsets
    off[k] = rng.normal(0, 2.0, (int(k.sum()), 3)).astype(np.float32)
    return gps, off, np.stack([e, nn], 1)


def frame_gps_near(pos, rng, error=(0.0, 2.0, 10.0)):
    """A fix a few metres from position pos (east, north), with one of the given errors."""
    return gps_row(pos[0] + rng.normal(0, 3), pos[1] + rng.normal(0, 3), rng.normal(0, 3), error=error[int(rng.integers(len(error)))],
                   stamp=5000.0 + rng.random())


def hand_cases():
    """(place gps [n, 5], offsets [n, 3], frame gps, radius, expected compared [n]) at the edges of the gate.  Every place sits on the
    frame's own fix, so its ENU position is exactly 0 and the offset alone sets the distance."""
    frame = gps_row(0.0, 0.0, 0.0, error=5.0)
    below, above = np.nextafter(np.float32(10), np.float32(0)), np.nextafter(np.float32(10), np.float32(20))
    rows = [  # (offset, has fix, compared at radius 10 with error 5)
        ((below, 0, 0), True, True),        # one ulp inside the radius
        ((10, 0, 0), True, False),          # on the radius: the test is strict
        ((above, 0, 0), True, False),       # one ulp outside
        ((0, below, 0), True, True),
        ((0, 0, 4.9), True, True),          # height inside the error band: ignored
        ((0, 0, -5.0), True, True),         # on the band's edge: ignored
        ((0, 0, 15.0), True, False),        # 15 - 5 = 10: on the radius
        ((0, 0, 14.9), True, True),         # 9.9 < 10
        ((0, 0, -15.5), True, False),       # -15.5 + 5 = -10.5
        ((9, 0, 5.0 + 4.4), True, False),   # 81 + 4.4^2 > 100
        ((6, 0, 5.0 + 7.9), True, True),    # 36 + 62.41 < 100
        ((500, 500, 500), False, True),     # no fix: always compared
    ]
    gps = np.array([frame if fix else (0.0,) + frame[1:] for _, fix, _ in rows], np.float64)
    off = np.array([o for o, _, _ in rows], np.float32)
    want = np.array([w for _, _, w in rows], bool)
    return gps, off, frame, 10.0, want
