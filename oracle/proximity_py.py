"""CPU oracle of proximity detection by space in localisation mode — TEST INFRASTRUCTURE ONLY (tests/).

Restates, for one frame, the candidate search of Rtabmap::process (corelib/src/Rtabmap.cpp:2698-2934) and its effect on the global
hypothesis (:2894-2911, :3133-3196), in float32 where the reference computes in float:
  Graph.cpp:2239-2325    graph::findNearestNodes: squared distances summed x, y, z; rtflann's radius result sets keep dist < radius^2;
                         the angle filter compares pcl::getAngle3D of the two x axes (acos of the clamped dot product of the normalised
                         Eigen::Vector4f, w = 0) with the angle.  graph::findNearestNode (k = 1): the smallest squared distance; ties
                         go to the lowest id here (the reference's kd-tree order is not a function of the ids).
  Rtabmap.cpp:5303-5382  Rtabmap::getPaths with Memory::getNeighborsId (Memory.cpp:1703-1870: margins 0 .. maxGraphDepth-1 through
                         neighbour links, only through the candidates) and the ascending-id admission of the reached places.
  Rtabmap.cpp:1147-1176, :2796-2816   NearestPathKey; the distance is (currentPoseInv * pose).getNormSquared().
  Rtabmap.cpp:2822-2934  the walk in descending key order, the filtering radius capped by RGBD/MaxLoopClosureDistance, attempts
                         counted up to RGBD/ProximityMaxPaths.
Transforms are float 3x4 arrays; inverses are [R^T | -R^T t] (the reference's Eigen 4x4 inverse is not pinned to the last bit).
apply() takes the registrations' outcome (ok and the transform of each attempt) from outside; the GPU tests compare the registrations
with lcd_verify_batch of the same (place, frame) pairs.
"""
from __future__ import annotations

import math

import numpy as np

f32 = np.float32
PROXIMITY_SUPPRESSED = 12
LINK_LOCAL_SPACE, LINK_GLOBAL = 1, 2


def d2(a, b) -> np.float32:
    """squared distance of the positions of two poses [3, 4], x + y then + z"""
    dx, dy, dz = f32(a[0, 3]) - f32(b[0, 3]), f32(a[1, 3]) - f32(b[1, 3]), f32(a[2, 3]) - f32(b[2, 3])
    return f32(f32(dx * dx) + f32(dy * dy)) + f32(dz * dz)


def rel_norm2(a, b=None) -> np.float32:
    """(a^-1 * b).getNormSquared() (b = None: a^-1's own translation)"""
    v = []
    for i in range(3):
        ti = f32(f32(f32(a[0, i]) * f32(a[0, 3])) + f32(f32(a[1, i]) * f32(a[1, 3]))) + f32(f32(a[2, i]) * f32(a[2, 3]))
        bi = f32(0) if b is None else f32(f32(f32(a[0, i]) * f32(b[0, 3])) + f32(f32(a[1, i]) * f32(b[1, 3]))) + f32(f32(a[2, i]) * f32(b[2, 3]))
        v.append(f32(bi - ti))
    return f32(f32(v[0] * v[0]) + f32(v[1] * v[1])) + f32(v[2] * v[2])


def angle_rad(degrees) -> np.float32:
    """_proximityAngle *= M_PI/180.0f (Rtabmap.cpp:609-612), stored as a float"""
    return f32(float(f32(degrees)) * (math.pi / 180.0))


def angle_ok(a, b, angle) -> bool:
    angle = f32(angle)
    if not angle > 0:
        return True

    def unit(p):
        x, y, z = f32(p[0, 0]), f32(p[1, 0]), f32(p[2, 0])
        n = f32(math.sqrt(f32(f32(x * x) + f32(z * z)) + f32(y * y)))
        return f32(x / n), f32(y / n), f32(z / n)

    (ax, ay, az), (bx, by, bz) = unit(a), unit(b)
    rad = float(f32(f32(f32(ax * bx) + f32(az * bz)) + f32(ay * by)))
    rad = min(1.0, max(-1.0, rad))
    return math.acos(rad) <= float(angle)


def find_nearest_nodes(target, poses: dict, radius) -> dict:
    """graph::findNearestNodes(target, poses, radius): id -> squared distance, ids >= 1"""
    r2 = f32(f32(radius) * f32(radius))
    ids = np.array(sorted(poses), np.int64)
    if not len(ids):
        return {}
    t = np.stack([poses[int(i)][:, 3] for i in ids]).astype(np.float32)  # element-wise float32: the same roundings as d2()
    dx, dy, dz = f32(target[0, 3]) - t[:, 0], f32(target[1, 3]) - t[:, 1], f32(target[2, 3]) - t[:, 2]
    d = (dx * dx + dy * dy) + dz * dz
    return {int(i): f32(v) for i, v in zip(ids, d) if i >= 1 and v < r2}


def nearest_node(ids, dist: dict) -> int:
    best = 0
    for i in sorted(ids):
        if best == 0 or dist[i] < dist[best]:
            best = i
    return best


def neighbors_id(start: int, max_depth: int, links: dict, nodes: set) -> set:
    """Memory::getNeighborsId(start, max_depth, 0, true, true, true, true, nodes): the places reached through neighbour links in margins
    0 .. max_depth-1 (all with max_depth 0), never stepping through a place outside `nodes`"""
    ids, margin, m = set(), {start}, 0
    while (max_depth == 0 or m < max_depth) and margin:
        nxt = set()
        for i in sorted(margin, reverse=True):
            if i in ids or i not in nodes:
                continue
            ids.add(i)
            for j in links.get(i, ()):
                if j not in ids:
                    nxt.add(j)
        margin, m = nxt, m + 1
    return ids


def get_paths(nearest: dict, links: dict, max_depth: int, stats: dict | None = None) -> dict:
    """Rtabmap::getPaths: nearest id -> the path's ids (ascending).  stats (optional) counts the branches taken: "rejected" reached places
    left for a later path by the ascending-id admission, "lost" paths dropped because their start already had one, "longest" path."""
    stats = {} if stats is None else stats
    for k in ("rejected", "lost", "longest"):
        stats.setdefault(k, 0)
    nodes = set(nearest)
    left = set(nearest)
    paths = {}
    while left:
        start = nearest_node(left, nearest)
        path = []
        for i in sorted(neighbors_id(start, max_depth, links, nodes)):
            if i not in left:
                continue
            if not path or any(j in path for j in links.get(i, ())):
                path.append(i)
                left.discard(i)
            else:
                stats["rejected"] += 1
        if start in paths:
            stats["lost"] += 1
        paths.setdefault(start, path)  # std::map::insert keeps the first path of a start
        stats["longest"] = max(stats["longest"], len(paths[start]))
    return paths


def path_key(path, likelihood: dict, current, poses):
    """NearestPathKey (likelihood, id, distance) of one path (:2800-2815)"""
    hl, hid, sd = f32(0), path[0], f32(-1)
    for i in path:
        v = f32(likelihood.get(i, 0.0))
        d = rel_norm2(current, poses[i])
        if v > hl or (v == hl and (sd < 0 or d < sd)):
            hl, hid, sd = v, i, d
    return hl, hid, sd


def key_sort(k):
    """descending NearestPathKey order: likelihood descending, then distance ascending, then id descending"""
    return (-float(k[0]), float(k[2]), -k[1])


def filtering_radius(path_filtering_radius, max_loop_closure_distance) -> np.float32:
    fr, mld = f32(path_filtering_radius), f32(max_loop_closure_distance)
    if mld > 0 and (fr <= 0 or mld < fr):
        fr = mld
    return fr


def detect(current, poses: dict, links: dict, likelihood: dict, local_radius=10.0, angle=45.0, max_paths=3, max_graph_depth=50,
           path_filtering_radius=1.0, max_loop_closure_distance=0.0, stats: dict | None = None):
    """Steps 1-4 for one frame (stats: see get_paths).  poses: id -> float32 [3, 4]; links: id -> neighbour ids; likelihood: id -> adjusted likelihood.
    Returns (nearest ids -> d2, paths, attempts [((likelihood, id, distance), candidate id)])."""
    nearest = find_nearest_nodes(current, poses, local_radius)
    paths = get_paths(nearest, links, max_graph_depth, stats)
    keys = sorted((path_key(p, likelihood, current, poses) + (p,) for p in paths.values()), key=key_sort)
    angle = angle_rad(angle)
    r2 = f32(f32(local_radius) * f32(local_radius))
    fr = filtering_radius(path_filtering_radius, max_loop_closure_distance)
    attempts = []
    for kl, kid, kd, path in keys:
        if max_paths > 0 and len(attempts) >= max_paths:
            break
        kept = [i for i in path if nearest[i] < r2 and angle_ok(current, poses[i], angle)]
        cand = kid if (kl > 0 and kid in kept) else nearest_node(kept, nearest)
        if cand > 0 and (fr <= 0 or nearest[cand] < f32(fr * fr)):
            attempts.append(((kl, kid, kd), cand))
    return nearest, paths, attempts


def apply(nearest: dict, attempts, results, loop_id: int, status: int, path_filtering_radius=1.0, max_loop_closure_distance=0.0):
    """The registrations' outcome and the suppression of the global hypothesis.  results: one (ok, transform [3, 4]) per attempt.
    Returns (accepted flags, link types, suppressed id, loop_id, status, global verification skipped)."""
    fr = filtering_radius(path_filtering_radius, max_loop_closure_distance)
    accepted, types, suppressed = [], [], 0
    for (_, cand), (ok, T) in zip(attempts, results):
        acc = bool(ok) and (fr <= 0 or rel_norm2(np.asarray(T, np.float32)) <= f32(fr * fr))
        accepted.append(acc)
        t = LINK_LOCAL_SPACE if acc else 0
        if acc and loop_id > 0 and loop_id in nearest:
            if cand == loop_id:
                t, suppressed = LINK_GLOBAL, cand
            elif suppressed == 0:
                suppressed = cand
        types.append(t)
    skip = False
    if loop_id > 0 and suppressed:
        skip = True
        if suppressed != loop_id:
            loop_id, status = 0, PROXIMITY_SUPPRESSED
    return accepted, types, suppressed, loop_id, status, skip
