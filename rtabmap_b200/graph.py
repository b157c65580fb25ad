"""The two graph walks of rtabmap::Memory a localisation map needs, on the host, for the tables of lcd_clients_set_map and
lcd_clients_set_map_gps.  They run once per map, not per frame.

  bayes_neighbors    Memory::getNeighborsId (Memory.cpp:1703-1870) as BayesFilter::generatePrediction calls it (BayesFilter.cpp:329):
                     getNeighborsId(id, len(PredictionLC) - 1, 0, false, false, true, true).  Neighbour links (kNeighbor,
                     kNeighborMerged) step one margin out; loop-closure links keep the margin (incrementMarginOnLoop = false);
                     local-space closures are not followed (ignoreLocalSpaceLoopIds); only places of the working memory are reached
                     (maxCheckedInDatabase = 0).  Margins 0 .. depth - 1.
  prediction_tables  generatePrediction's columns (BayesFilter.cpp:329-391) in the CSR form of lcd_clients_set_map: places in id order, a
                     place and the places at its margin 0 (merged through loop closures) share the table of whichever comes first.
  gps_of_places      Memory::getGPS(id, gps, offsetENU, false, maxGraphDepth) (Memory.cpp:4507-4553): a place without a fix takes the
                     fix of the nearest place that has one (getNeighborsId with every link one margin, the nearest margin first, then
                     ascending id), and the offset of its pose from that place through graph::computePath (Graph.cpp:1997-2160).

The graph is the caller's: the place-to-place links of the Link table (dbio.read_links), as each place stores them (from_id = the
place).  Landmark links are not read, so places that observe the same landmark are not joined at margin 0 as the reference's landmark
index joins them (Memory.cpp:1850-1885).  Intermediate nodes (weight -1) are not supported: dbio refuses maps that hold them.
"""
from __future__ import annotations

import heapq
from collections import deque

import numpy as np

# Link::Type (Link.h:41-52, DatabaseSchema.sql.in:57)
NEIGHBOR, GLOBAL_CLOSURE, LOCAL_SPACE_CLOSURE, LOCAL_TIME_CLOSURE, USER_CLOSURE, VIRTUAL_CLOSURE, NEIGHBOR_MERGED, POSE_PRIOR, LANDMARK, \
    GRAVITY = range(10)
NEIGHBOR_TYPES = (NEIGHBOR, NEIGHBOR_MERGED)

# Bayes/PredictionLC's default (Parameters.h:363), each value through a float as setPredictionLC reads it (BayesFilter.cpp:70-101)
DEFAULT_PREDICTION_LC = [float(np.float32(v)) for v in (0.1, 0.36, 0.30, 0.16, 0.062, 0.0151, 0.00255, 0.000324, 2.5e-05, 1.3e-06, 4.8e-08,
                                                         1.2e-09, 1.9e-11, 2.2e-13, 1.7e-15, 8.5e-18, 2.9e-20, 6.9e-23)]


def _adjacency(places, from_id, to_id, link_type):
    """{place: [(to, type), ...]} in stored order (from_id, to_id ascending), for links whose from_id is a place; self links dropped."""
    adj = {int(p): [] for p in places}
    for a, b, t in zip(np.asarray(from_id).tolist(), np.asarray(to_id).tolist(), np.asarray(link_type).tolist()):
        if a != b and a in adj:
            adj[a].append((b, t))
    return adj


def bayes_neighbors(places, links, depth: int) -> dict:
    """{place: {neighbour: margin}} of every place, as generatePrediction's call of getNeighborsId returns it.  `links`: an object with
    from_id, to_id and type arrays (dbio.Links); `depth` = len(PredictionLC) - 1."""
    adj = _adjacency(places, links.from_id, links.to_id, links.type)
    step = {}
    for p, out in adj.items():
        # margin step of each followed link: 1 for neighbour links, 0 for loop closures, not followed for local-space closures
        step[p] = [(b, 1 if t in NEIGHBOR_TYPES else 0) for b, t in out if b in adj and t != LOCAL_SPACE_CLOSURE]
    return {p: _walk01(p, step, depth) for p in adj}


def _walk01(start: int, step: dict, depth: int) -> dict:
    """Breadth-first by margin, each margin closed over its 0-steps before the next one starts: the margin of a place is the least
    number of neighbour links on a path to it; places at margin >= depth are not reached."""
    out = {}
    if depth <= 0:
        return out
    cur = deque([start])
    m = 0
    while cur and m < depth:
        nxt = []
        while cur:
            u = cur.popleft()
            if u in out:
                continue
            out[u] = m
            for v, w in step[u]:
                if v not in out:
                    (cur.append if w == 0 else nxt.append)(v)
        cur = deque(nxt)
        m += 1
    return out


def prediction_tables(places, neighbors: dict):
    """(ids, col_ptr, nbr_row, nbr_level) for lcd_clients_set_map: ids = [-1] + places ascending (the virtual place first), and each
    place's column listing (row of the neighbour in ids, its margin) in ascending neighbour id; the virtual place's column is empty."""
    ids = [-1] + sorted(int(p) for p in places)
    index = {p: k for k, p in enumerate(ids) if p > 0}
    cols = {}
    for pid in ids[1:]:
        if index[pid] in cols:
            continue
        nb = sorted(neighbors[pid].items())
        entries = [(index[k], m) for k, m in nb if k in index]
        for k, m in nb:
            if m == 0 and k in index:
                cols[index[k]] = entries
    counts = np.array([len(cols.get(c, ())) for c in range(len(ids))], np.int64)
    col_ptr = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
    flat = [e for c in range(len(ids)) for e in cols.get(c, ())]
    rows = np.array([r for r, _ in flat], np.int32)
    levels = np.array([m for _, m in flat], np.int32)
    return np.array(ids, np.int32), col_ptr, rows, levels


def neighbor_links(places, links):
    """(nbr_ptr, nbr_ids) of lcd_clients_set_map_poses: each place's kNeighbor / kNeighborMerged links in stored order."""
    adj = _adjacency(places, links.from_id, links.to_id, links.type)
    lists = [[b for b, t in adj[int(p)] if t in NEIGHBOR_TYPES] for p in places]
    ptr = np.concatenate([[0], np.cumsum([len(x) for x in lists])]).astype(np.int64)
    return ptr, np.array([b for x in lists for b in x], np.int32)


# ---------------------------------------------------------------------------------------------------------- Memory::getGPS ------
def _yaw(R) -> np.float32:
    """Transform::theta: the yaw of pcl::getEulerAngles, atan2(r10, r00) in float."""
    return np.float32(np.arctan2(np.float32(R[1, 0]), np.float32(R[0, 0])))


def _rz(theta) -> np.ndarray:
    c, s = np.cos(np.float32(theta)), np.sin(np.float32(theta))
    return np.array([[c, -s, 0], [s, c, 0], [0, 0, 1]], np.float32)


def _compose(a: np.ndarray, b: np.ndarray) -> np.ndarray:
    """a * b of two 3x4 float transforms."""
    out = np.empty((3, 4), np.float32)
    out[:, :3] = a[:, :3] @ b[:, :3]
    out[:, 3] = a[:, :3] @ b[:, 3] + a[:, 3]
    return out


def compute_path(start: int, end: int, links_of: dict):
    """graph::computePath(start, end, memory, lookInDatabase=false) with its defaults (updateNewCosts = false, distance costs): the
    pose of `end` relative to `start` along the path, or None when no path joins them.  A place keeps the pose and cost of the link
    that first reached it; places come off the queue by least cost so far, in float.  Equal costs come off in the order they were
    reached (std::priority_queue leaves that order to its heap)."""
    nodes = {start: (np.float32(0), np.eye(3, 4, dtype=np.float32))}
    pq = [(np.float32(0), 0, start)]
    seq = 1
    while pq:
        _, _, u = heapq.heappop(pq)
        if u == end:
            return nodes[u][1] if u != start else None   # a path of one node: path.size() < 2
        cost, pose = nodes[u]
        for v, T in links_of.get(u, ()):
            if v in nodes:
                continue
            t = T[:, 3]
            c = np.float32(cost + np.float32(np.sqrt(np.float32(t[0] * t[0] + t[1] * t[1] + t[2] * t[2]))))
            nodes[v] = (c, _compose(pose, T))
            heapq.heappush(pq, (c, seq, v))
            seq += 1
    return None


def gps_of_places(places, gps: np.ndarray, poses: np.ndarray, links, max_graph_depth: int = 0):
    """(gps [n, 6] float64, offset_enu [n, 3] float32) of every place: its own fix (stamp > 0) with a zero offset, else what
    Memory::getGPS finds for it, else no fix (zeros).  gps [n, 6]: (stamp, longitude, latitude, altitude, error, bearing) from Node.gps;
    poses [n, 3, 4]: the places' Node.pose (Signature::getPose); links: every place-to-place link with its transform."""
    places = [int(p) for p in places]
    row = {p: k for k, p in enumerate(places)}
    gps = np.asarray(gps, np.float64).reshape(len(places), 6)
    poses = np.asarray(poses, np.float32).reshape(len(places), 3, 4)
    has_fix = gps[:, 0] > 0.0
    out_gps = np.where(has_fix[:, None], gps, 0.0)
    out_off = np.zeros((len(places), 3), np.float32)
    if has_fix.all() or not has_fix.any():
        return out_gps, out_off
    links_of = {p: [] for p in places}
    adj = {p: [] for p in places}
    for a, b, T in zip(np.asarray(links.from_id).tolist(), np.asarray(links.to_id).tolist(), np.asarray(links.transform, np.float32)):
        if a != b and a in links_of:
            links_of[a].append((b, T))
            if b in row:
                adj[a].append(b)
    for k, p in enumerate(places):
        if has_fix[k]:
            continue
        # getNeighborsId(p, maxGraphDepth, 0, true, false, true): every link one margin out; candidates by margin, then by id
        seen = {p}
        level = [p]
        m = 0
        found = False
        while level and (max_graph_depth == 0 or m < max_graph_depth) and not found:
            for s in sorted(level):
                if has_fix[row[s]]:
                    rel = compute_path(s, p, links_of)
                    if rel is not None:
                        g = gps[row[s]]
                        R_s = poses[row[s], :, :3]
                        theta = np.float32(np.float32((-(g[5] - 90.0)) * np.pi / 180.0) - _yaw(R_s))
                        out_gps[k] = g
                        out_off[k] = _rz(theta) @ (R_s @ rel[:, 3])
                        found = True
                        break
            nxt = set()
            for u in level:
                for v in adj[u]:
                    if v not in seen:
                        seen.add(v)
                        nxt.add(v)
            level = list(nxt)
            m += 1
    return out_gps, out_off
