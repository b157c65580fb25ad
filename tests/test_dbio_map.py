"""Opening a localisation map from an RTAB-Map database, the part that needs no GPU: the readers of rtabmap_b200/dbio.py on databases
with the reference's table layout (corelib/src/resources/DatabaseSchema.sql.in), compressData2 / uncompressData, the two graph walks
of rtabmap_b200/graph.py against oracle/bayes_py.py and a restatement of Memory::getGPS, and every refusal of open_localization_map,
which must leave the engine untouched."""
import sqlite3
import struct
import zlib

import numpy as np
import pytest

from bayes_cases import PATTERNS, likelihood, n_levels, with_vp
from oracle.bayes_py import BayesFilterOracle, graph_tables, parse_prediction_lc, prediction_columns
from rtabmap_b200 import LcdError, dbio, graph

# the tables of the reference schema the loader reads, column for column (names and order are the format)
SCHEMA = """
CREATE TABLE Node (id INTEGER NOT NULL, map_id INTEGER NOT NULL, weight INTEGER, stamp FLOAT, pose BLOB, ground_truth_pose BLOB,
                   velocity BLOB, label TEXT, gps BLOB, env_sensors BLOB, time_enter DATE, PRIMARY KEY (id));
CREATE TABLE Link (from_id INTEGER NOT NULL, to_id INTEGER NOT NULL, type INTEGER NOT NULL, information_matrix BLOB NOT NULL,
                   transform BLOB, user_data BLOB);
CREATE TABLE Word (id INTEGER NOT NULL, descriptor_size INTEGER NOT NULL, descriptor BLOB NOT NULL, time_enter DATE, PRIMARY KEY (id));
CREATE TABLE Feature (node_id INTEGER NOT NULL, word_id INTEGER NOT NULL, pos_x FLOAT NOT NULL, pos_y FLOAT NOT NULL, size INTEGER NOT NULL,
                      dir FLOAT NOT NULL, response FLOAT NOT NULL, octave INTEGER NOT NULL, depth_x FLOAT, depth_y FLOAT, depth_z FLOAT,
                      descriptor_size INTEGER, descriptor BLOB);
CREATE TABLE GlobalDescriptor (node_id INTEGER NOT NULL, type INTEGER NOT NULL, info BLOB, data BLOB NOT NULL);
CREATE TABLE Admin (version TEXT, preview_image BLOB, opt_cloud BLOB, opt_ids BLOB, opt_poses BLOB, opt_last_localization BLOB,
                    opt_polygons_size INTEGER, opt_polygons BLOB, opt_tex_coords BLOB, opt_tex_materials BLOB, opt_map BLOB,
                    opt_map_x_min FLOAT, opt_map_y_min FLOAT, opt_map_resolution FLOAT, time_enter DATE);
CREATE UNIQUE INDEX IDX_Node_id on Node (id);
CREATE INDEX IDX_Feature_node_id on Feature (node_id);
CREATE INDEX IDX_GlobalDescriptor_node_id on GlobalDescriptor (node_id);
CREATE INDEX IDX_Link_from_id on Link (from_id);
"""
INFO = np.eye(6).tobytes()


def yaw_pose(x, y, yaw):
    c, s = np.cos(yaw), np.sin(yaw)
    return np.array([[c, -s, 0, x], [s, c, 0, y], [0, 0, 1, 0]], np.float32)


def relative(a, b):
    """inv(a) * b of two 3x4 poses: the transform a link from a to b stores"""
    R = a[:, :3].T.astype(np.float64)
    out = np.empty((3, 4), np.float32)
    out[:, :3] = R @ b[:, :3]
    out[:, 3] = R @ (b[:, 3].astype(np.float64) - a[:, 3])
    return out


def make_map_db(path, word_ids, vocab, nodes, features, links=(), opt=None, gps=None, gdesc=None, version="0.21.0", weights=None,
                poses=None):
    """nodes: ids; features: rows (node, word, x, y, depth (x, y, z) or None, descriptor bytes) inserted in the order given; links:
    (from, to, type[, transform 3x4]); opt: (ids, poses [n, 3, 4]); gps: {node: 6 doubles}; gdesc: rows (node, type, matrix)."""
    con = sqlite3.connect(path)
    con.executescript(SCHEMA)
    con.execute("INSERT INTO Admin(version, opt_ids, opt_poses) VALUES(?,?,?);",
                (version, None if opt is None else dbio.compress_data(np.asarray(opt[0], np.int32).reshape(1, -1)),
                 None if opt is None else dbio.compress_data(np.asarray(opt[1], np.float32).reshape(1, -1))))
    weights = weights or {}
    poses = poses if poses is not None else {}
    con.executemany("INSERT INTO Node(id, map_id, weight, stamp, pose, gps) VALUES(?,?,?,?,?,?);",
                    [(int(n), int(n) % 2, int(weights.get(int(n), 1)), float(n),
                      np.asarray(poses.get(int(n), np.eye(3, 4)), np.float32).tobytes(),
                      None if gps is None or int(n) not in gps else np.asarray(gps[int(n)], np.float64).tobytes()) for n in nodes])
    con.executemany("INSERT INTO Word(id, descriptor_size, descriptor) VALUES(?,?,?);",
                    [(int(i), vocab.shape[1], vocab[k].tobytes()) for k, i in enumerate(word_ids)])
    con.executemany("INSERT INTO Feature(node_id, word_id, pos_x, pos_y, size, dir, response, octave, depth_x, depth_y, depth_z, descriptor_size,"
                    " descriptor) VALUES(?,?,?,?,31,0,0,0,?,?,?,?,?);",
                    [(int(n), int(w), float(x), float(y), *((None,) * 3 if d is None else tuple(float(v) for v in d)),
                      len(b) // (4 if vocab.dtype == np.float32 else 1), b) for n, w, x, y, d, b in features])
    con.executemany("INSERT INTO Link(from_id, to_id, type, information_matrix, transform) VALUES(?,?,?,?,?);",
                    [(int(l[0]), int(l[1]), int(l[2]), INFO, np.asarray(l[3] if len(l) > 3 else np.eye(3, 4), np.float32).tobytes()) for l in links])
    for n, t, m in gdesc or ():
        con.execute("INSERT INTO GlobalDescriptor(node_id, type, data) VALUES(?,?,?);", (int(n), int(t), dbio.compress_data(m)))
    con.commit()
    con.close()


class RecordingEngine:
    """The Engine calls the loader makes, recorded (CPU tests); the store's row limit as lcd_sig_add_batch enforces it."""

    def __init__(self, desc_type=0, desc_dim=32):
        self.desc_type, self.desc_dim, self.calls = desc_type, desc_dim, []
        self.last_word_id = 0

    def gdesc_dim(self):
        return 0

    def __getattr__(self, name):
        def call(*args):
            if name == "sig_add_batch" and np.asarray(args[1]).shape[1] > 4096:
                raise LcdError(-3, "at most 4096 features per signature")
            self.calls.append((name, args))
        return call


def small_map(rng, dtype=np.uint8, n_nodes=6, per_node=(5, 40)):
    width = 32 if dtype == np.uint8 else 64
    W = 120
    vocab = rng.integers(0, 256, (W, width)).astype(np.uint8) if dtype == np.uint8 else rng.normal(size=(W, width)).astype(np.float32)
    word_ids = np.arange(1, W + 1, dtype=np.int32)
    nodes = list(range(1, n_nodes + 1))
    feats = []
    for n in nodes:
        for _ in range(int(rng.integers(*per_node))):
            w = int(rng.integers(1, W + 1)) if rng.random() > 0.1 else -1
            d = None if rng.random() < 0.15 else rng.normal(size=3)
            desc = (rng.integers(0, 256, width).astype(np.uint8) if dtype == np.uint8 else rng.normal(size=width).astype(np.float32)).tobytes()
            feats.append((n, w, rng.uniform(0, 640), rng.uniform(0, 480), d, desc))
    order = rng.permutation(len(feats))           # rows of all nodes interleaved, in any order
    return vocab, word_ids, nodes, [feats[k] for k in order]


@pytest.mark.parametrize("dtype", [np.uint8, np.float32])
def test_readers_return_what_was_written(tmp_path, dtype):
    rng = np.random.default_rng(5)
    vocab, word_ids, nodes, feats = small_map(rng, dtype)
    poses = {n: yaw_pose(n * 1.0, 0.5 * n, 0.1 * n) for n in nodes}
    links = [(a, a + 1, graph.NEIGHBOR, relative(poses[a], poses[a + 1])) for a in nodes[:-1]]
    links += [(a + 1, a, graph.NEIGHBOR, relative(poses[a + 1], poses[a])) for a in nodes[:-1]]
    links += [(1, 5, graph.GLOBAL_CLOSURE), (5, 1, graph.GLOBAL_CLOSURE), (2, 4, graph.LOCAL_SPACE_CLOSURE), (3, 6, graph.NEIGHBOR_MERGED)]
    links += [(2, -7, graph.LANDMARK), (3, 3, graph.POSE_PRIOR), (4, 4, graph.GRAVITY)]          # not place-to-place: dropped
    opt_ids = np.array(nodes[::-1], np.int32)
    opt_poses = np.stack([poses[n] for n in opt_ids])
    gps = {1: (10.0, -73.6, 45.5, 30.0, 4.0, 90.0), 4: (12.0, -73.61, 45.51, 31.0, 2.5, 180.0)}
    g = rng.normal(size=(len(nodes), 16)).astype(np.float32)
    db = str(tmp_path / "map.db")
    make_map_db(db, word_ids, vocab, nodes, feats, links, (opt_ids, opt_poses), gps, [(n, 1, g[k:k + 1]) for k, n in enumerate(nodes)],
                poses=poses)

    sig = dbio.read_signatures(db)
    assert list(sig.ids) == nodes and list(sig.map_id) == [n % 2 for n in nodes] and list(sig.weight) == [1] * len(nodes)
    width = vocab.shape[1]
    for k, n in enumerate(nodes):
        # the reference's row order: ascending word id; rows of one word in the order SQLite keeps them (the order they were written)
        mine = sorted([f for f in feats if f[0] == n], key=lambda f: f[1])
        c = int(sig.count[k])
        assert c == len(mine)
        assert list(sig.word_ids[k, :c]) == [f[1] for f in mine]
        assert np.array_equal(sig.uv[k, :c], np.array([[f[2], f[3]] for f in mine], np.float32))
        want_xyz = np.array([[np.nan] * 3 if f[4] is None else f[4] for f in mine], np.float32)
        assert np.array_equal(sig.xyz[k, :c], want_xyz, equal_nan=True)
        assert sig.descriptors.dtype == dtype and np.array_equal(sig.descriptors[k, :c], np.stack([np.frombuffer(f[5], dtype) for f in mine]))
        assert not sig.word_ids[k, c:].any() and np.isnan(sig.xyz[k, c:]).all()
    assert sig.descriptors.shape[2] == width and np.isnan(sig.xyz[sig.word_ids != 0]).any()
    sub = dbio.read_signatures(db, [4, 2])
    assert list(sub.ids) == [4, 2] and sub.count[0] == sig.count[3]

    ln = dbio.read_links(db)
    kept = sorted([l for l in links if l[1] > 0 and l[0] != l[1]], key=lambda l: (l[0], l[1]))
    assert [(a, b, t) for a, b, t in zip(ln.from_id.tolist(), ln.to_id.tolist(), ln.type.tolist())] == [l[:3] for l in kept]
    for k, l in enumerate(kept):
        assert np.array_equal(ln.transform[k], np.asarray(l[3] if len(l) > 3 else np.eye(3, 4), np.float32))

    ids, p = dbio.read_optimized_poses(db)
    assert np.array_equal(ids, opt_ids) and np.array_equal(p, opt_poses)
    ids, gp, pose = dbio.read_gps(db)
    assert list(ids) == nodes and np.array_equal(gp[0], gps[1]) and np.array_equal(gp[3], gps[4]) and not gp[[1, 2, 4, 5]].any()
    assert np.array_equal(pose, np.stack([poses[n] for n in nodes]))
    ids, gd = dbio.read_global_descriptors(db, [2, 3, 99])
    assert list(ids) == [2, 3] and np.array_equal(gd, g[1:3])


@pytest.mark.parametrize("m", [np.arange(-40, 60, dtype=np.int32).reshape(4, 25), np.random.default_rng(1).normal(size=(3, 7)).astype(np.float32),
                               np.arange(24, dtype=np.uint8).reshape(2, 4, 3), np.zeros((1, 0), np.float32)])
def test_compress_round_trip(m):
    back = dbio.uncompress_data(dbio.compress_data(m))
    assert back.dtype == m.dtype and back.shape == m.shape and np.array_equal(back, m)


def test_a_blob_laid_out_as_compressData2_decodes():
    """zlib's compress() of the bytes, then rows, cols and the OpenCV type as three native ints (Compression.cpp:239-266)"""
    m = np.random.default_rng(2).normal(size=(1, 36)).astype(np.float32)
    blob = zlib.compress(m.tobytes(), 6) + struct.pack("=iii", 1, 36, 5)      # CV_32FC1 = 5
    assert np.array_equal(dbio.uncompress_data(blob), m)
    ids = np.array([[3, 1, 2]], np.int32)
    assert np.array_equal(dbio.uncompress_data(zlib.compress(ids.tobytes()) + struct.pack("=iii", 1, 3, 4)), ids)   # CV_32SC1 = 4
    assert dbio.uncompress_data(b"").size == 0
    with pytest.raises(dbio.DbFormatError):
        dbio.uncompress_data(zlib.compress(bytes(10)) + struct.pack("=iii", 1, 3, 5))


def graph_links(kind, places, rng):
    """(links, partners) of bayes_cases' chain / loops / merged graphs, and the same as Link rows: links one margin apart as kNeighbor
    (the chain) or kNeighborMerged (the extra ones), partners at margin 0 as loop closures, each stored from both places; plus a
    local-space closure, which the walk must ignore."""
    n = len(places)
    links = [(places[i], places[i + 1]) for i in range(n - 1)]
    partners = []
    extra = []
    if kind == "loops":
        for _ in range(max(1, n // 20)):
            a, b = rng.choice(n, 2, replace=False)
            extra.append((places[a], places[b]))
    elif kind == "merged":
        for _ in range(max(1, n // 15)):
            a, b = rng.choice(n, 2, replace=False)
            partners.append((places[a], places[b]))
    rows = []
    closure = [graph.GLOBAL_CLOSURE, graph.LOCAL_TIME_CLOSURE, graph.USER_CLOSURE, graph.VIRTUAL_CLOSURE]
    for a, b in links:
        rows += [(a, b, graph.NEIGHBOR), (b, a, graph.NEIGHBOR)]
    for a, b in extra:
        rows += [(a, b, graph.NEIGHBOR_MERGED), (b, a, graph.NEIGHBOR_MERGED)]
    for k, (a, b) in enumerate(partners):
        rows += [(a, b, closure[k % 4]), (b, a, closure[k % 4])]
    rows += [(places[0], places[-1], graph.LOCAL_SPACE_CLOSURE), (places[-1], places[0], graph.LOCAL_SPACE_CLOSURE)]
    rows.sort()
    arr = np.array(rows, np.int32)
    return links + extra, partners, dbio.Links(arr[:, 0], arr[:, 1], arr[:, 2], np.zeros((len(rows), 3, 4), np.float32))


@pytest.mark.parametrize("kind", ["chain", "loops", "merged"])
@pytest.mark.parametrize("pattern", ["default", "trunc5", "zerodiag"])
def test_neighbour_tables_equal_the_oracle_walk(kind, pattern):
    rng = np.random.default_rng(sum(map(ord, kind + pattern)))
    places = list(range(3, 3 + 2 * 150, 2))           # ids with gaps
    links, partners, rows = graph_links(kind, places, rng)
    lc = parse_prediction_lc(PATTERNS[pattern])
    levels = n_levels(PATTERNS[pattern])
    want = graph_tables(places, levels, links, partners)
    got = graph.bayes_neighbors(places, rows, len(lc) - 1)
    assert got == want
    ids, cp, r, lv = graph.prediction_tables(places, got)
    wcp, wr, wlv = prediction_columns(with_vp(places, True), want.__getitem__)
    assert list(ids) == with_vp(places, True) and np.array_equal(cp, wcp) and np.array_equal(r, wr) and np.array_equal(lv, wlv)
    # and the same posterior through the oracle as the hand-built tables of the Bayes tests
    a, b = BayesFilterOracle(PATTERNS[pattern]), BayesFilterOracle(PATTERNS[pattern])
    for t in range(4):
        like = likelihood(with_vp(places, True), t, rng)
        pa = a.compute_posterior_sparse(with_vp(places, True), like, got.__getitem__)
        pb = b.compute_posterior_sparse(with_vp(places, True), like, want.__getitem__)
        assert np.array_equal(pa, pb)


def test_places_outside_the_working_memory_are_not_walked():
    """maxCheckedInDatabase = 0: a place that was not loaded neither appears in a table nor joins two loaded places"""
    rows = dbio.Links(np.array([1, 2, 2, 3], np.int32), np.array([2, 1, 3, 2], np.int32), np.zeros(4, np.int32), np.zeros((4, 3, 4), np.float32))
    assert graph.bayes_neighbors([1, 3], rows, 5) == {1: {1: 0}, 3: {3: 0}}
    assert graph.bayes_neighbors([1, 2, 3], rows, 2) == {1: {1: 0, 2: 1}, 2: {2: 0, 1: 1, 3: 1}, 3: {3: 0, 2: 1}}


# ------------------------------------------------------------------------------------------------ Memory::getGPS ----------------
def get_gps_restated(pid, places, gps, poses, links, max_graph_depth=0):
    """Memory::getGPS(pid, gps, offsetENU, false, maxGraphDepth) (Memory.cpp:4507-4553), statement by statement, in float64."""
    k = places.index(pid)
    if gps[k][0] != 0.0:
        return gps[k], np.zeros(3)
    loaded = set(places)
    by_from = {}
    for a, b, T in links:
        by_from.setdefault(a, []).append((b, T))
    # getNeighborsId(id, maxGraphDepth, 0, incrementMarginOnLoop=true, ...): every link one margin out, loaded places only
    ids, next_margin, m = {}, {pid}, 0
    while (max_graph_depth == 0 or m < max_graph_depth) and next_margin:
        cur = sorted(next_margin, reverse=True)
        next_margin = set()
        for j in cur:
            if j not in ids and j in loaded:
                ids[j] = m
                for b, _ in sorted(by_from.get(j, []), key=lambda x: x[0]):
                    if b not in ids and b != j:
                        next_margin.add(b)
        m += 1
    for margin, s in sorted((v, i) for i, v in ids.items()):
        ks = places.index(s)
        if gps[ks][0] > 0.0:
            # graph::computePath(s, pid): Dijkstra by distance, a node keeps the pose of the link that first reached it
            nodes = {s: (0.0, np.eye(4))}
            closed, path = set(), None
            while True:
                open_ = [(c, i) for i, (c, _) in nodes.items() if i not in closed]
                if not open_:
                    break
                c, u = min(open_)
                closed.add(u)
                if u == pid:
                    path = nodes[u][1]
                    break
                for b, T in sorted(by_from.get(u, []), key=lambda x: x[0]) if u in loaded else []:
                    if b != u and b not in nodes:
                        T4 = np.vstack([T.astype(np.float64), [0, 0, 0, 1]])
                        nodes[b] = (c + float(np.linalg.norm(T[:, 3].astype(np.float64))), nodes[u][1] @ T4)
            if path is not None:
                R = poses[ks][:, :3].astype(np.float64)
                theta = (-(gps[ks][5] - 90.0)) * np.pi / 180.0 - np.arctan2(R[1, 0], R[0, 0])
                Rz = np.array([[np.cos(theta), -np.sin(theta), 0], [np.sin(theta), np.cos(theta), 0], [0, 0, 1]])
                return gps[ks], Rz @ R @ path[:3, 3]
    return np.zeros(6), np.zeros(3)


@pytest.mark.parametrize("max_graph_depth", [0, 3])
def test_gps_offsets_equal_the_restatement(max_graph_depth):
    """A trajectory of 60 places with a branch, loop closures, a second session unlinked from the first, fixes on some places; places
    without a fix take the nearest fix through the graph, offset by the path's pose in ENU."""
    rng = np.random.default_rng(11 + max_graph_depth)
    places = list(range(1, 61))
    poses = {p: yaw_pose(rng.uniform(-20, 20), rng.uniform(-20, 20), rng.uniform(-3, 3)) for p in places}
    pairs = [(p, p + 1) for p in range(1, 40)] + [(12, 41)] + [(p, p + 1) for p in range(41, 50)] + [(p, p + 1) for p in range(51, 60)]
    pairs += [(5, 30), (8, 45)]                      # loop closures: a second way through the graph
    links = []
    for a, b in pairs:
        links.append((a, b, relative(poses[a], poses[b])))
        links.append((b, a, relative(poses[b], poses[a])))
    links.sort(key=lambda l: (l[0], l[1]))
    gps = np.zeros((60, 6))
    for p in (1, 17, 33, 47, 52):
        gps[p - 1] = (100.0 + p, -73.5 + 1e-4 * p, 45.4 + 1e-4 * p, 20.0 + p, 3.0, rng.uniform(0, 360))
    gps[58] = 0.0                                    # session 2 (51-60) has one fix, at 52
    arr = dbio.Links(np.array([l[0] for l in links], np.int32), np.array([l[1] for l in links], np.int32), np.zeros(len(links), np.int32),
                     np.stack([l[2] for l in links]))
    pose_arr = np.stack([poses[p] for p in places])
    got_gps, got_off = graph.gps_of_places(places, gps, pose_arr, arr, max_graph_depth)
    n_offsets = 0
    for k, p in enumerate(places):
        wg, wo = get_gps_restated(p, places, gps, pose_arr, links, max_graph_depth)
        assert np.array_equal(got_gps[k], wg), f"place {p}"
        assert np.allclose(got_off[k], wo, rtol=1e-5, atol=2e-4), f"place {p}: {got_off[k]} != {wo}"
        n_offsets += bool(gps[k, 0] == 0 and wg[0] > 0)
    assert n_offsets > 10
    assert (got_gps[:, 0] > 0).all() if max_graph_depth == 0 else (got_gps[:, 0] == 0).any()


# ------------------------------------------------------------------------------------------------ the one call ------------------
def world_db(tmp_path, rng, name="map.db", **kw):
    vocab, word_ids, nodes, feats = small_map(rng)
    poses = {n: yaw_pose(0.7 * n, 0.2 * n, 0.05 * n) for n in nodes}
    links = [l for a in nodes[:-1] for l in ((a, a + 1, 0, relative(poses[a], poses[a + 1])), (a + 1, a, 0, relative(poses[a + 1], poses[a])))]
    args = dict(links=links, opt=(np.array(nodes, np.int32), np.stack([poses[n] for n in nodes])), gps={2: (5.0, -73.6, 45.5, 30.0, 4.0, 45.0)},
                gdesc=[(n, 1, np.full((1, 8), n, np.float32)) for n in nodes], poses=poses)
    args.update(kw)
    db = str(tmp_path / name)
    make_map_db(db, word_ids, vocab, nodes, feats, **args)
    return db, vocab, word_ids, nodes, feats


def test_open_sets_every_table_in_order(tmp_path):
    rng = np.random.default_rng(8)
    db, vocab, word_ids, nodes, feats = world_db(tmp_path, rng)
    eng = RecordingEngine()
    res = dbio.open_localization_map(eng, db)
    names = [c[0] for c in eng.calls]
    assert names == ["add_words", "update", "load_csr", "set_ni", "sig_add_batch", "sig_words_add_batch", "clients_set_map",
                     "clients_set_map_poses", "clients_set_map_gps", "gdesc_add"]
    assert list(res.places) == nodes and res.poses_set and res.gps_set and res.n_gps_fixes == 1 and res.n_gps_offsets == len(nodes) - 1
    assert res.n_global_descriptors == len(nodes) and res.skipped == {} and res.n_features == len(feats)
    # the same dictionary and inverted index as cold_start
    cold = RecordingEngine()
    dbio.cold_start(cold, db)
    for a, b in zip(cold.calls, eng.calls[:4]):
        assert a[0] == b[0] and all(np.array_equal(x, y) for x, y in zip(a[1], b[1]))
    ids, cp, r, lv, lc, vpp = eng.calls[6][1]
    assert list(ids) == [-1] + nodes and lc == graph.DEFAULT_PREDICTION_LC and vpp == 0.9
    # without optimised poses, GPS fixes and global descriptors: each part skipped, and said so
    db2, *_ = world_db(tmp_path, np.random.default_rng(8), "bare.db", opt=None, gps=None, gdesc=None)
    eng2 = RecordingEngine()
    res2 = dbio.open_localization_map(eng2, db2)
    assert [c[0] for c in eng2.calls] == names[:7] and set(res2.skipped) == {"poses", "gps", "global_descriptors"}
    # poses that do not cover every place: proximity is not set up
    db3, *_ = world_db(tmp_path, np.random.default_rng(8), "partial.db", opt=(np.array([1, 2], np.int32), np.stack([np.eye(3, 4)] * 2)))
    res3 = dbio.open_localization_map(RecordingEngine(), db3)
    assert not res3.poses_set and "poses" in res3.skipped


def test_bad_signatures_and_a_subset(tmp_path):
    rng = np.random.default_rng(9)
    vocab, word_ids, nodes, feats = small_map(rng)
    db = str(tmp_path / "map.db")
    make_map_db(db, word_ids, vocab, nodes + [7], feats)       # node 7 has no Feature rows
    assert list(dbio.open_localization_map(RecordingEngine(), db).places) == nodes + [7]
    res = dbio.open_localization_map(RecordingEngine(), db, bad_signatures_ignored=True)
    assert list(res.places) == nodes and list(res.dropped_bad_signatures) == [7]
    eng = RecordingEngine()
    assert list(dbio.open_localization_map(eng, db, node_ids=[5, 2, 3]).places) == [2, 3, 5]
    assert list(eng.calls[-1][1][0]) == [-1, 2, 3, 5]


def refused(tmp_path, name, engine=None, **kw):
    rng = np.random.default_rng(12)
    vocab, word_ids, nodes, feats = small_map(rng)
    mutate = kw.pop("mutate", None)
    if mutate:
        vocab, word_ids, nodes, feats, kw = mutate(vocab, word_ids, nodes, feats, kw)
    db = str(tmp_path / f"{name}.db")
    make_map_db(db, word_ids, vocab, nodes, feats, **kw)
    eng = engine or RecordingEngine()
    with pytest.raises(dbio.DbFormatError) as ex:
        dbio.open_localization_map(eng, db)
    return eng, str(ex.value)


def test_refusals_leave_the_engine_untouched(tmp_path):
    cases = {
        "old": dict(version="0.12.4"),
        "intermediate": dict(weights={3: -1}),
        "missing_word": dict(mutate=lambda v, w, n, f, kw: (v[:-10], w[:-10], n, f + [(1, int(w[-1]), 1.0, 1.0, None, bytes(32))], kw)),
        "mixed_sizes": dict(mutate=lambda v, w, n, f, kw: (v, w, n, f + [(2, 1, 1.0, 1.0, None, bytes(16))], kw)),
        "opt_lengths": dict(opt=(np.array([1, 2, 3], np.int32), np.zeros((2, 3, 4), np.float32))),
        "gdesc_type": dict(gdesc=[(1, 2, np.zeros((1, 4), np.float32))]),
        "gdesc_two": dict(gdesc=[(1, 1, np.zeros((1, 4), np.float32)), (1, 1, np.ones((1, 4), np.float32))]),
    }
    for name, kw in cases.items():
        eng, msg = refused(tmp_path, name, **kw)
        assert eng.calls == [], f"{name}: {eng.calls[0][0]} was called ({msg})"
    # another descriptor size or type than the engine's
    for k, eng in enumerate((RecordingEngine(desc_dim=64), RecordingEngine(desc_type=1, desc_dim=32))):
        eng, msg = refused(tmp_path, f"engine_{k}", engine=eng)
        assert eng.calls == [] and "engine holds" in msg
    # more Feature rows on one node than the stores take: the engine's own message, and its only call is the refused one
    big = lambda v, w, n, f, kw: (v, w, n, f + [(4, 1, 1.0, 1.0, None, bytes(32))] * 4100, kw)
    eng, msg = refused(tmp_path, "capacity", mutate=big)
    assert "at most 4096 features per signature" in msg and [c[0] for c in eng.calls] == []
