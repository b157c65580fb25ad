"""Time dbio.open_localization_map on a C2-sized map (BASELINE configs[1]: 10 000 nodes x 1 000 features, 49 152 words), phase by phase:
the SQLite reads, the two graph walks and the uploads into the engine.  Each engine call is followed by lcd_synchronize, so an upload's
time includes its device work.  Without a GPU (--host-only) only the reads and walks run.

  python tools/time_open_map.py [--nodes 10000] [--features 1000] [--words 49152] [--host-only] [--db PATH]

The database is written to a temporary directory (or PATH, reused when it exists)."""
from __future__ import annotations

import argparse
import os
import sqlite3
import sys
import tempfile
import time
from pathlib import Path

import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
sys.path.insert(0, str(Path(__file__).resolve().parents[1] / "tests"))

from rtabmap_b200 import dbio, graph, synth  # noqa: E402

TIMES: dict[str, float] = {}


def timed(mod, name, label):
    fn = getattr(mod, name)

    def wrap(*a, **k):
        t = time.perf_counter()
        try:
            return fn(*a, **k)
        finally:
            TIMES[label] = TIMES.get(label, 0.0) + time.perf_counter() - t
    setattr(mod, name, wrap)


class SyncedEngine:
    """every engine call timed up to lcd_synchronize"""

    def __init__(self, eng):
        self._e = eng

    def __getattr__(self, name):
        f = getattr(self._e, name)
        if not callable(f):
            return f

        def call(*a, **k):
            t = time.perf_counter()
            r = f(*a, **k)
            self._e.synchronize()
            TIMES["upload " + name] = TIMES.get("upload " + name, 0.0) + time.perf_counter() - t
            return r
        return call

    def __setattr__(self, name, value):
        if name == "_e":
            object.__setattr__(self, name, value)
        else:
            setattr(self._e, name, value)


def write_map(path, n_nodes, feats, n_words, seed=2):
    from test_dbio_map import SCHEMA, INFO, relative, yaw_pose

    rng = np.random.default_rng(seed)
    vocab = synth.make_binary_vocabulary(n_words, 32, 1)
    ids = np.arange(1, n_words + 1, dtype=np.int32)
    m = synth.make_map(ids, n_nodes, feats, seed=seed)
    con = sqlite3.connect(path)
    con.executescript(SCHEMA)
    poses = [yaw_pose(0.5 * k, 0.1 * (k % 50), 0.01 * k) for k in range(n_nodes + 1)]
    opt = np.stack(poses[1:])
    con.execute("INSERT INTO Admin(version, opt_ids, opt_poses) VALUES('0.21.0',?,?);",
                (dbio.compress_data(m.sig_ids.reshape(1, -1)), dbio.compress_data(opt.reshape(1, -1))))
    con.executemany("INSERT INTO Node(id, map_id, weight, stamp, pose, gps) VALUES(?,0,1,?,?,?);",
                    [(int(s), float(s), poses[s].tobytes(),
                      np.array([s, -73.6 + 1e-5 * s, 45.5, 30, 3, 0.0]).tobytes() if s % 20 == 1 else None) for s in m.sig_ids.tolist()])
    con.executemany("INSERT INTO Word(id, descriptor_size, descriptor) VALUES(?,32,?);", [(int(i), vocab[k].tobytes()) for k, i in enumerate(ids)])
    for s0 in range(0, n_nodes, 500):
        rows = []
        for s in range(s0, min(n_nodes, s0 + 500)):
            d = vocab[m.sig_words[s] - 1]
            z = rng.uniform(0.5, 5, feats)
            for j in range(feats):
                rows.append((s + 1, int(m.sig_words[s, j]), float(j % 640), float(j % 480), 0.1, 0.2, float(z[j]), d[j].tobytes()))
        con.executemany("INSERT INTO Feature(node_id, word_id, pos_x, pos_y, size, dir, response, octave, depth_x, depth_y, depth_z, "
                        "descriptor_size, descriptor) VALUES(?,?,?,?,31,0,0,0,?,?,?,32,?);", rows)
    links = []
    for s in range(1, n_nodes):
        links += [(s, s + 1, 0, relative(poses[s], poses[s + 1])), (s + 1, s, 0, relative(poses[s + 1], poses[s]))]
    for s in range(1, n_nodes - 300, 97):
        links += [(s, s + 300, 1, relative(poses[s], poses[s + 300])), (s + 300, s, 1, relative(poses[s + 300], poses[s]))]
    con.executemany("INSERT INTO Link(from_id, to_id, type, information_matrix, transform) VALUES(?,?,?,?,?);",
                    [(a, b, t, INFO, T.tobytes()) for a, b, t, T in links])
    g = np.abs(rng.normal(size=(n_nodes, 256))).astype(np.float32)
    con.executemany("INSERT INTO GlobalDescriptor(node_id, type, data) VALUES(?,1,?);",
                    [(int(s), dbio.compress_data(g[s - 1:s])) for s in m.sig_ids.tolist()])
    con.commit()
    con.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nodes", type=int, default=10000)
    ap.add_argument("--features", type=int, default=1000)
    ap.add_argument("--words", type=int, default=49152)
    ap.add_argument("--host-only", action="store_true")
    ap.add_argument("--db", default=None)
    a = ap.parse_args()
    tmp = None
    db = a.db
    if db is None:
        tmp = tempfile.TemporaryDirectory()
        db = os.path.join(tmp.name, "c2.db")
    if not os.path.exists(db):
        t = time.perf_counter()
        write_map(db, a.nodes, a.features, a.words)
        print(f"wrote {db}: {a.nodes} nodes x {a.features} features, {a.words} words in {time.perf_counter() - t:.1f} s "
              f"({os.path.getsize(db) / 2**20:.0f} MiB)")
    for name in ("read_version", "read_node_ids", "read_signatures", "read_dictionary", "read_links", "read_optimized_poses", "read_gps",
                 "read_global_descriptors"):
        timed(dbio, name, "sqlite " + name)
    timed(graph, "bayes_neighbors", "walk getNeighborsId (Bayes)")
    timed(graph, "prediction_tables", "walk prediction tables")
    timed(graph, "gps_of_places", "walk getGPS")
    timed(graph, "neighbor_links", "walk proximity links")
    if a.host_only:
        class HostOnly:
            desc_type, desc_dim = 0, 32

            def gdesc_dim(self):
                return 0

            def __getattr__(self, name):
                return lambda *x, **k: None
        eng, where = HostOnly(), "host phases only (no engine)"
    else:
        import torch

        from rtabmap_b200 import Engine

        eng = SyncedEngine(Engine(max_words=a.words + 1024, max_signatures=a.nodes + 2, max_queries=min(4096, a.features), max_batch=128))
        eng.clients_create(128)
        props = torch.cuda.get_device_properties(0)
        try:
            import pynvml  # noqa: F401
            pynvml.nvmlInit()
            h = pynvml.nvmlDeviceGetHandleByIndex(0)
            power = f"{pynvml.nvmlDeviceGetEnforcedPowerLimit(h) / 1000:.0f} W"
        except Exception:
            import subprocess
            try:
                power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                                       timeout=30).stdout.strip()
            except Exception:
                power = "power limit unknown"
        where = f"{props.name}, {power}"
    t = time.perf_counter()
    res = dbio.open_localization_map(eng, db)
    total = time.perf_counter() - t
    print(f"open_localization_map: {len(res.places)} places, {res.n_features} features, {res.n_words} words, {res.n_links} links, "
          f"{res.n_gps_fixes} fixes + {res.n_gps_offsets} offsets, {res.n_global_descriptors} global descriptors; skipped {res.skipped}")
    print(f"on {where}")
    for k, v in TIMES.items():
        print(f"  {k:40s} {v * 1e3:10.1f} ms")
    rest = total - sum(TIMES.values())
    print(f"  {'checks and array assembly':40s} {rest * 1e3:10.1f} ms")
    print(f"  {'total':40s} {total * 1e3:10.1f} ms")
    if tmp is not None:
        tmp.cleanup()


if __name__ == "__main__":
    main()
