"""Open a localisation map from an RTAB-Map database: the dictionary, the inverted index, the signature and word stores, the Bayes map,
the optimised poses, the GPS of every place and the global descriptors (SURVEY.md 8(f) next #3), and save the dictionary back.

Host-side I/O only: SQLite rows in, the arrays the C ABI takes out.  Follows the reference's SQLite driver
(corelib/src/DBDriverSqlite3.cpp) on the tables of corelib/src/resources/DatabaseSchema.sql.in:

  Node(id, map_id, weight, stamp, pose BLOB, ..., gps BLOB, ...)             :16-29
  Link(from_id, to_id, type, information_matrix BLOB, transform BLOB, ...)   :54-63
  Word(id, descriptor_size, descriptor BLOB, time_enter)                      :66-72
  Feature(node_id, word_id, pos_x, pos_y, size, dir, response, octave, depth_x, depth_y, depth_z, descriptor_size, descriptor)   :74-89
  GlobalDescriptor(node_id, type, info BLOB, data BLOB)                        :91-97
  Admin(version, ..., opt_ids BLOB, opt_poses BLOB, ...)                      :119-

  read_dictionary      DBDriverSqlite3::loadQuery(VWDictionary &, lastStateOnly)  :3541-3620: words ORDER BY id; a blob as long as
                       descriptor_size is CV_8U, one 4x as long is CV_32F, anything else is fatal; last word id = the largest id
  read_inverted_index  what Memory::enableWordsRef (Memory.cpp:7005-7030) rebuilds from the signatures' word lists: one reference per
                       Feature row with word_id > 0 (multiplicity kept), and Ni = ALL Feature rows of the node
                       (DBDriverSqlite3::getInvertedIndexNiQuery :2775-2790: count(word_id) ... WHERE node_id = ?)
  write_dictionary     DBDriverSqlite3::saveQuery(const std::list<VisualWord *> &) :4734: INSERT INTO Word(id, descriptor_size, descriptor)
  read_node_ids        getAllNodeIdsQuery(ids, ignoreChildren=true) :2457-2520, as Memory::loadDataFromDb calls it for
                       Mem/InitWMWithAllNodes=true (Memory.cpp:239-252): every node with weight > -9
  read_signatures      loadSignaturesQuery :3010-3200 (Node: map_id, weight) and loadWordsQuery :3850-3990 (Feature rows of each node
                       with the reference's own statement, so in its row order: that order is the keypoint index)
  read_links           getAllLinksQuery :2600-2640: ORDER BY from_id, to_id; landmark, pose-prior and gravity links dropped
  read_optimized_poses loadOptimizedPosesQuery :5228-5290: Admin.opt_ids / opt_poses through uncompress_data
  read_gps             Node.gps, 6 doubles (DatabaseSchema.sql.in:25), and Node.pose for Memory::getGPS's offsets
  read_global_descriptors  loadSignaturesQuery's GlobalDescriptor part :3415-3460, data through uncompress_data
  compress_data / uncompress_data  rtabmap::compressData2 / uncompressData (Compression.cpp:239-300)
  cold_start           dictionary + inverted index into an engine
  open_localization_map  all of the above into an engine, in one call, refusing a map the engine cannot serve before any change

The FLANN index blob (Admin.dictionary_index, :3622-3660) is not read: the engine searches exhaustively and keeps no tree.  Images,
depth and calibration (Data) are not read either.  A map's stored 3-D points (Feature.depth_*) are already in each place's base frame,
whatever its localTransform, and are loaded as they are; the clients' own cameras (K, image size and localTransform of
SensorData::cameraModels()[0]) are set with Engine.clients_set_cameras.  Databases older than 0.13.0 (the Map_Node_Word era) are refused.
"""
from __future__ import annotations

import sqlite3
import zlib
from dataclasses import dataclass

import numpy as np


class DbFormatError(ValueError):
    pass


@dataclass
class DictionaryRows:
    ids: np.ndarray          # int32 [n], ascending
    descriptors: np.ndarray  # uint8 [n, size] or float32 [n, size]
    last_word_id: int


@dataclass
class InvertedIndexRows:
    word_ids: np.ndarray  # int32 [n_words], ascending: words that have at least one reference
    row_ptr: np.ndarray   # int64 [n_words + 1]
    sig: np.ndarray       # int32 [nnz] signature (node) id, ascending inside a word
    cnt: np.ndarray       # int32 [nnz] occurrences of the word in that signature
    sig_ids: np.ndarray   # int32 [n_sigs], ascending: every node that has Feature rows
    ni: np.ndarray        # int32 [n_sigs] number of Feature rows of the node (Memory::getNi)


def _connect(path: str) -> sqlite3.Connection:
    con = sqlite3.connect(f"file:{path}?mode=ro", uri=True)
    con.row_factory = None
    return con


def read_dictionary(path: str, last_state_only: bool = False) -> DictionaryRows:
    con = _connect(path)
    try:
        q = "SELECT id, descriptor_size, descriptor FROM Word "
        if last_state_only:
            q += "WHERE time_enter >= (SELECT MAX(time_enter) FROM Info) "  # databases >= 0.11.11 (:3557-3561)
        rows = con.execute(q + "ORDER BY id;").fetchall()
    finally:
        con.close()
    if not rows:
        return DictionaryRows(np.zeros(0, np.int32), np.zeros((0, 0), np.uint8), 0)
    size = int(rows[0][1])
    first = len(rows[0][2])
    if first == size:
        dtype, width = np.uint8, size
    elif first // 4 == size:
        dtype, width = np.float32, size
    else:
        raise DbFormatError(f"Saved buffer size ({first} bytes) is not the same as descriptor size ({size})")
    ids = np.empty(len(rows), np.int32)
    desc = np.empty((len(rows), width), dtype)
    row_bytes = width * np.dtype(dtype).itemsize
    for i, (wid, dsize, blob) in enumerate(rows):
        # one dictionary = one descriptor type and width (VWDictionary::update asserts it when it builds the index, VWDictionary.cpp:557-558, :600-601, :670-671)
        if int(dsize) != size or len(blob) != row_bytes:
            raise DbFormatError(f"word {wid}: descriptor of {len(blob)} bytes / size {dsize} in a dictionary of {row_bytes} bytes / size {size}")
        ids[i] = wid
        desc[i] = np.frombuffer(blob, dtype=dtype, count=width)
    return DictionaryRows(ids, desc, int(ids.max()))


def read_inverted_index(path: str, node_ids=None) -> InvertedIndexRows:
    """node_ids: restrict to these signatures (the working memory being reloaded); None = every node of the Feature table."""
    con = _connect(path)
    try:
        rows = np.array(con.execute("SELECT node_id, word_id FROM Feature;").fetchall(), dtype=np.int64).reshape(-1, 2)
    finally:
        con.close()
    if node_ids is not None:
        rows = rows[np.isin(rows[:, 0], np.asarray(list(node_ids), np.int64))]
    return _inverted_index(rows)


def _inverted_index(rows: np.ndarray) -> InvertedIndexRows:
    """rows: int64 [n, 2] (node id, word id), one per Feature row."""
    if rows.shape[0] == 0:
        z = np.zeros(0, np.int32)
        return InvertedIndexRows(z, np.zeros(1, np.int64), z, z, z, z)
    sig_ids, ni = np.unique(rows[:, 0], return_counts=True)
    refs = rows[rows[:, 1] > 0]
    # (word, signature) pairs with their multiplicity, words ascending, signatures ascending inside a word
    key = refs[:, 1] * (int(sig_ids.max()) + 1) + refs[:, 0]
    uniq, cnt = np.unique(key, return_counts=True)
    w = uniq // (int(sig_ids.max()) + 1)
    s = uniq % (int(sig_ids.max()) + 1)
    word_ids, first = np.unique(w, return_index=True)
    row_ptr = np.concatenate([first, [len(w)]]).astype(np.int64)
    return InvertedIndexRows(word_ids.astype(np.int32), row_ptr, s.astype(np.int32), cnt.astype(np.int32), sig_ids.astype(np.int32), ni.astype(np.int32))


def write_dictionary(path: str, ids, descriptors) -> int:
    """Append words to the Word table (the table must exist: the reference creates it from DatabaseSchema.sql); returns the row count."""
    ids = np.asarray(ids, np.int32)
    d = np.ascontiguousarray(descriptors)
    if d.dtype not in (np.uint8, np.float32) or d.ndim != 2 or len(d) != len(ids):
        raise DbFormatError("descriptors must be uint8 or float32 [n, size], one row per id")
    con = sqlite3.connect(path)
    try:
        with con:
            con.executemany("INSERT INTO Word(id, descriptor_size, descriptor) VALUES(?,?,?);",
                            [(int(i), int(d.shape[1]), d[k].tobytes()) for k, i in enumerate(ids)])
    finally:
        con.close()
    return len(ids)


def cold_start(engine, path: str, node_ids=None) -> tuple[DictionaryRows, InvertedIndexRows]:
    """Load dictionary + inverted index of a database into an engine created for its descriptor type: the device-side equivalent of
    Memory::init -> DBDriver::load(VWDictionary) + enableWordsRef for the reloaded signatures."""
    words = read_dictionary(path)
    index = read_inverted_index(path, node_ids)
    _load_dictionary_and_index(engine, words, index)
    return words, index


def _load_dictionary_and_index(engine, words: DictionaryRows, index: InvertedIndexRows):
    if len(words.ids):
        engine.add_words(words.ids, words.descriptors)
        engine.last_word_id = words.last_word_id
        engine.update()
    if len(index.word_ids):
        missing = np.setdiff1d(index.word_ids, words.ids)
        if len(missing):
            raise DbFormatError(f"{len(missing)} words referenced by Feature rows are not in the Word table (first: {int(missing[0])})")
        engine.load_csr(index.word_ids, index.row_ptr, index.sig, index.cnt)
    if len(index.sig_ids):
        engine.set_ni(index.sig_ids, index.ni)
    return words, index


# ------------------------------------------------------------------------------------------------ compressed matrices ----------
# OpenCV depth codes (CV_8U .. CV_64F) and the numpy types of their elements; type = depth + ((channels - 1) << 3)
_CV_DEPTHS = (np.uint8, np.int8, np.uint16, np.int16, np.int32, np.float32, np.float64)


def compress_data(m: np.ndarray) -> bytes:
    """rtabmap::compressData2 (Compression.cpp:239-266): zlib's compress() of the matrix's bytes, then rows, cols and the OpenCV type as
    three native ints.  m: [rows, cols] or [rows, cols, channels] of one of the OpenCV depths."""
    m = np.ascontiguousarray(m)
    if m.ndim == 1:
        m = m.reshape(1, -1)
    dt = np.dtype(m.dtype).newbyteorder("=")
    depth = next((k for k, t in enumerate(_CV_DEPTHS) if np.dtype(t) == dt), None)
    if depth is None or m.ndim not in (2, 3):
        raise DbFormatError(f"compress_data takes a 2-D or 3-D matrix of an OpenCV depth, got {m.dtype} {m.shape}")
    ch = 1 if m.ndim == 2 else m.shape[2]
    return zlib.compress(m.tobytes()) + np.array([m.shape[0], m.shape[1], depth + ((ch - 1) << 3)], np.int32).tobytes()


def uncompress_data(blob) -> np.ndarray:
    """rtabmap::uncompressData (Compression.cpp:269-300): the last three ints are rows, cols and the OpenCV type; the rest is zlib.
    Returns [rows, cols] (or [rows, cols, channels]); an empty array for a blob shorter than three ints."""
    b = bytes(blob or b"")
    if len(b) < 12:
        return np.zeros((0, 0), np.uint8)
    rows, cols, typ = (int(v) for v in np.frombuffer(b[-12:], np.int32))
    depth, ch = typ & 7, (typ >> 3) + 1
    if depth >= len(_CV_DEPTHS) or rows < 0 or cols < 0:
        raise DbFormatError(f"compressed matrix of type {typ} and size {rows} x {cols}")
    try:
        raw = zlib.decompress(b[:-12])
    except zlib.error as ex:
        raise DbFormatError(f"compressed matrix: {ex}") from None
    dt = np.dtype(_CV_DEPTHS[depth])
    if len(raw) != rows * cols * ch * dt.itemsize:
        raise DbFormatError(f"compressed matrix of {rows} x {cols} x {ch} {dt.name} holds {len(raw)} bytes")
    m = np.frombuffer(raw, dt).copy()
    return m.reshape(rows, cols) if ch == 1 else m.reshape(rows, cols, ch)


# ------------------------------------------------------------------------------------------------ readers of the map ------------
def _version(v: str) -> tuple:
    """uStrNumCmp's order on dotted versions"""
    return tuple(int(x) if x.isdigit() else 0 for x in str(v).split("."))


def _has_table(con, name: str) -> bool:
    return con.execute("SELECT 1 FROM sqlite_master WHERE type='table' AND name=?;", (name,)).fetchone() is not None


def read_version(path: str) -> str:
    """Admin.version (the version of RTAB-Map that created the database); "" without an Admin row."""
    con = _connect(path)
    try:
        if not _has_table(con, "Admin"):
            return ""
        row = con.execute("SELECT version FROM Admin;").fetchone()
    finally:
        con.close()
    return str(row[0]) if row and row[0] is not None else ""


def read_node_ids(path: str) -> np.ndarray:
    """Every node Memory::loadDataFromDb loads with Mem/InitWMWithAllNodes=true: getAllNodeIdsQuery(ids, ignoreChildren=true)
    (DBDriverSqlite3.cpp:2467-2478), whose link clause holds for every node, leaves weight > -9.  int32, ascending."""
    con = _connect(path)
    try:
        rows = con.execute("SELECT DISTINCT id FROM Node WHERE weight>-9 ORDER BY id;").fetchall()
    finally:
        con.close()
    return np.array([r[0] for r in rows], np.int32)


@dataclass
class Signatures:
    ids: np.ndarray          # int32 [n] node ids, in the order asked for
    map_id: np.ndarray       # int32 [n] Node.map_id
    weight: np.ndarray       # int32 [n] Node.weight (-1: intermediate node)
    count: np.ndarray        # int32 [n] Feature rows of each node
    word_ids: np.ndarray     # int32 [n, cap] Feature.word_id in row order (padding 0)
    uv: np.ndarray           # float32 [n, cap, 2] (pos_x, pos_y)
    xyz: np.ndarray          # float32 [n, cap, 3] (depth_x, depth_y, depth_z), NULL -> NaN (padding NaN)
    descriptors: np.ndarray  # uint8 or float32 [n, cap, size] (padding 0)


_FEATURE_ROWS = ("SELECT word_id, pos_x, pos_y, size, dir, response, octave, depth_x, depth_y, depth_z, descriptor_size, descriptor "
                 "FROM Feature WHERE node_id = ?  ORDER BY word_id;")   # loadWordsQuery's statement (:3856-3880), byte for byte


def read_signatures(path: str, node_ids=None) -> Signatures:
    """The Feature rows of each node with the reference's own statement (loadWordsQuery, DBDriverSqlite3.cpp:3850-3990): WHERE node_id = ?
    ORDER BY word_id, so rows of one word come in the order SQLite gives them, as they do in the reference.  That order is the keypoint
    index of Signature::setWords, and through it the word order verification and Reg/RepeatOnce see.  A NULL depth is NaN; a descriptor
    blob of descriptor_size bytes is CV_8U, of 4x that CV_32F, anything else (or a row without a descriptor) is a DbFormatError, and so
    are two descriptor types or sizes in one map.  Node.map_id and Node.weight come from loadSignaturesQuery (:3010-3110).
    node_ids None = read_node_ids(path)."""
    ids = read_node_ids(path) if node_ids is None else np.asarray(list(node_ids), np.int32).reshape(-1)
    con = _connect(path)
    try:
        info = {}
        for nid, map_id, weight in con.execute("SELECT id, map_id, weight FROM Node;"):
            info[int(nid)] = (int(map_id), int(weight) if weight is not None else 0)
        per_node = [con.execute(_FEATURE_ROWS, (int(n),)).fetchall() for n in ids.tolist()]
    finally:
        con.close()
    missing = [int(n) for n in ids.tolist() if int(n) not in info]
    if missing:
        raise DbFormatError(f"{len(missing)} nodes are not in the Node table (first: {missing[0]})")
    n = len(ids)
    count = np.array([len(r) for r in per_node], np.int32)
    cap = int(count.max(initial=0))
    size, dtype = None, np.uint8
    for nid, rows in zip(ids.tolist(), per_node):
        for r in rows:
            dsize, blob = r[10], r[11]
            blen = len(blob) if blob is not None else 0
            if dsize is None or int(dsize) <= 0 or blen == 0:
                raise DbFormatError(f"node {nid}: a Feature row of word {r[0]} has no descriptor")
            dt = np.uint8 if blen == int(dsize) else np.float32 if blen == 4 * int(dsize) else None
            if dt is None:
                raise DbFormatError(f"node {nid}: saved buffer size ({blen} bytes) is not the same as descriptor size ({dsize})")
            if size is None:
                size, dtype = int(dsize), dt
            elif int(dsize) != size or dt != dtype:
                raise DbFormatError(f"node {nid}: a descriptor of {blen} bytes / size {dsize} in a map of {np.dtype(dtype).name} descriptors of size {size}")
            break   # the first row fixes the node's type; every row is checked below through its length
    size = size or 0
    row_bytes = size * np.dtype(dtype).itemsize
    word_ids = np.zeros((n, cap), np.int32)
    uv = np.zeros((n, cap, 2), np.float32)
    xyz = np.full((n, cap, 3), np.nan, np.float32)
    desc = np.zeros((n, cap, size), dtype)
    for k, (nid, rows) in enumerate(zip(ids.tolist(), per_node)):
        c = len(rows)
        if not c:
            continue
        cols = list(zip(*rows))
        if any(d != size for d in cols[10]) or any(b is None or len(b) != row_bytes for b in cols[11]):
            raise DbFormatError(f"node {nid}: descriptors of different sizes in a map of {np.dtype(dtype).name} descriptors of size {size}")
        word_ids[k, :c] = np.array(cols[0], np.int64)
        uv[k, :c, 0] = np.array(cols[1], np.float64)
        uv[k, :c, 1] = np.array(cols[2], np.float64)
        for j in range(3):
            xyz[k, :c, j] = np.array(cols[7 + j], np.float64)          # None -> NaN, as the reference's SQLITE_NULL branch
        desc[k, :c] = np.frombuffer(b"".join(cols[11]), dtype).reshape(c, size)
    map_id = np.array([info[int(x)][0] for x in ids.tolist()], np.int32)
    weight = np.array([info[int(x)][1] for x in ids.tolist()], np.int32)
    return Signatures(ids.astype(np.int32), map_id, weight, count, word_ids, uv, xyz, desc)


@dataclass
class Links:
    from_id: np.ndarray    # int32 [n]
    to_id: np.ndarray      # int32 [n]
    type: np.ndarray       # int32 [n] Link::Type (graph.NEIGHBOR ...)
    transform: np.ndarray  # float32 [n, 3, 4] (zeros: a null transform)


def read_links(path: str) -> Links:
    """getAllLinksQuery (DBDriverSqlite3.cpp:2600-2640): SELECT from_id, to_id, type, transform FROM Link ORDER BY from_id, to_id.  Type
    codes are the schema's (kNeighbor=0 ... kLandmark=8, and kGravity=9, Link.h:41-52).  Landmark links (a negative to_id), pose priors
    and gravity links (from == to) do not join two places and are dropped.  A transform blob that is not 12 floats is a null transform,
    as the reference reads it."""
    con = _connect(path)
    try:
        rows = con.execute("SELECT from_id, to_id, type, transform FROM Link ORDER BY from_id, to_id;").fetchall()
    finally:
        con.close()
    rows = [r for r in rows if int(r[2]) not in (7, 8, 9) and int(r[1]) > 0 and int(r[0]) > 0 and int(r[0]) != int(r[1])]
    T = np.zeros((len(rows), 3, 4), np.float32)
    for k, r in enumerate(rows):
        if r[3] is not None and len(r[3]) == 48:
            T[k] = np.frombuffer(r[3], np.float32).reshape(3, 4)
    return Links(np.array([r[0] for r in rows], np.int32), np.array([r[1] for r in rows], np.int32), np.array([r[2] for r in rows], np.int32), T)


def read_optimized_poses(path: str):
    """loadOptimizedPosesQuery (DBDriverSqlite3.cpp:5228-5290): (ids int32 [n], poses float32 [n, 3, 4]) from Admin.opt_ids / opt_poses,
    or None when the row holds no poses.  opt_ids must be CV_32SC1 and opt_poses CV_32FC1 with 12 values per id (the reference asserts
    both); anything else is a DbFormatError."""
    con = _connect(path)
    try:
        row = con.execute("SELECT opt_ids, opt_poses FROM Admin;").fetchone() if _has_table(con, "Admin") else None
    finally:
        con.close()
    if row is None or not row[1]:
        return None
    ids = uncompress_data(row[0]) if row[0] else np.zeros((1, 0), np.int32)
    poses = uncompress_data(row[1])
    if ids.dtype != np.int32 or ids.ndim != 2 or poses.dtype != np.float32 or poses.ndim != 2:
        raise DbFormatError(f"opt_ids must be CV_32SC1 and opt_poses CV_32FC1, got {ids.dtype} {ids.shape} and {poses.dtype} {poses.shape}")
    if ids.size * 12 != poses.size:
        raise DbFormatError(f"{ids.size} optimised pose ids for {poses.size} pose values (12 per id)")
    return ids.reshape(-1).copy(), poses.reshape(-1, 3, 4).copy()


def read_gps(path: str, node_ids=None):
    """(ids int32 [n], gps float64 [n, 6], pose float32 [n, 3, 4]) of the nodes (all of read_node_ids when None): Node.gps as
    (stamp, longitude, latitude, altitude, error, bearing) (DatabaseSchema.sql.in:25; a missing blob or one of another size reads as
    zeros, no fix, as at DBDriverSqlite3.cpp:3160-3168) and Node.pose, the pose Memory::getGPS turns offsets with (zeros when absent).
    Databases before 0.14.0 have no gps column: every place then reads without a fix."""
    ids = read_node_ids(path) if node_ids is None else np.asarray(list(node_ids), np.int32).reshape(-1)
    with_gps = _version(read_version(path)) >= (0, 14, 0)
    con = _connect(path)
    try:
        q = "SELECT id, pose, gps FROM Node;" if with_gps else "SELECT id, pose, NULL FROM Node;"
        rows = {int(r[0]): r for r in con.execute(q)}
    finally:
        con.close()
    gps = np.zeros((len(ids), 6), np.float64)
    pose = np.zeros((len(ids), 3, 4), np.float32)
    for k, nid in enumerate(ids.tolist()):
        r = rows.get(int(nid))
        if r is None:
            raise DbFormatError(f"node {nid} is not in the Node table")
        if r[1] is not None and len(r[1]) == 48:
            pose[k] = np.frombuffer(r[1], np.float32).reshape(3, 4)
        if r[2] is not None and len(r[2]) == 48:
            gps[k] = np.frombuffer(r[2], np.float64)
    return ids.astype(np.int32), gps, pose


def read_global_descriptors(path: str, node_ids=None):
    """(ids int32 [n] ascending, descriptors float32 [n, dim]) of the GlobalDescriptor table (DBDriverSqlite3.cpp:3415-3460), data
    through uncompress_data, restricted to node_ids when given.  The engine's store holds one fp32 row per signature, so only type 1, one
    row per node and a 1 x dim CV_32F matrix of one dim for the whole map are accepted; anything else is a DbFormatError.  Databases
    without the table (before 0.20.0) have none."""
    con = _connect(path)
    try:
        rows = con.execute("SELECT node_id, type, data FROM GlobalDescriptor ORDER BY node_id;").fetchall() if _has_table(con, "GlobalDescriptor") else []
    finally:
        con.close()
    if node_ids is not None:
        keep = set(int(x) for x in np.asarray(list(node_ids)).reshape(-1).tolist())
        rows = [r for r in rows if int(r[0]) in keep]
    ids = np.array([r[0] for r in rows], np.int32)
    if len(ids) and np.any(np.diff(ids) == 0):
        raise DbFormatError(f"node {int(ids[np.nonzero(np.diff(ids) == 0)[0][0]])} has more than one global descriptor")
    out = []
    for nid, typ, data in rows:
        if int(typ) != 1:
            raise DbFormatError(f"node {nid}: global descriptor of type {typ} (only type 1 is supported)")
        m = uncompress_data(data)
        if m.dtype != np.float32 or m.ndim != 2 or m.shape[0] != 1 or m.shape[1] == 0:
            raise DbFormatError(f"node {nid}: global descriptor must be a 1 x dim CV_32F matrix, got {m.dtype} {m.shape}")
        if out and m.shape[1] != len(out[0]):
            raise DbFormatError(f"node {nid}: global descriptor of {m.shape[1]} dimensions in a map of {len(out[0])}")
        out.append(m[0])
    return ids, (np.stack(out) if out else np.zeros((0, 0), np.float32))


# ------------------------------------------------------------------------------------------------ the one call ------------------
MAX_FEATURES_PER_NODE = 4096   # rows per signature the engine's stores accept (lcd_sig_add_batch / lcd_sig_words_add_batch, lcd_b200.h)


@dataclass
class LocalizationMap:
    """What open_localization_map loaded.  `skipped` names each optional part that was not set, and why."""
    places: np.ndarray        # int32 [n] ascending: the map's real places (lcd_clients_set_map's ids after the virtual place)
    n_words: int              # dictionary words
    n_features: int           # Feature rows in the stores
    cap: int                  # rows per signature in the stores
    n_links: int              # place-to-place links read
    dropped_bad_signatures: np.ndarray   # int32: nodes without Feature rows left out (bad_signatures_ignored)
    poses_set: bool
    n_gps_fixes: int          # places with their own fix
    n_gps_offsets: int        # places that took a neighbour's fix through Memory::getGPS
    gps_set: bool
    n_global_descriptors: int
    skipped: dict


def _probe_capacity(engine, sigs: Signatures, k: int):
    """The engine refuses a store row size over its limit before it changes anything: pass its own message on."""
    from .capi import LcdError

    cap = int(sigs.count[k])
    try:
        engine.sig_add_batch(sigs.ids[k:k + 1], np.zeros((1, cap, engine.desc_dim), sigs.descriptors.dtype), np.zeros((1, cap, 3), np.float32),
                             [cap])
    except LcdError as ex:
        raise DbFormatError(f"node {int(sigs.ids[k])} has {cap} Feature rows: {ex}") from ex
    raise DbFormatError(f"node {int(sigs.ids[k])} has {cap} Feature rows, more than {MAX_FEATURES_PER_NODE}")


def open_localization_map(engine, path: str, node_ids=None, prediction_lc=None, virtual_place_prior: float = 0.9,
                          bad_signatures_ignored: bool = False, gps_max_graph_depth: int = 0) -> LocalizationMap:
    """Everything a localisation service needs from an RTAB-Map database, into an engine created for the map's descriptors, in the
    order a caller would set it by hand:

      1. the dictionary and the inverted index (cold_start)            lcd_dict_add_words, lcd_index_load_csr, lcd_index_set_ni
      2. the verification store: descriptors and 3-D points per place  lcd_sig_add_batch
      3. the word store: word ids and keypoints per place (VhEp)       lcd_sig_words_add_batch
      4. the Bayes map: places, neighbour tables, PredictionLC         lcd_clients_set_map (graph.bayes_neighbors / prediction_tables)
      5. optimised poses and neighbour links (proximity by space)      lcd_clients_set_map_poses, when Admin.opt_poses covers every place
      6. the GPS of every place, with Memory::getGPS's offsets          lcd_clients_set_map_gps, when any place has a fix
      7. global descriptors                                            lcd_gdesc_add, when the table has rows for the places

    node_ids None = every node (Mem/InitWMWithAllNodes=true, Memory.cpp:239-252); bad_signatures_ignored (Mem/BadSignaturesIgnored)
    leaves out nodes without Feature rows (Memory.cpp:262-263); prediction_lc = Bayes/PredictionLC values (graph.DEFAULT_PREDICTION_LC
    when None); gps_max_graph_depth = getGPS's maxGraphDepth (0: unlimited, as Rtabmap.cpp:2066 calls it).  Clients are the caller's
    (Engine.clients_create, before or after).

    Refused with DbFormatError before the engine is touched, so that it stays as it was: a database older than 0.13.0, intermediate
    nodes (weight -1), a Feature word missing from Word, descriptors of mixed sizes or of another type or size than the engine's, opt_ids
    and opt_poses of different lengths, global descriptors the store cannot hold, and a node with more Feature rows than the engine's
    stores accept (with the engine's own LCD_ERR_CAPACITY message).

    3-D points are in each place's base frame whatever its localTransform and are loaded as stored (Data.calibration is not read);
    each localisation client's camera is Engine.clients_set_cameras's."""
    from . import graph
    from .capi import LCD_DESC_U8

    version = read_version(path)
    if not version or _version(version) < (0, 13, 0):
        raise DbFormatError(f"database version {version or '(no Admin row)'} is older than 0.13.0 (Map_Node_Word tables) and is not supported")
    lc = list(graph.DEFAULT_PREDICTION_LC if prediction_lc is None else prediction_lc)
    ids = read_node_ids(path) if node_ids is None else np.unique(np.asarray(list(node_ids), np.int32))
    sigs = read_signatures(path, ids)
    inter = sigs.ids[sigs.weight == -1]
    if len(inter):
        raise DbFormatError(f"{len(inter)} intermediate nodes (weight -1, first: {int(inter[0])}): the decision does not support them")
    dropped = sigs.ids[sigs.count == 0] if bad_signatures_ignored else np.zeros(0, np.int32)
    if len(dropped):
        keep = sigs.count > 0
        sigs = Signatures(sigs.ids[keep], sigs.map_id[keep], sigs.weight[keep], sigs.count[keep], sigs.word_ids[keep], sigs.uv[keep],
                          sigs.xyz[keep], sigs.descriptors[keep])
    places = sigs.ids
    # the engine's descriptors: dictionary and Feature rows alike
    want_dt = np.uint8 if engine.desc_type == LCD_DESC_U8 else np.float32
    words = read_dictionary(path)
    for what, dt, size, n in (("Word", words.descriptors.dtype, words.descriptors.shape[1], len(words.ids)),
                              ("Feature", sigs.descriptors.dtype, sigs.descriptors.shape[2], int(sigs.count.sum()))):
        if n and (dt != want_dt or size != engine.desc_dim):
            raise DbFormatError(f"{what} descriptors are {np.dtype(dt).name} of size {size}; the engine holds {np.dtype(want_dt).name} of size {engine.desc_dim}")
    valid = np.arange(sigs.word_ids.shape[1])[None, :] < sigs.count[:, None]
    flat_nodes = np.broadcast_to(places[:, None], sigs.word_ids.shape)[valid].astype(np.int64)
    flat_words = sigs.word_ids[valid].astype(np.int64)
    index = _inverted_index(np.stack([flat_nodes, flat_words], 1))
    missing = np.setdiff1d(index.word_ids, words.ids)
    if len(missing):
        raise DbFormatError(f"{len(missing)} words referenced by Feature rows are not in the Word table (first: {int(missing[0])})")
    cap = int(sigs.count.max(initial=0))
    if cap > MAX_FEATURES_PER_NODE:
        _probe_capacity(engine, sigs, int(np.argmax(sigs.count)))
    # graph tables, poses, GPS, global descriptors: every check before the first engine call
    links = read_links(path)
    tables = graph.prediction_tables(places, graph.bayes_neighbors(places, links, len(lc) - 1)) if len(places) else None
    skipped = {}
    opt = read_optimized_poses(path)
    poses = None
    if opt is None:
        skipped["poses"] = "Admin.opt_poses is empty: proximity by space is not set up"
    else:
        row = {int(i): k for k, i in enumerate(opt[0].tolist())}
        uncovered = [int(p) for p in places.tolist() if int(p) not in row]
        if uncovered:
            skipped["poses"] = f"{len(uncovered)} places have no optimised pose (first: {uncovered[0]}): proximity by space is not set up"
        elif len(places):
            poses = opt[1][[row[int(p)] for p in places.tolist()]]
    _, gps_raw, node_pose = read_gps(path, places)
    n_fix = int((gps_raw[:, 0] > 0).sum())
    gps = offsets = None
    if n_fix:
        gps, offsets = graph.gps_of_places(places, gps_raw, node_pose, links, gps_max_graph_depth)
    else:
        skipped["gps"] = "no place has a GPS fix"
    g_ids, g_desc = read_global_descriptors(path, places)
    if not len(g_ids):
        skipped["global_descriptors"] = "the GlobalDescriptor table has no rows for the places"
    elif engine.gdesc_dim() not in (0, g_desc.shape[1]):
        raise DbFormatError(f"global descriptors of {g_desc.shape[1]} dimensions; the engine holds {engine.gdesc_dim()}")

    # the engine, in the order a caller sets it by hand
    _load_dictionary_and_index(engine, words, index)
    if cap:
        engine.sig_add_batch(places, sigs.descriptors, sigs.xyz, sigs.count)
        engine.sig_words_add_batch(places, sigs.word_ids, sigs.uv, sigs.count)
    if tables is not None:
        engine.clients_set_map(tables[0], tables[1], tables[2], tables[3], lc, virtual_place_prior)
        if poses is not None:
            engine.clients_set_map_poses(places, poses, *graph.neighbor_links(places, links))
        if gps is not None:
            engine.clients_set_map_gps(places, gps[:, :5], offsets)
    else:
        skipped["map"] = "no places"
    if len(g_ids):
        engine.gdesc_add(g_ids, g_desc)
    n_offsets = int(((gps_raw[:, 0] <= 0) & (gps[:, 0] > 0)).sum()) if gps is not None else 0
    return LocalizationMap(places, len(words.ids), int(sigs.count.sum()), cap, len(links.from_id), dropped.astype(np.int32), poses is not None,
                           n_fix, n_offsets, gps is not None, len(g_ids), skipped)
