"""Hand cases for the restatement of proximity detection by space (oracle/proximity_py.py), one per branch of Rtabmap::process's
candidate search (Rtabmap.cpp:2698-2934), Rtabmap::getPaths (:5303-5382) and the suppression of the global hypothesis
(:2894-2911, :3193-3196).  Distances are chosen far from the radius and angle boundaries."""
import math

import numpy as np

from oracle import proximity_py as px


def pose(x, y, z=0.0, yaw_deg=0.0):
    c, s = math.cos(math.radians(yaw_deg)), math.sin(math.radians(yaw_deg))
    return np.array([[c, -s, 0, x], [s, c, 0, y], [0, 0, 1, z]], np.float32)


def chain(ids):
    links = {}
    for a, b in zip(ids, ids[1:]):
        links.setdefault(a, []).append(b)
        links.setdefault(b, []).append(a)
    return links


HERE = pose(0, 0)


def test_nothing_in_radius():
    poses = {1: pose(20, 0), 2: pose(0, -15)}
    nearest, paths, attempts = px.detect(HERE, poses, chain([1, 2]), {}, local_radius=10)
    assert nearest == {} and paths == {} and attempts == []


def test_zero_likelihood_paths_are_walked_nearest_first():
    # two separate chains; with every likelihood 0 the keys order by distance, the nearer path first
    poses = {1: pose(0.9, 0), 2: pose(1.5, 0), 5: pose(-0.4, 0), 6: pose(-2.0, 0)}
    links = {**chain([1, 2]), **chain([5, 6])}
    nearest, paths, attempts = px.detect(HERE, poses, links, {}, path_filtering_radius=1.0)
    assert paths == {5: [5, 6], 1: [1, 2]}
    assert [a[1] for a in attempts] == [5, 1]
    assert attempts[0][0][0] == 0 and attempts[0][0][1] == 5 and np.isclose(attempts[0][0][2], 0.16)


def test_ascending_id_admission_and_the_lost_path():
    # nearest place 2 links only to 3, 3 links to 1: the search from 2 reaches {1, 2, 3}; 1 is admitted first (the path is empty), 2 does
    # not link to 1 and waits, 3 links to 1.  The next round starts from 2 again, and std::map::insert drops that second path of 2.
    poses = {1: pose(3, 0), 2: pose(0.5, 0), 3: pose(2, 0)}
    links = {1: [3], 2: [3], 3: [1, 2]}
    stats = {}
    nearest, paths, _ = px.detect(HERE, poses, links, {}, stats=stats)
    assert paths == {2: [1, 3]} and stats == {"rejected": 1, "lost": 1, "longest": 2}
    # getNeighborsId never steps through a place outside the radius: 4 links 1 and 2 but lies outside
    poses = {1: pose(0.5, 0), 2: pose(1.0, 0), 4: pose(30, 0)}
    _, paths, _ = px.detect(HERE, poses, {1: [4], 2: [4], 4: [1, 2]}, {})
    assert paths == {1: [1], 2: [2]}
    # maxGraphDepth bounds the margins: depth 2 reaches 1 and its neighbours only
    poses = {i: pose(0.3 * i, 0) for i in range(1, 6)}
    _, paths, _ = px.detect(HERE, poses, chain([1, 2, 3, 4, 5]), {}, max_graph_depth=2)
    assert paths == {1: [1, 2], 3: [3, 4], 5: [5]}


def test_highest_likelihood_wins_the_key_and_the_pick():
    poses = {1: pose(0.2, 0), 2: pose(0.6, 0), 3: pose(0.8, 0)}
    _, _, attempts = px.detect(HERE, poses, chain([1, 2, 3]), {2: 3.0, 3: 1.0})
    assert attempts == [((np.float32(3.0), 2, px.rel_norm2(HERE, poses[2])), 2)]


def test_angle_filter():
    # the key's place faces the other way: it is filtered out and the nearest place left is taken
    poses = {1: pose(0.3, 0, yaw_deg=120), 2: pose(0.6, 0, yaw_deg=10)}
    _, _, attempts = px.detect(HERE, poses, chain([1, 2]), {1: 2.0})
    assert attempts[0][1] == 2
    _, _, attempts = px.detect(HERE, poses, chain([1, 2]), {1: 2.0}, angle=0)       # 0 = no angle filter
    assert attempts[0][1] == 1
    # every place of the path filtered: no candidate, no attempt
    _, _, attempts = px.detect(HERE, {1: pose(0.3, 0, yaw_deg=90)}, {}, {})
    assert attempts == []


def test_filtering_radius_and_its_max_loop_closure_distance_cap():
    poses = {1: pose(0.8, 0)}
    assert len(px.detect(HERE, poses, {}, {}, path_filtering_radius=1.0)[2]) == 1
    assert px.detect(HERE, poses, {}, {}, path_filtering_radius=0.5)[2] == []
    assert px.detect(HERE, poses, {}, {}, path_filtering_radius=1.0, max_loop_closure_distance=0.5)[2] == []
    assert len(px.detect(HERE, poses, {}, {}, path_filtering_radius=0.0, max_loop_closure_distance=2.0)[2]) == 1
    assert len(px.detect(HERE, {1: pose(5, 0)}, {}, {}, path_filtering_radius=0.0)[2]) == 1   # off
    assert px.filtering_radius(1.0, 3.0) == np.float32(1.0) and px.filtering_radius(0.0, 0.0) == 0


def test_max_paths_counts_attempts_only():
    # five separate places; the two nearest-keyed by likelihood are beyond the filtering radius and are not attempts
    poses = {1: pose(3, 0), 2: pose(4, 0), 3: pose(0.2, 0), 4: pose(0.4, 0), 5: pose(0.6, 0)}
    like = {1: 5.0, 2: 4.0}
    _, paths, attempts = px.detect(HERE, poses, {}, like, max_paths=2, path_filtering_radius=1.0)
    assert len(paths) == 5 and [a[1] for a in attempts] == [3, 4]
    _, _, attempts = px.detect(HERE, poses, {}, like, max_paths=3, path_filtering_radius=0.0)
    assert [a[1] for a in attempts] == [1, 2, 3]


def test_suppression_by_the_same_and_by_another_place():
    poses = {1: pose(0.3, 0), 7: pose(-0.5, 0)}
    nearest, _, attempts = px.detect(HERE, poses, {}, {})
    assert [a[1] for a in attempts] == [1, 7]
    ok = (True, pose(0.1, 0))
    # the global hypothesis 7 is registered by proximity: accepted stays, kGlobalClosure, no second registration
    acc, types, sup, loop, status, skip = px.apply(nearest, attempts, [ok, ok], 7, 8)
    assert acc == [True, True] and types == [px.LINK_LOCAL_SPACE, px.LINK_GLOBAL] and sup == 7 and (loop, status, skip) == (7, 8, True)
    # only the other place registers: the hypothesis is suppressed
    acc, types, sup, loop, status, skip = px.apply(nearest, attempts, [ok, (False, pose(0, 0))], 7, 8)
    assert sup == 1 and (loop, status, skip) == (0, px.PROXIMITY_SUPPRESSED, True)
    # a hypothesis outside the radius is untouched; a transform over the filtering radius is not accepted
    acc, types, sup, loop, status, skip = px.apply(nearest, attempts, [ok, ok], 9, 8)
    assert sup == 0 and (loop, status, skip) == (9, 8, False) and types == [1, 1]
    acc, _, sup, loop, status, _ = px.apply(nearest, attempts, [(True, pose(2.0, 0)), (True, pose(1.5, 0))], 7, 8)
    assert acc == [False, False] and sup == 0 and loop == 7
