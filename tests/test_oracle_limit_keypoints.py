"""The oracle's Feature2D::limitKeypoints (vector<bool> variant) against a std::multimap<float, int> reverse walk compiled here with the
host C++ compiler, and the word list Memory::createSignature assembles from it: bad-signature gate, quantizedToRawIndices, negative ids."""
import shutil
import subprocess

import numpy as np
import pytest

from oracle import feature2d_py as f2d
from oracle import limit_py as lim

# the reference's loop (Features2d.cpp:412-477, ssc = false), reading "n max r0 r1 ..." (responses as float bit patterns) per line
MULTIMAP_WALK = r"""
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <map>
#include <vector>
int main()
{
	int n, maxKeypoints;
	while (std::scanf("%d %d", &n, &maxKeypoints) == 2)
	{
		std::vector<float> response(n);
		for (int i = 0; i < n; ++i)
		{
			unsigned bits;
			std::scanf("%u", &bits);
			std::memcpy(&response[i], &bits, 4);
		}
		std::vector<bool> inliers;
		if (maxKeypoints > 0 && n > maxKeypoints)
		{
			inliers.resize(n, false);
			std::multimap<float, int> hessianMap;
			for (int i = 0; i < n; ++i) hessianMap.insert(std::pair<float, int>(std::fabs(response[i]), i));
			std::multimap<float, int>::reverse_iterator iter = hessianMap.rbegin();
			for (int k = 0; k < maxKeypoints && iter != hessianMap.rend(); ++k, ++iter) inliers[iter->second] = true;
		}
		else
			inliers.resize(n, true);
		for (int i = 0; i < n; ++i) std::putchar(inliers[i] ? '1' : '0');
		std::putchar('\n');
	}
	return 0;
}
"""


@pytest.fixture(scope="module")
def multimap_walk(tmp_path_factory):
    cxx = shutil.which("g++") or shutil.which("c++")
    if cxx is None:
        pytest.skip("no C++ compiler")
    d = tmp_path_factory.mktemp("limit")
    src = d / "walk.cpp"
    src.write_text(MULTIMAP_WALK)
    exe = d / "walk"
    r = subprocess.run([cxx, "-O1", "-o", str(exe), str(src)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr

    def run(cases):
        lines = [f"{len(r)} {k} " + " ".join(str(int(b)) for b in np.asarray(r, np.float32).view(np.uint32)) for r, k in cases]
        out = subprocess.run([str(exe)], input="\n".join(lines) + "\n", capture_output=True, text=True, timeout=60)
        assert out.returncode == 0, out.stderr
        res = out.stdout.split("\n")
        return [np.array([c == "1" for c in res[i]], bool) for i in range(len(cases))]

    return run


def cases():
    rng = np.random.default_rng(5)
    out = []
    planted = rng.choice(np.float32([1e-4, 2e-4, 3e-4, 5e-4]), 200).astype(np.float32)     # long runs of equal responses
    for k in (1, 37, 50, 51, 100, 199, 200, 500):
        out.append((planted, k))
    cont = rng.normal(0, 1e-3, 300).astype(np.float32)                                     # negative responses: fabs ranks them
    cont[::7] = -cont[1::7][: len(cont[::7])]                                              # +r and -r tie
    for k in (1, 150, 299, 300, 301):
        out.append((cont, k))
    zeros = np.float32([0.0, -0.0, 0.0, 1e-3, -0.0, -1e-3, 0.0, -0.0])                     # -0.0 and 0.0 are one key
    for k in (1, 2, 3, 4, 7, 8):
        out.append((zeros, k))
    out.append((np.zeros(0, np.float32), 5))                                               # n = 0
    out.append((np.float32([3.0]), 1))
    out.append((np.float32([3.0, 3.0]), 1))
    big = rng.integers(0, 64, 4096).astype(np.float32) * np.float32(1e-5)                  # n = 4096, ties cut by K
    for k in (1, 1000, 4095, 4096, 5000, 0):
        out.append((big, k))
    return out


def test_limit_keypoints_inliers_equals_the_multimap_walk(multimap_walk):
    cs = cases()
    ref = multimap_walk(cs)
    for (r, k), want in zip(cs, ref):
        got = lim.limit_keypoints_inliers(r, k)
        assert got.dtype == bool and len(got) == len(r)
        assert np.array_equal(got, want), (len(r), k)
        assert got.sum() == (min(k, len(r)) if k > 0 else len(r))


def test_limit_keypoints_inliers_takes_keypoints_and_rows():
    import cv2

    r = np.float32([0.5, -0.7, 0.5, 0.1])
    kps = [cv2.KeyPoint(float(i), 0.0, 7.0, -1.0, float(v)) for i, v in enumerate(r)]
    rows = np.zeros((4, 6), np.float32)
    rows[:, 4] = r
    want = np.array([False, True, True, False])                                            # 0.7, then the later 0.5
    assert np.array_equal(lim.limit_keypoints_inliers(kps, 2), want)
    assert np.array_equal(lim.limit_keypoints_inliers(rows, 2), want)
    # and the older selection helper keeps the same set
    kept = f2d.limit_keypoints(kps, 2)
    assert sorted(int(k.pt[0]) for k in kept) == [1, 2]


def _fake_quantize(raw):
    return 1000 + np.asarray(raw)                                                          # a word id that names its keypoint


def test_word_ids_negative_numbering_in_keypoint_order():
    r = np.float32([0.1, 0.9, 0.2, 0.9, 0.05, 0.3, 0.9])
    words, raw = lim.signature_word_ids(r, 4, 0.5, 4, _fake_quantize)
    # picked: the three 0.9 (indices 1, 3, 6) and 0.3 (5), in ascending keypoint order
    assert raw.tolist() == [1, 3, 5, 6]
    assert words.tolist() == [-1, 1001, -2, 1003, -3, 1005, 1006]
    # no limit: every keypoint quantised
    words, raw = lim.signature_word_ids(r, 0, 0.5, 4, _fake_quantize)
    assert raw.tolist() == list(range(7)) and words.tolist() == [1000 + i for i in range(7)]
    # n <= K: every keypoint
    words, raw = lim.signature_word_ids(r, 7, 0.5, 4, _fake_quantize)
    assert raw.tolist() == list(range(7))
    # K = n - 1: only the weakest is left out, and it is -1
    words, _ = lim.signature_word_ids(r, 6, 0.0, 0, _fake_quantize)
    assert words.tolist() == [1000, 1001, 1002, 1003, -1, 1005, 1006]
    # n = 0
    words, raw = lim.signature_word_ids(np.zeros(0, np.float32), 4, 0.5, 4, _fake_quantize)
    assert len(words) == 0 and len(raw) == 0


def test_bad_signature_gate_truncates_like_the_reference():
    # int(0.5f * float(501)) = 250: 249 keypoints are a bad signature, 250 are not
    assert lim.bad_sign_threshold(0.5, 501) == 250
    assert lim.bad_sign_threshold(0.5, 500) == 250
    assert lim.bad_sign_threshold(0.0, 500) == 0 and lim.bad_sign_threshold(0.5, 0) == 0
    assert lim.bad_sign_threshold(0.3, 10) == int(np.float32(0.3) * np.float32(10))
    rng = np.random.default_rng(2)
    called = []

    def q(raw):
        called.append(len(raw))
        return _fake_quantize(raw)

    bad, raw = lim.signature_word_ids(rng.random(249).astype(np.float32), 200, 0.5, 501, q)
    assert bad.tolist() == [-(i + 1) for i in range(249)] and len(raw) == 0 and called == []
    good, raw = lim.signature_word_ids(rng.random(250).astype(np.float32), 200, 0.5, 501, q)
    assert called == [200] and len(raw) == 200 and (good > 0).sum() == 200 and (good < 0).sum() == 50
    assert sorted(good[good < 0].tolist()) == list(range(-50, 0)) and np.all(np.diff(good[good < 0]) < 0)
