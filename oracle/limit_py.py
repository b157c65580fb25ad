"""CPU oracle of Memory::createSignature's keypoint split — TEST INFRASTRUCTURE ONLY (tests/).

Which keypoints of a detected frame are quantised and which word id each keypoint gets (corelib/src/Memory.cpp:5945-6100):
  bad-signature gate       descriptors.rows >= int(Kp/BadSignRatio * meanWordsPerLocation)   Memory.cpp:5945-5947, :6051-6058
  strongest-N mask         Feature2D::limitKeypoints(keypoints, inliers, ...), ssc = false   Features2d.cpp:412-477
  word list                quantizedToRawIndices, -1, -2, ... for the other keypoints        Memory.cpp:5954-6100
"""
from __future__ import annotations

import numpy as np


def _responses(kps) -> np.ndarray:
    """responses of cv2.KeyPoint objects, of [n,6] keypoint rows (column 4) or of a 1-D array"""
    if isinstance(kps, np.ndarray):
        return np.ascontiguousarray(kps[:, 4] if kps.ndim == 2 else kps, np.float32)
    return np.array([k.response for k in kps], np.float32)


def limit_keypoints_inliers(kps, max_keypoints: int) -> np.ndarray:
    """Feature2D::limitKeypoints(keypoints, inliers, maxKeypoints, imageSize, ssc=false) (Features2d.cpp:412-477), the vector<bool>
    variant: a mask of the kept keypoints, their order unchanged.  The multimap<float, int> of fabs(response) walked in reverse keeps
    the strongest and, among equal responses, the later index (equal keys stay in insertion order)."""
    r = np.abs(_responses(kps))
    n = len(r)
    keep = np.ones(n, bool)
    if max_keypoints > 0 and n > max_keypoints:
        order = sorted(range(n), key=lambda i: (float(r[i]), i), reverse=True)
        keep[:] = False
        keep[order[:max_keypoints]] = True
    return keep


def bad_sign_threshold(bad_sign_ratio: float, mean_words: int) -> int:
    """int(_badSignRatio * float(meanWordsPerLocation)) of Memory::createSignature (Memory.cpp:5947), in float"""
    return int(np.float32(bad_sign_ratio) * np.float32(mean_words))


def signature_word_ids(kps, max_features: int, bad_sign_ratio: float, mean_words: int, quantize):
    """The word list Memory::createSignature assembles (Memory.cpp:5945-6100) for the keypoints kps: the bad-signature gate, the limit
    (limit_keypoints_inliers), the picked rows in ascending keypoint order (quantizedToRawIndices) handed to quantize(indices) -> their
    word ids, and -1, -2, ... in keypoint order for every other keypoint.  Returns (word ids [n] int32, quantizedToRawIndices)."""
    n = len(_responses(kps))
    if n == 0 or n < bad_sign_threshold(bad_sign_ratio, mean_words):
        return -np.arange(1, n + 1, dtype=np.int32), np.zeros(0, np.int64)
    raw = np.flatnonzero(limit_keypoints_inliers(kps, max_features)) if max_features > 0 and n > max_features else np.arange(n)
    words = np.zeros(n, np.int32)
    if len(raw):
        words[raw] = np.asarray(quantize(raw), np.int32)
    neg = np.ones(n, bool)
    neg[raw] = False
    words[neg] = -np.arange(1, int(neg.sum()) + 1, dtype=np.int32)
    return words, raw
