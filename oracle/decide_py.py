"""CPU oracle of Rtabmap::process's loop-closure decision for one localisation client — TEST INFRASTRUCTURE ONLY (tests/).

A literal restatement of corelib/src/Rtabmap.cpp for one client in localisation mode (Mem/IncrementalMemory=false):
  :1263-1265  lastHighestHypothesis = _highestHypothesis; _highestHypothesis = (0, 0); _loopClosureHypothesis = (0, 0)
  :2143-2158  the highest real-place posterior, scanned in descending id order with a strict '>', its value replaced by
              1 - posterior(virtual place)
  :2162-2226  the threshold (RGBD/AggressiveLoopThr when the frame allows it and it is lower), then the single-hypothesis, ratio and
              last-null rejections; the under-ratio status below the threshold
  :2229-2233  small displacement / too fast movement: _highestHypothesis = lastHighestHypothesis
  :3156-3191  the verification of the accepted hypothesis: a failed registration, or a transform longer than
              RGBD/MaxLoopClosureDistance, clears _loopClosureHypothesis.first (_highestHypothesis is not touched)
The epipolar check (Rtabmap/VerifyLoopClosureHypothesis) and proximity detection are not restated.  The posterior comes from outside
(BayesFilter: oracle/bayes_py.py or the reference's compiled BayesFilter.cpp); statuses and flags are those of lcd_b200.h.
"""
from __future__ import annotations

import numpy as np

FRAME_SKIP, FRAME_HOLD, FRAME_AGGRESSIVE = 1, 2, 4
(SKIPPED, HELD, NO_HYPOTHESIS, UNDER_THRESHOLD, UNDER_RATIO, SINGLE_HYPOTHESIS, RATIO, LAST_NULL, ACCEPTED, VERIFY_REJECTED,
 DISTANCE_REJECTED) = range(11)

f32 = np.float32


class DecideClient:
    """One Rtabmap instance's decision state: _highestHypothesis as (id, float value)."""

    def __init__(self, loop_thr=0.11, aggressive_loop_thr=0.05, loop_ratio=0.0, max_loop_closure_distance=0.0):
        self.loop_thr = f32(loop_thr)
        self.aggressive_loop_thr = f32(aggressive_loop_thr)
        self.loop_ratio = f32(loop_ratio)
        self.max_loop_closure_distance = f32(max_loop_closure_distance)
        self.highest = (0, f32(0))

    def reset(self):
        self.highest = (0, f32(0))

    def decide(self, ids, posterior, flags: int = 0):
        """(highest_id, highest_value, loop_id, status) of one frame.  ids / posterior: the posterior map in ascending id order (ids[0] the
        virtual place); ignored for skipped and held frames."""
        last = self.highest
        highest = (0, f32(0))
        loop = (0, f32(0))
        if flags & FRAME_SKIP:
            status = SKIPPED
        elif flags & FRAME_HOLD:
            highest = last
            status = HELD
        else:
            post = np.asarray(posterior, np.float32)
            status = NO_HYPOTHESIS
            if len(post):
                for i in range(len(post) - 1, -1, -1):          # const_reverse_iterator over the std::map
                    if ids[i] > 0 and post[i] > highest[1]:
                        highest = (int(ids[i]), post[i])
                highest = (highest[0], f32(f32(1) - post[0]))  # 1 - posterior.begin()->second
            if highest[0] > 0:
                thr = self.loop_thr
                if (flags & FRAME_AGGRESSIVE) and thr > self.aggressive_loop_thr:
                    thr = self.aggressive_loop_thr
                if highest[1] >= thr:
                    if len(post) <= 2 and thr > 0:
                        status = SINGLE_HYPOTHESIS
                    elif self.loop_ratio > 0 and last[1] and highest[1] < f32(self.loop_ratio * last[1]):
                        status = RATIO
                    elif self.loop_ratio > 0 and last[1] == 0:
                        status = LAST_NULL
                    else:
                        loop = highest
                        status = ACCEPTED
                elif highest[1] < f32(self.loop_ratio * last[1]):
                    status = UNDER_RATIO
                else:
                    status = UNDER_THRESHOLD
        self.highest = highest
        return highest[0], highest[1], loop[0], status

    def verified(self, decision, ok: bool, translation=(0.0, 0.0, 0.0)):
        """The decision after Memory::computeTransform of its accepted hypothesis: ok = a transform was found, translation = its (x, y, z)."""
        hid, hval, loop_id, status = decision
        if status != ACCEPTED:
            return decision
        if not ok:
            return hid, hval, 0, VERIFY_REJECTED
        x, y, z = (f32(v) for v in translation)
        norm = f32(np.sqrt(f32(f32(f32(x * x) + f32(y * y)) + f32(z * z))))   # Transform::getNorm = uNorm(x, y, z)
        if self.max_loop_closure_distance > 0 and norm > self.max_loop_closure_distance:
            return hid, hval, 0, DISTANCE_REJECTED
        return decision
