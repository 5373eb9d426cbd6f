"""The episode-return rule of include/pcl.h (pcl_bind_episodes), on the host.

Over per-step arrays of what the engine produced, [T, B] each: reward (int or float),
has_reward and the plot frame after the step.  A step that skipped an env (a frozen env, an
env a masked reset left alone) is marked in `ran` and changes nothing.  The sums are plain
Python float additions in step order, which is what the device must reproduce bit for bit.
"""

import numpy as np


def returns(reward, has_reward, frame, ran=None, start=None):
  """f64 [T, B]: each env's episode return after every step.

  R = r at a step whose frame is 0 (a (re)start), else R + r, with r = float(reward) where
  has_reward and 0.0 where not.  `start` f64 [B]: R before step 0 (default 0.0); `ran`
  bool [T, B]: False where the step wrote nothing for the env (default: every step ran).
  """
  reward, has_reward, frame = np.asarray(reward), np.asarray(has_reward), np.asarray(frame)
  T, B = frame.shape
  ran = np.ones((T, B), bool) if ran is None else np.asarray(ran, bool)
  ret = [0.0] * B if start is None else [float(x) for x in start]
  out = np.zeros((T, B), np.float64)
  for t in range(T):
    for e in range(B):
      if ran[t, e]:
        r = float(reward[t, e]) if has_reward[t, e] else 0.0
        ret[e] = r if frame[t, e] == 0 else ret[e] + r
      out[t, e] = ret[e]
  return out


def same_bits(a, b):
  """Are two f64 arrays equal bit for bit (so -0.0 != 0.0, and NaN == the same NaN)?"""
  a = np.ascontiguousarray(a, dtype=np.float64)
  b = np.ascontiguousarray(b, dtype=np.float64)
  return a.shape == b.shape and np.array_equal(a.view(np.uint64), b.view(np.uint64))
