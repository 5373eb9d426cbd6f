"""Per-step time of a trajectory of cropped feature planes, three ways.

  A: a Python loop of play() + to_feature_array(chars, crop_spec=...) per step
  B: one rollout() of T steps with an ObservationToFeatureArray over the same window
  C: that rollout captured once in a CUDA graph and replayed

Workloads as tools/crop_observe_bench.py: scrolly_maze at 64 x 64 and four_rooms, a 9 x 9
window with pad ' ' and margins (None, None), float32 planes of every game character.  The
three paths run on three engines of the same games and the same seeded actions, alternating
within one call: each repeat times every path in turn.  Per path and repeat: CUDA-event
time per step over `--rollouts` rollouts of `--steps` steps after `--warmup` rollouts (the
stream's time, which includes any wait for the host), then, in a separate profiled run of
`--profile-rollouts` rollouts, the device time of its kernels and copies per step: summed,
and busy (the union of their intervals).  Before timing, the trajectories (rewards,
discounts, dones, planes) of A, B and C are checked equal.  Prints JSON lines, the card's
name, power limit and maximum SM clock first, read in the same run.

    python tools/rollout_bench.py [--batch 4096] [--steps 128] [--rollouts 10] [--warmup 2]
                                  [--repeats 3] [--out FILE]
"""

import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

import numpy as np                                              # noqa: E402

from compiled_bench import card                                # noqa: E402
from crop_observe_bench import games                           # noqa: E402
from pycolab_b200 import batched, rendering                    # noqa: E402


class Path(object):
  """One way of producing a trajectory, on its own engine."""

  def __init__(self, kind, game_name, B, spec, actions):
    self.kind, self.spec, self.actions = kind, spec, actions
    self.eng = eng = batched.BatchedEngine(games(game_name), batch=B)
    self.chars = eng.chars
    self.state = eng.new_crop_state()
    self.observer = rendering.ObservationToFeatureArray(self.chars)
    self.traj = self.graph = None
    eng.its_showtime()

  def rollout(self):
    """T steps; returns (reward, discount, done, planes) [T, B, ...]."""
    import torch
    eng = self.eng
    if self.kind == 'A':
      keep = [[], [], [], []]
      for t in range(self.actions.shape[0]):
        eng.play(self.actions[t])
        planes = eng.to_feature_array(self.chars, crop_spec=self.spec, state=self.state)
        for k, x in enumerate((eng.reward, eng.discount, eng.done, planes)):
          keep[k].append(x.clone())
      return tuple(torch.stack(k) for k in keep)
    if self.kind == 'B' or self.graph is None:
      self.traj = eng.rollout(self.actions, observer=self.observer, crop_spec=self.spec,
                              state=self.state, out=self.traj)
      if self.kind == 'C':                 # captured once, after a rollout built the buffers
        torch.cuda.synchronize()
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph):
          eng.rollout(self.actions, observer=self.observer, crop_spec=self.spec,
                      state=self.state, out=self.traj)
    else:
      self.graph.replay()
    return self.traj.reward, self.traj.discount, self.traj.done, self.traj.view

  def step_time(self):
    """One rollout's work, for the timed loops: A keeps nothing but the stream's work."""
    if self.kind != 'A':
      self.rollout()
      return
    for t in range(self.actions.shape[0]):
      self.eng.play(self.actions[t])
      self.eng.to_feature_array(self.chars, crop_spec=self.spec, state=self.state)


def time_path(path, rollouts, warmup):
  import torch
  for _ in range(warmup):
    path.step_time()
  torch.cuda.synchronize()
  start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  start.record()
  for _ in range(rollouts):
    path.step_time()
  stop.record()
  stop.synchronize()
  return start.elapsed_time(stop) * 1000.0 / (rollouts * path.actions.shape[0])


def device_time(path, rollouts):
  """Device time of the kernels and copies of `rollouts` rollouts, per step (us): their
  summed durations, and the time the device was busy with at least one of them (launches
  with programmatic dependent launch start before their predecessor ends and wait inside,
  so the sum counts such overlaps twice); and the kernel names seen, from torch.profiler."""
  import torch
  from torch.profiler import ProfilerActivity, profile
  torch.cuda.synchronize()
  with profile(activities=[ProfilerActivity.CUDA]) as prof:
    for _ in range(rollouts):
      path.step_time()
    torch.cuda.synchronize()
  total, names, spans = 0.0, set(), []
  for ev in prof.events():
    if ev.device_type == torch.autograd.DeviceType.CUDA:
      total += ev.device_time
      names.add(ev.name[:60])
      spans.append((ev.time_range.start, ev.time_range.end))
  busy, end = 0.0, None
  for lo, hi in sorted(spans):
    if end is None or lo > end:
      busy, end = busy + hi - lo, hi
    elif hi > end:
      busy, end = busy + hi - end, hi
  steps = rollouts * path.actions.shape[0]
  return total / steps, busy / steps, sorted(names)


def main():
  import torch
  ap = argparse.ArgumentParser()
  ap.add_argument('--batch', type=int, default=4096)
  ap.add_argument('--steps', type=int, default=128, help='T, the steps of one rollout')
  ap.add_argument('--rollouts', type=int, default=10)
  ap.add_argument('--warmup', type=int, default=2)
  ap.add_argument('--repeats', type=int, default=3)
  ap.add_argument('--profile-rollouts', type=int, default=2)
  ap.add_argument('--games', nargs='+', default=['scrolly_maze64', 'four_rooms'])
  ap.add_argument('--out', default=None, help='also append the lines to this file')
  args = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit('rollout_bench needs a CUDA device: nothing is timed without one')
  lines = [{'card': card(), 'device': torch.cuda.get_device_name(0)}]
  print(json.dumps(lines[0]), flush=True)
  B, T = args.batch, args.steps
  spec = batched.scrolling_crop_spec(9, 9, 0, pad_char=' ', scroll_margins=(None, None))
  for game_name in args.games:
    rs = np.random.RandomState(0)
    actions = torch.from_numpy(rs.randint(0, 5, (T, B)).astype(np.int32)).cuda()
    paths = dict((k, Path(k, game_name, B, spec, actions)) for k in 'ABC')
    same = True
    for _ in range(2):                     # C's first rollout is eager, its second a replay
      outs = dict((k, p.rollout()) for k, p in paths.items())
      torch.cuda.synchronize()
      same &= all(bool(torch.equal(a, b)) for k in 'BC' for a, b in zip(outs['A'], outs[k]))
    line = dict(game=game_name, batch=B, window=[9, 9], planes=len(paths['A'].chars),
                rollout_steps=T, outputs_identical=bool(same), rollouts=args.rollouts,
                warmup_rollouts=args.warmup, us_per_step={k: [] for k in 'ABC'},
                device_us_per_step={}, device_busy_us_per_step={})
    for _ in range(args.repeats):
      for k, p in paths.items():
        line['us_per_step'][k].append(round(time_path(p, args.rollouts, args.warmup), 3))
    for k, p in paths.items():
      us, busy, names = device_time(p, args.profile_rollouts)
      line['device_us_per_step'][k] = round(us, 3)
      line['device_busy_us_per_step'][k] = round(busy, 3)
      line['device_kernels_%s' % k] = names
    line['median_us_per_step'] = dict((k, float(np.median(v)))
                                      for k, v in line['us_per_step'].items())
    print(json.dumps(line), flush=True)
    lines.append(line)
    for p in paths.values():
      p.eng.close()
  if args.out:
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, 'a') as f:
      for line in lines:
        f.write(json.dumps(line) + '\n')


if __name__ == '__main__':
  main()
