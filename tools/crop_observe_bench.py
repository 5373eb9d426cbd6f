"""Per-step time of an agent's network input from a cropped view: the step, the 9 x 9
egocentric crop and its one-hot planes, three ways.

  A: play() + crop() + torch one_hot / permute / cast
  B: play() with the cropper attached (scrolly_maze: inside the step kernel) + torch one-hot
  C: play() + to_feature_array(chars, crop_spec=...) or to_array(one-hot, crop_spec=...):
     one pcl_crop_observe launch from the board

Workloads: scrolly_maze at 64 x 64 and four_rooms (no crop epilogue), a 9 x 9 window with
pad ' ' and margins (None, None), float32 planes (ObservationToFeatureArray) and uint8
planes (ObservationToArray with a one-hot mapping).  The three paths run on three engines
of the same games and the same seeded actions, alternating within one call: each repeat
times every path in turn.  Per path and repeat: CUDA-event time per step over `--steps`
steps after `--warmup` (the stream's time, which includes any wait for the host), then,
in a separate profiled run of `--profile-steps` steps, the device time of its kernels and
copies per step.  Before timing, the outputs of A, B and C are checked equal at the timed
size for `--check-steps` steps.  Prints JSON lines: the card's name, power limit and
maximum SM clock first, read in the same run.

    python tools/crop_observe_bench.py [--batch 4096] [--steps 1000] [--warmup 100]
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
from pycolab_b200 import batched, levels, lowering             # noqa: E402


def games(name):
  from pycolab_b200.games import scrolly_maze
  from pycolab_b200.games.classics import four_rooms
  if name == 'scrolly_maze64':
    return [lowering.lower(scrolly_maze.make_game(*levels.scrolly_maze_level(1000 + i)))
            for i in range(4)]
  return [lowering.lower(four_rooms.make_game())]


class Path(object):
  """One way of producing the planes, on its own engine."""

  def __init__(self, kind, game_name, B, spec, elem):
    import torch
    self.kind, self.elem, self.spec = kind, elem, spec
    self.eng = eng = batched.BatchedEngine(games(game_name), batch=B)
    self.chars = eng.chars
    self.state = eng.new_crop_state()
    self.view = eng.attach_cropper(spec, state=self.state) if kind == 'B' else None
    lut = np.zeros(256, np.int64)
    lut[[ord(ch) for ch in self.chars]] = np.arange(len(self.chars))
    self.lut = torch.from_numpy(lut).cuda()
    self.onehot = dict((ch, tuple(int(ch == x) for x in self.chars)) for ch in self.chars)
    self.dtype = torch.float32 if elem == 'float32' else torch.uint8
    eng.its_showtime()

  def step(self, actions):
    import torch
    self.eng.play(actions)
    if self.kind == 'C':
      if self.elem == 'float32':
        return self.eng.to_feature_array(self.chars, crop_spec=self.spec, state=self.state)
      return self.eng.to_array(self.onehot, dtype=np.uint8, crop_spec=self.spec,
                               state=self.state)
    crop = self.view if self.kind == 'B' else self.eng.crop(self.spec, state=self.state)
    hot = torch.nn.functional.one_hot(self.lut[crop.long()], len(self.chars))
    return hot.permute(0, 3, 1, 2).to(self.dtype)


def time_path(path, actions, steps, warmup):
  import torch
  for t in range(warmup):
    path.step(actions[t % len(actions)])
  torch.cuda.synchronize()
  start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  start.record()
  for t in range(steps):
    path.step(actions[t % len(actions)])
  stop.record()
  stop.synchronize()
  return start.elapsed_time(stop) * 1000.0 / steps        # us per step


def device_time(path, actions, steps):
  """Device time of the kernels and copies of `steps` steps, per step (us), and the
  kernel names seen, from torch.profiler."""
  import torch
  from torch.profiler import ProfilerActivity, profile
  torch.cuda.synchronize()
  with profile(activities=[ProfilerActivity.CUDA]) as prof:
    for t in range(steps):
      path.step(actions[t % len(actions)])
    torch.cuda.synchronize()
  total, names = 0.0, set()
  for ev in prof.events():
    if ev.device_type == torch.autograd.DeviceType.CUDA:
      total += ev.device_time
      names.add(ev.name[:60])
  return total / steps, sorted(names)


def main():
  import torch
  ap = argparse.ArgumentParser()
  ap.add_argument('--batch', type=int, default=4096)
  ap.add_argument('--steps', type=int, default=1000)
  ap.add_argument('--warmup', type=int, default=100)
  ap.add_argument('--repeats', type=int, default=3)
  ap.add_argument('--profile-steps', type=int, default=200)
  ap.add_argument('--check-steps', type=int, default=20)
  ap.add_argument('--games', nargs='+', default=['scrolly_maze64', 'four_rooms'])
  ap.add_argument('--out', default=None, help='also append the lines to this file')
  args = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit('crop_observe_bench needs a CUDA device: nothing is timed without one')
  lines = [{'card': card(), 'device': torch.cuda.get_device_name(0)}]
  print(json.dumps(lines[0]), flush=True)
  B = args.batch
  spec = batched.scrolling_crop_spec(9, 9, 0, pad_char=' ', scroll_margins=(None, None))
  for game_name in args.games:
    for elem in ('float32', 'uint8'):
      paths = dict((k, Path(k, game_name, B, spec, elem)) for k in 'ABC')
      rs = np.random.RandomState(0)
      actions = [torch.from_numpy(rs.randint(0, 5, B).astype(np.int32)).cuda()
                 for _ in range(64)]
      same = True
      for t in range(args.check_steps):                   # identical outputs, every path
        outs = dict((k, p.step(actions[t])) for k, p in paths.items())
        same &= all(bool(torch.equal(outs['A'], outs[k].contiguous())) for k in 'BC')
      C = len(paths['C'].chars)
      line = dict(game=game_name, elem=elem, batch=B, window=[9, 9], planes=C,
                  bytes_per_step=B * 81 * C * (4 if elem == 'float32' else 1),
                  outputs_identical=bool(same), steps=args.steps, warmup=args.warmup,
                  us_per_step={k: [] for k in 'ABC'}, device_us_per_step={},
                  attached_in_kernel=bool(paths['B'].eng._attached[3]))
      for r in range(args.repeats):
        for k, p in paths.items():
          line['us_per_step'][k].append(round(time_path(p, actions, args.steps,
                                                        args.warmup), 3))
      for k, p in paths.items():
        us, names = device_time(p, actions, args.profile_steps)
        line['device_us_per_step'][k] = round(us, 3)
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
