"""Step time of the compiled program (csrc/compiled.cu) against a hand-written kernel.

four_rooms (examples/classics/four_rooms.py) runs twice on one H100: once on
PCL_PROG_CLASSICS, the kernel written for it, and once on PCL_PROG_COMPILED, interpreting
the bytecode compiled from a PlayerSprite.update() with the example's logic.  Both step
the same seeded actions through `pcl_run` (one C call per timed window), timed with CUDA
events after a warm-up, at each batch size.  The two must agree on every board, reward
and done flag of the last step.  Prints one JSON line per batch size and one with the
card's name, power limit and maximum SM clock, read in the same run (the clock the
kernels ran at is not sampled).

    python tools/compiled_bench.py [--batch 4096 65536] [--steps 1000] [--warmup 100]
"""

import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np                                              # noqa: E402

from pycolab_b200 import ascii_art, batched, compiler, lowering  # noqa: E402
from pycolab_b200.games.classics import four_rooms             # noqa: E402


class FourRoomsPlayer(four_rooms.PlayerSprite):
  """four_rooms.py's PlayerSprite.update: actions 0-3 walk N S W E; (4, 3) pays 1.0 and
  ends the episode."""

  def update(self, actions, board, layers, backdrop, things, the_plot):
    del layers, backdrop, things
    if actions == 0:
      self._north(board, the_plot)
    elif actions == 1:
      self._south(board, the_plot)
    elif actions == 2:
      self._west(board, the_plot)
    elif actions == 3:
      self._east(board, the_plot)
    if self.position == (4, 3):
      the_plot.add_reward(1.0)
      the_plot.terminate_episode()


def card():
  out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm',
                        '--format=csv,noheader'], capture_output=True, text=True)
  return out.stdout.strip().splitlines()[0] if out.returncode == 0 else 'unknown'


def time_run(eng, actions, steps, warmup):
  import torch
  eng.run(actions[:warmup])
  torch.cuda.synchronize()
  start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  start.record()
  eng.run(actions[warmup:warmup + steps])
  stop.record()
  stop.synchronize()
  return start.elapsed_time(stop) * 1000.0 / steps      # us per step


def main():
  import torch
  ap = argparse.ArgumentParser()
  ap.add_argument('--batch', type=int, nargs='+', default=[4096, 65536])
  ap.add_argument('--steps', type=int, default=1000)
  ap.add_argument('--warmup', type=int, default=100)
  ap.add_argument('--repeats', type=int, default=3)
  args = ap.parse_args()
  compiler.register(FourRoomsPlayer)
  compiled = lowering.lower(ascii_art.ascii_art_to_game(
      four_rooms.GAME_ART, what_lies_beneath=' ', sprites={'P': FourRoomsPlayer}))
  stock = lowering.lower(four_rooms.make_game())
  assert compiled.program != stock.program
  print(json.dumps({'card': card()}), flush=True)
  for B in args.batch:
    rs = np.random.RandomState(B)
    T = args.warmup + args.steps
    actions = torch.from_numpy(rs.randint(0, 4, size=(T, B)).astype(np.int32)).cuda()
    engines = {'compiled': batched.BatchedEngine([compiled], batch=B),
               'classics': batched.BatchedEngine([stock], batch=B)}
    for eng in engines.values():
      eng.its_showtime()
    times = {name: [] for name in engines}
    for _ in range(args.repeats):                # alternate the two programs
      for name, eng in engines.items():
        times[name].append(time_run(eng, actions, args.steps, args.warmup))
    a, b = engines['compiled'], engines['classics']
    torch.cuda.synchronize()
    same = (bool((a.board == b.board).all()) and bool((a.done == b.done).all()) and
            bool((a.has_reward == b.has_reward).all()) and
            bool((a.reward == b.reward.double()).all()))
    print(json.dumps({'batch': B, 'steps': args.steps, 'warmup': args.warmup,
                      'us_per_step': {k: [round(x, 2) for x in v] for k, v in times.items()},
                      'same_outputs': same}), flush=True)
    if not same:
      sys.exit('compiled and hand-written four_rooms disagree at B=%d' % B)


if __name__ == '__main__':
  main()
