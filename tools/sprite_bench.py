"""Step time of a game with plain Sprites on the compiled step program (csrc/compiled.cu).

`bounce` of tests/sprite_games.py (a plain-Sprite ball that draws from NumPy's generator, a
MazeWalker paddle and a brick drape, two levels alternating over the batch) steps seeded
actions through `pcl_run` (one C call per timed window), timed with CUDA events after a
warm-up, three runs at each batch size.  Prints one JSON line with the card's name, power
limit and maximum SM clock, read in the same run, and one per batch size.

With `--ab PARENT_LIB`, it then times games without plain Sprites on two builds in
alternating processes: tools/compiled_bench.py and tools/scrolling_bench.py run with
PCL_LIB_PATH set to PARENT_LIB ("parent") and to this tree's library ("new"), parent first,
for `--rounds` rounds.  Their lines are printed tagged with the build and the round.

    python tools/sprite_bench.py [--batch 4096 65536] [--steps 1000] [--warmup 100]
                                 [--ab PARENT_LIB [--rounds 2]]
"""

import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

import numpy as np                                              # noqa: E402

from compiled_bench import card, time_run                      # noqa: E402
from pycolab_b200 import _lib, batched, compat, compiler, lowering   # noqa: E402


def sprite_games():
  """tests/sprite_games.py on this package."""
  compat.uninstall()
  try:
    return compat.load_example(os.path.join(ROOT, 'tests', 'sprite_games.py'))
  finally:
    compat.uninstall()


def bounce(args):
  import torch
  games = sprite_games()
  compiler.register(*games.CLASSES)
  lowered = [lowering.lower(games.make_bounce(level)) for level in (0, 1)]
  print(json.dumps({'card': card()}), flush=True)
  for B in args.batch:
    rs = np.random.RandomState(B)
    T = args.warmup + args.steps
    actions = torch.from_numpy(rs.randint(0, 3, size=(T, B)).astype(np.int32)).cuda()
    eng = batched.BatchedEngine(lowered, batch=B, rng_seed=1)
    eng.its_showtime()
    times = [time_run(eng, actions, args.steps, args.warmup) for _ in range(args.repeats)]
    torch.cuda.synchronize()
    errors = int((eng.error_codes() != 0).sum())
    print(json.dumps({'game': 'bounce', 'batch': B, 'steps': args.steps,
                      'warmup': args.warmup, 'levels': 2,
                      'us_per_step': [round(x, 2) for x in times], 'env_errors': errors}),
          flush=True)
    if errors:
      sys.exit('bounce latched errors at B=%d' % B)


def ab(args):
  """The existing compiled benchmarks on the parent library and on this tree's."""
  builds = [('parent', os.path.abspath(args.ab)), ('new', _lib.LIB_PATH)]
  benches = [('compiled_bench', []),
             ('scrolling_bench', ['--batch', '4096', '--steps', str(args.scroll_steps),
                                  '--warmup', '20'])]
  for rnd in range(1, args.rounds + 1):
    for bench, extra in benches:
      for build, lib in builds:
        env = dict(os.environ, PCL_LIB_PATH=lib)
        out = subprocess.run([sys.executable, os.path.join(ROOT, 'tools', bench + '.py')] + extra,
                             env=env, check=True, capture_output=True, text=True).stdout
        for line in out.splitlines():
          rec = json.loads(line)
          print(json.dumps(dict({'bench': bench, 'build': build, 'round': rnd}, **rec)),
                flush=True)


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--batch', type=int, nargs='+', default=[4096, 65536])
  ap.add_argument('--steps', type=int, default=1000)
  ap.add_argument('--warmup', type=int, default=100)
  ap.add_argument('--repeats', type=int, default=3)
  ap.add_argument('--ab', default=None, help='the parent build of libpcl.so')
  ap.add_argument('--rounds', type=int, default=2)
  ap.add_argument('--scroll-steps', type=int, default=200)
  args = ap.parse_args()
  bounce(args)
  if args.ab:
    ab(args)


if __name__ == '__main__':
  main()
