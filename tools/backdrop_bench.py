"""Step time of a game whose Backdrop has compiled update() code (csrc/compiled.cu
backdrop_step) against the hand-written river of PCL_PROG_CLASSICS (csrc/classics.cu).

The fluvial pair of tests/backdrop_games.py (a MazeWalker swimmer and a Backdrop whose rows
1-3 roll west on even frames, registered with `pycolab_b200.compiler`) and
pycolab_b200.games.fluvial_natation (the same game on the classics kernel) step the same
seeded actions through `pcl_run` (one C call per timed window): `--warmup` steps, then
`--steps` timed with CUDA events, three runs per program, alternating, on the stock level and
on `levels.fluvial_level()`, at each batch size.  After each pair of runs the two programs'
boards, rewards, discounts and done flags must be equal; the script exits non-zero if they
are not.  Prints one JSON line with the card's name, power limit and maximum SM clock, read
in the same run, and one per (level, batch size, program).

With `--ab PARENT_TREE`, it then times games without a compiled Backdrop on two builds in
alternating processes: tools/compiled_bench.py and tools/sprite_bench.py of PARENT_TREE (a
checkout of the parent commit with its library built, "parent") and of this tree ("new"),
parent first, for `--rounds` rounds.  Each build runs with its own binding: this tree's
binding requires `pcl_bind_backdrop`, which a parent library does not export.  Their lines
are printed tagged with the build and the round.

    python tools/backdrop_bench.py [--batch 4096 65536] [--steps 1000] [--warmup 100]
                                   [--ab PARENT_TREE [--rounds 2]] [--out FILE.jsonl]
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
from pycolab_b200 import _lib, batched, compat, compiler, levels, lowering   # noqa: E402
from pycolab_b200.games import fluvial_natation                # noqa: E402


def backdrop_games():
  """tests/backdrop_games.py on this package."""
  compat.uninstall()
  try:
    return compat.load_example(os.path.join(ROOT, 'tests', 'backdrop_games.py'))
  finally:
    compat.uninstall()


def fluvial(args, emit):
  import torch
  games = backdrop_games()
  compiler.register(*games.CLASSES)
  emit({'card': card()})
  same = True
  for level, art in (('stock', list(fluvial_natation.GAME_ART)), ('generated', levels.fluvial_level())):
    for B in args.batch:
      rs = np.random.RandomState(B)
      T = args.warmup + args.steps
      actions = torch.from_numpy(rs.choice([0, 1, 2], size=(T, B), p=[.2, .6, .2])
                                 .astype(np.int32)).cuda()
      engines = {'compiled': batched.BatchedEngine([lowering.lower(games.make_fluvial(art))],
                                                   batch=B),
                 'classics': batched.BatchedEngine([fluvial_natation.make_game(art)], batch=B)}
      assert engines['compiled'].game.program == _lib.PROG_COMPILED
      assert engines['classics'].game.program == _lib.PROG_CLASSICS
      times = {name: [] for name in engines}
      for eng in engines.values():
        eng.its_showtime()
      for _ in range(args.repeats):
        for name, eng in engines.items():
          times[name].append(time_run(eng, actions, args.steps, args.warmup))
        torch.cuda.synchronize()
        a, b = engines['compiled'], engines['classics']
        for field in ('board', 'reward', 'has_reward', 'discount', 'done'):
          same = same and bool((getattr(a, field) == getattr(b, field)).all())
      for name, eng in engines.items():
        emit({'game': 'fluvial', 'level': level, 'program': name, 'batch': B,
              'steps': args.steps, 'warmup': args.warmup,
              'us_per_step': [round(x, 2) for x in times[name]],
              'env_errors': int((eng.error_codes() != 0).sum()), 'outputs_equal': same})
  if not same:
    sys.exit('the compiled and classics programs produced different outputs')


def ab(args, emit):
  """Benchmarks of games without a compiled Backdrop, on the parent library and on this
  tree's."""
  builds = [('parent', os.path.abspath(args.ab)), ('new', ROOT)]
  env = {k: v for k, v in os.environ.items() if k != 'PCL_LIB_PATH'}
  for rnd in range(1, args.rounds + 1):
    for bench in ('compiled_bench', 'sprite_bench'):
      for build, tree in builds:
        out = subprocess.run([sys.executable, os.path.join(tree, 'tools', bench + '.py')],
                             env=env, cwd=tree, check=True, capture_output=True, text=True).stdout
        for line in out.splitlines():
          emit(dict({'bench': bench, 'build': build, 'round': rnd}, **json.loads(line)))


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--batch', type=int, nargs='+', default=[4096, 65536])
  ap.add_argument('--steps', type=int, default=1000)
  ap.add_argument('--warmup', type=int, default=100)
  ap.add_argument('--repeats', type=int, default=3)
  ap.add_argument('--ab', default=None, help="a checkout of the parent commit, its library built")
  ap.add_argument('--rounds', type=int, default=2)
  ap.add_argument('--out', default=None, help='also append every line to this file')
  args = ap.parse_args()
  sink = open(args.out, 'a') if args.out else None

  def emit(rec):
    line = json.dumps(rec)
    print(line, flush=True)
    if sink is not None:
      sink.write(line + '\n')
      sink.flush()
  fluvial(args, emit)
  if args.ab:
    ab(args, emit)


if __name__ == '__main__':
  main()
