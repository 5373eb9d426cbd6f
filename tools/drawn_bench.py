"""Step time of compiled code that draws from the global generators, against the same
game without draws.

The monsters game of tests/drawn_games.py (a player, two wandering monsters, a fruit that
respawns at random) runs twice on one H100, both levels alternating over the envs: once
as written, and once with each draw replaced by an int expression of the frame number in
the same place.  Each env and step of the drawing game makes four draws (two float
comparisons for the player's bonus and trap, one randint and one choice for the
monsters), two more when the fruit is eaten; a float draw takes two MT19937 outputs,
an int draw one or more.  Both step the same seeded actions through `pcl_run` (one C call
per timed window), timed with CUDA events after a warm-up, three alternating repeats per
batch size.  The same run steps a fresh drawing engine and checks sampled envs against the
oracle (oracle/compiled.py) every step, and reads the card's name, power limit and
maximum SM clock (the clock the kernels ran at is not sampled).

    python tools/drawn_bench.py [--batch 4096 65536] [--steps 1000] [--warmup 100]

Prints one JSON line per batch size, µs per step for both games and the extra cost per
draw (the difference divided by four draws per env).
"""

import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
sys.path.insert(0, os.path.join(ROOT, 'tools'))

import numpy as np                                                # noqa: E402

import trajectory                                                 # noqa: E402
from oracle import compiled as ocompiled                          # noqa: E402
from compiled_bench import card, time_run                         # noqa: E402
from pycolab_b200 import batched, compat, compiler, lowering      # noqa: E402

DRAWS_PER_ENV_STEP = 4


def load_games():
  saved = {k: v for k, v in sys.modules.items() if k == 'pycolab' or k.startswith('pycolab.')}
  compat.uninstall()
  try:
    return compat.load_example(os.path.join(ROOT, 'tests', 'drawn_games.py'))
  finally:
    compat.uninstall()
    sys.modules.update(saved)


def fixed_classes(g):
  """The monsters' classes with every draw replaced by an int expression."""

  class Player(g.Player):
    def update(self, actions, board, layers, backdrop, things, the_plot):
      if actions == 0:
        self._north(board, the_plot)
      elif actions == 1:
        self._south(board, the_plot)
      elif actions == 2:
        self._west(board, the_plot)
      elif actions == 3:
        self._east(board, the_plot)
      elif actions == 5:
        the_plot.terminate_episode()
      if the_plot.frame % 10 == 3:
        self.bonuses += 1
        the_plot.add_reward(1)
      if the_plot.frame % 20 == 19:
        the_plot.terminate_episode(0.5)
      if self.position == things['a'].position or self.position == things['b'].position:
        the_plot.add_reward(-3)
        the_plot.terminate_episode()

  class NumpyMonster(g.NumpyMonster):
    def update(self, actions, board, layers, backdrop, things, the_plot):
      move = the_plot.frame % 4
      if move == 0:
        self._north(board, the_plot)
      elif move == 1:
        self._south(board, the_plot)
      elif move == 2:
        self._west(board, the_plot)
      else:
        self._east(board, the_plot)

  class PythonMonster(g.PythonMonster):
    def update(self, actions, board, layers, backdrop, things, the_plot):
      move = (the_plot.frame * 3 + 1) % 4
      if move == 0:
        self._north(board, the_plot)
      elif move == 1:
        self._south(board, the_plot)
      elif move == 2:
        self._west(board, the_plot)
      elif move == 3:
        self._east(board, the_plot)

  class Fruit(g.Fruit):
    def update(self, actions, board, layers, backdrop, things, the_plot):
      player = things['P'].position
      if self.curtain[player]:
        self.curtain[player] = False
        self.eaten += 1
        the_plot.add_reward(5)
        row = 1 + the_plot.frame % 4
        col = 1 + the_plot.frame % 8
        self.curtain[row, col] = True

  return {'P': Player, 'a': NumpyMonster, 'b': PythonMonster, 'f': Fruit}


def make_levels(g, classes):
  out = []
  for level in range(2):
    game = g.ascii_art.ascii_art_to_game(
        g.MONSTERS_ART[level], what_lies_beneath=' ',
        sprites={ch: classes[ch] for ch in 'Pab'}, drapes={'f': classes['f']},
        update_schedule=[['P', 'a', 'b'], ['f']], z_order='fabP')
    out.append(lowering.lower(game))
  return out


def check_against_oracle(levels, B, steps, seed=3):
  """Step a fresh drawing engine of B envs; compare 8 sampled envs with the oracle."""
  import torch
  eng = batched.BatchedEngine(levels, batch=B, rng_seed=seed)
  rs = np.random.RandomState(B)
  table = rs.randint(0, 6, size=(steps, B)).astype(np.int32)
  sample = sorted({0, 1, B - 2, B - 1} | set(rs.randint(2, B - 2, size=4).tolist()))
  want = {e: trajectory.run_trajectory(
      lambda e=e, w=ocompiled.seeded_words(levels[e % 2], seed + e):
      ocompiled.make_world(levels[e % 2], w), table[:, e].tolist()) for e in sample}
  res = eng.its_showtime()
  actions = torch.from_numpy(table).cuda()
  for t in range(steps + 1):
    if t > 0:
      res = eng.play(actions[t - 1])
    boards, reward = res.board.cpu().numpy(), res.reward.cpu().numpy()
    done = res.done.cpu().numpy()
    for e in sample:
      w = want[e]
      if not ((boards[e] == w['boards'][t]).all() and reward[e] == w['reward'][t] and
              done[e] == w['game_over'][t]):
        return False
  return int((eng.error_codes() != 0).sum()) == 0


def main():
  import torch
  ap = argparse.ArgumentParser()
  ap.add_argument('--batch', type=int, nargs='+', default=[4096, 65536])
  ap.add_argument('--steps', type=int, default=1000)
  ap.add_argument('--warmup', type=int, default=100)
  ap.add_argument('--repeats', type=int, default=3)
  ap.add_argument('--check-steps', type=int, default=200)
  args = ap.parse_args()
  g = load_games()
  compiler.register(*g.CLASSES)
  fixed = fixed_classes(g)
  compiler.register(*fixed.values())
  games = {'drawn': make_levels(g, {'P': g.Player, 'a': g.NumpyMonster, 'b': g.PythonMonster,
                                    'f': g.Fruit}),
           'fixed': make_levels(g, fixed)}
  assert games['drawn'][0].program_arg[1] == 2 and games['fixed'][0].program_arg[1] == 0
  print(json.dumps({'card': card()}), flush=True)
  for B in args.batch:
    rs = np.random.RandomState(B)
    T = args.warmup + args.steps
    actions = torch.from_numpy(rs.randint(0, 6, size=(T, B)).astype(np.int32)).cuda()
    engines = {name: batched.BatchedEngine(levels, batch=B) for name, levels in games.items()}
    for eng in engines.values():
      eng.its_showtime()
    times = {name: [] for name in engines}
    for _ in range(args.repeats):                # alternate the two games
      for name, eng in engines.items():
        times[name].append(time_run(eng, actions, args.steps, args.warmup))
    extra = min(times['drawn']) - min(times['fixed'])
    same = check_against_oracle(games['drawn'], B, args.check_steps)
    print(json.dumps({'batch': B, 'steps': args.steps, 'warmup': args.warmup,
                      'us_per_step': {k: [round(x, 2) for x in v] for k, v in times.items()},
                      'extra_ns_per_draw': round(extra * 1000.0 / (B * DRAWS_PER_ENV_STEP), 4),
                      'oracle_checked_steps': args.check_steps, 'oracle_match': same}),
          flush=True)
    if not same:
      sys.exit('the drawing engine disagrees with the oracle at B=%d' % B)


if __name__ == '__main__':
  main()
