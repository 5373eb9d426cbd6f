"""Cases for the un-occluded layers and the curtain export (csrc/render.cu layers_kernel,
behind pcl_layers and pcl_export_curtain): each step program whose curtains the kernel
reads, at the board shapes and pitches the kernel and the step kernels branch on, under
each level binding.

layers_kernel works in 16-column segments: W around 16, 32 and 64 gives a ragged last
segment and bit rows or pattern windows that cross a 32-bit word; pitch = ceil16(W) + 16
and + 64 give segments wholly past the board, which must come out 0 and read nothing.
A level binding says where the static arrays of env e live:
  SHARED   one game: every env reads one copy (stride 0);
  POOL     several games that differ in their patterns and bits, read through d_level;
  PER_ENV  share_levels=False: every array is a per-env copy.

`status` is what pcl_create answers for the case's spec (test_layer_cases.py asks it on
the CPU): every pitch listed here is accepted.  `batch` is 1, 5 or 37 by turns, and at
least 5 for a pool, so that envs read more than one level.  Every case restarts envs inside
its run: the walks quit where the program has a quit action (env 0 always once), and
shockwave's walk heads north long enough to end episodes on its own.  scrolly_maze's walk
quits whenever the player stands on a coin the '@' drape has not yet collected (a scroll
onto it): that quit collects the coin with no '@' motion, so the frame after it shows the
coin window's stale slot (the cell stays in the curtain until the next refresh).
Imports on the CPU; every game is built lazily by the case's `build`.
"""

import collections

import numpy as np

import scrolly_shapes as ss
from rim_sweep import BATCHES, PER_ENV, POOL, SHARED, ceil16

# build() -> Built.  games: lowered games (env e plays games[e % len(games)]);
# make_world(e): a fresh oracle world for env e; draw(rs, T, B): int actions [T, B];
# rng_seed for BatchedEngine; steps: T.
Built = collections.namedtuple('Built', 'games make_world draw rng_seed steps')
Case = collections.namedtuple('Case', 'id program shape pitch binding status batch build')
STEPS = 12


def _batch(i, binding):
  B = BATCHES[i % len(BATCHES)]
  return max(B, 5) if binding == POOL else B


def pitches(W):
  return (ceil16(W), ceil16(W) + 16, ceil16(W) + 64)


def _n_games(binding):
  return 1 if binding == SHARED else 2


def _draw(n, p=None, quit_action=None, quit_p=0.0):
  def draw(rs, T, B):
    a = rs.choice(n, size=(T, B), p=p)
    if quit_action is not None:
      a[rs.random_sample((T, B)) < quit_p] = quit_action
      a[T // 3, 0] = quit_action             # env 0 restarts inside the run at every B
    return a.astype(np.int32)
  return draw


# ------------------------------------------------------------------- scrolly_maze
# (name, board, world, margins, corners of the levels or None)
SCROLLY = [
    ('9x1', (9, 1), (25, 41), ss.NO_MARGINS, None),
    ('6x15', (6, 15), (18, 45), ss.DEFAULT_MARGINS, None),
    ('5x16', (5, 16), (17, 45), ss.DEFAULT_MARGINS, None),
    ('7x17', (7, 17), (19, 51), ss.DEFAULT_MARGINS, None),
    ('8x31', (8, 31), (20, 75), ss.DEFAULT_MARGINS, None),
    ('11x33', (11, 33), (25, 81), ss.DEFAULT_MARGINS, None),
    ('9x63', (9, 63), (21, 121), ss.DEFAULT_MARGINS, None),
    ('9x64', (9, 64), (21, 121), ss.DEFAULT_MARGINS, None),
    ('8x65', (8, 65), (20, 121), ss.DEFAULT_MARGINS, None),
    ('20x20', (20, 20), (34, 61), ss.DEFAULT_MARGINS, None),
    ('33x33', (33, 33), (45, 71), ss.DEFAULT_MARGINS, None),
    # windows whose corner starts left of pattern columns 32, 64 and 96 and walks across
    ('12x20_sweep', (12, 20), (22, 161), ss.DEFAULT_MARGINS, [(5, 20), (5, 56), (5, 84)]),
]


def _scrolly_build(board, world, margins, corners, pitch, n):
  def build():
    arts = [ss.open_level(40 + i, board, world, corner=None if corners is None else corners[i])
            for i in range(n)]
    games = [ss.lowered(ss.facade_game(*a, margins=margins), pitch, repack=board[1] == 1)
             for a in arts]
    make_world = lambda e: ss.oracle_world(*arts[e % n], margins=margins)
    return Built(games, make_world, _scrolly_walk(make_world), 0, 3 * STEPS)
  return build


def coin_under_player(world):
  """Does the player stand on a coin of the '@' pattern that is not yet collected?"""
  coins, player = world.things['@'], world.things['P']
  return bool(coins.pattern[coins.corner[0] + player.row, coins.corner[1] + player.col])


def _scrolly_walk(make_world):
  """Moves (action 4 stays), a quit with probability 0.02 and at T // 3 for env 0, and a
  quit whenever coin_under_player.  Replays the oracle to know where the player stands,
  restarting a world as the lock-step does: an env that ended plays its next action on a
  fresh world."""
  def draw(rs, T, B):
    a = np.zeros((T, B), np.int32)
    for e in range(B):
      world = make_world(e)
      world.its_showtime()
      for t in range(T):
        if world.game_over:
          world = make_world(e)
          world.its_showtime()
          a[t, e] = rs.choice(5)
          continue
        quit = coin_under_player(world) or rs.random_sample() < 0.02 or (e == 0 and t == T // 3)
        a[t, e] = 5 if quit else rs.choice(5, p=[.25, .25, .22, .22, .06])
        world.play(int(a[t, e]))
    return a
  return draw


def _scrolly_cases():
  out = []
  bindings = (SHARED, POOL, PER_ENV)
  for i, (name, board, world, margins, corners) in enumerate(SCROLLY):
    H, W = board
    for j, pitch in enumerate(pitches(W)):
      binding = bindings[(i + j) % 3]
      n = 3 if corners is not None else _n_games(binding)
      if corners is not None and binding == SHARED:
        binding = POOL
      out.append(Case('scrolly_maze-%s-p%d-%s' % (name, pitch, binding), 'scrolly_maze', board,
                      pitch, binding, 'ok', None,
                      _scrolly_build(board, world, margins, corners, pitch, n)))
  return out


# ------------------------------------------------------- bit-row programs
def _marauders_build(rows, cols, pitch, binding):
  def build():
    from pycolab_b200 import levels
    from pycolab_b200.games import extraterrestrial_marauders as marauders
    from oracle import games as ogames
    art = levels.marauders_level(rows, cols)
    rngs = {}

    def make_world(e):                        # the env's stream continues across restarts
      rngs.setdefault(e, np.random.RandomState(900 + e))
      return ogames.make_marauders(art, rngs[e])
    games = [ss.lowered(marauders.make_game(art), pitch) for _ in range(_n_games(binding))]
    return Built(games, make_world, _draw(5, [.24, .24, .24, .24, .04], quit_action=4), 900,
                 STEPS)
  return build


def _shockwave_build(rows, cols, pitch, binding):
  def build():
    from pycolab_b200 import levels
    from pycolab_b200.games import shockwave
    from oracle import games as ogames
    n = _n_games(binding)
    arts = [levels.shockwave_level(rows + cols + i, rows, cols, 0.5) for i in range(n)]
    rngs = {}

    def make_world(e):
      rngs.setdefault(e, np.random.RandomState(700 + e))
      return ogames.make_shockwave(arts[e % n], rngs[e])
    games = [ss.lowered(shockwave.make_game(a), pitch) for a in arts]
    # no quit action: mostly north, for long enough to reach the goal row or be caught
    return Built(games, make_world, _draw(4, [.7, .1, .1, .1]), 700, rows + 8)
  return build


def _ordeal_build(pitch, binding):
  def build():
    from pycolab_b200.games import ordeal
    from oracle import games as ogames
    games = [ss.lowered(ordeal.make_cavern(), pitch) for _ in range(_n_games(binding))]
    return Built(games, lambda e: ogames.make_ordeal('cavern', ordeal.GAME_ART_CAVERN),
                 _draw(4, quit_action=4, quit_p=0.02), 0, STEPS)
  return build


def _compiled_sampler_build(pitch, binding):
  """tests/sprite_games.py's sampler: plain Sprites at row -1 and column -1 by turns (the
  layers kernel wraps them as the render does), a Scrolly and bit-row drapes."""
  def build():
    import registered_games as rg
    from oracle import compiled as ocompiled
    from pycolab_b200 import compiler
    mod = rg.load('sprite_games.py')
    compiler.register(*mod.CLASSES)
    try:
      games = [ss.lowered(mod.make_sampler(level), pitch) for level in range(_n_games(binding))]
    finally:
      compiler.unregister(*mod.CLASSES)
    n = len(games)
    return Built(games, lambda e: ocompiled.make_world(games[e % n]),
                 _draw(9, quit_action=8, quit_p=0.02), 0, STEPS)
  return build


def _bit_row_cases():
  out = []
  for rows, cols in [(32, 64), (32, 39), (16, 64), (20, 63)]:
    for j, pitch in enumerate(pitches(cols)):
      binding = (SHARED, PER_ENV)[j % 2]
      out.append(Case('marauders-%dx%d-p%d-%s' % (rows, cols, pitch, binding), 'marauders',
                      (rows, cols), pitch, binding, 'ok', None,
                      _marauders_build(rows, cols, pitch, binding)))
  for rows, cols in [(32, 64), (31, 33), (32, 15), (12, 32), (12, 17)]:
    for j, pitch in enumerate(pitches(cols)):
      binding = (POOL, SHARED, PER_ENV)[j % 3]
      out.append(Case('shockwave-%dx%d-p%d-%s' % (rows, cols, pitch, binding), 'shockwave',
                      (rows, cols), pitch, binding, 'ok', None,
                      _shockwave_build(rows, cols, pitch, binding)))
  for j, pitch in enumerate(pitches(15)):
    binding = (SHARED, PER_ENV, SHARED)[j]
    out.append(Case('ordeal-cavern-p%d-%s' % (pitch, binding), 'ordeal', (8, 15), pitch, binding,
                    'ok', None, _ordeal_build(pitch, binding)))
  for j, pitch in enumerate(pitches(8)):
    binding = (POOL, PER_ENV, POOL)[j]
    out.append(Case('compiled-sampler-p%d-%s' % (pitch, binding), 'compiled', (5, 8), pitch,
                    binding, 'ok', None, _compiled_sampler_build(pitch, binding)))
  return out


CASES = [c._replace(batch=_batch(i, c.binding))
         for i, c in enumerate(_scrolly_cases() + _bit_row_cases())]


# ------------------------------------------------------------- programs with host hooks
# (id, program, which hook the facade serves: 'curtain' (pcl_layers refuses the handle)
# or 'layers', build)
def _hook_build(program):
  def build():
    import random
    from oracle import games as ogames
    from pycolab_b200 import levels, lowering
    if program == 'warehouse':
      from pycolab_b200.games import warehouse_manager
      arts = [levels.warehouse_level(20, shape=(24, 31), num_boxes=4, num_goals=6),
              levels.warehouse_level(77, shape=(24, 31), num_boxes=4, num_goals=6)]
      return Built([lowering.lower(warehouse_manager.make_game(a)) for a in arts],
                   lambda e: ogames.make_warehouse(arts[e % 2]),
                   _draw(5, quit_action=5, quit_p=0.02), 0, 30)
    if program == 'aperture':
      from pycolab_b200.games import aperture
      art = levels.aperture_level()
      return Built([lowering.lower(aperture.make_game(art))], lambda e: ogames.make_aperture(art),
                   _draw(9, quit_action=9, quit_p=0.02), 0, 30)
    if program == 'hello':
      from pycolab_b200.games import hello_world
      art = hello_world.HELLO_ART
      return Built([lowering.lower(hello_world.make_game(art))], lambda e: ogames.make_hello(art),
                   _draw(4, quit_action=4, quit_p=0.03), 0, 30)
    if program == 't_maze':
      from oracle import t_maze as otm
      from pycolab_b200.games import t_maze
      cfg = (1, False, 40, 2, 3)
      arts = [levels.t_maze_level(2 + i) for i in range(2)]
      random.seed(0)
      games = [lowering.lower(t_maze.make_game(*cfg, maze_art=m, cue_art=c)) for m, c in arts]
      rngs = {}

      def make_world(e):
        rngs.setdefault(e, (random.Random(8 + e), np.random.RandomState(8 + e)))
        return otm.make_t_maze(*arts[e % 2], *cfg, rng=rngs[e][0], np_rng=rngs[e][1])
      moves = _draw(5, quit_action=5, quit_p=0.02)           # 1..5 move or stay, 6 quits
      return Built(games, make_world, lambda rs, T, B: moves(rs, T, B) + 1, 8, 30)
    from oracle import box_world as obw
    from pycolab_b200.games import box_world
    pool = [levels.box_world_level(i, 8) for i in range(3)]
    return Built([lowering.lower(box_world.game_from_level(a, d, 20)) for a, d in pool],
                 lambda e: obw.make_box_world(*pool[e % 3], 20),
                 lambda rs, T, B: rs.randint(-1, 5, size=(T, B)).astype(np.int32), 0, 30)
  return build


HOOK_CASES = [(p, hook, _hook_build(p)) for p, hook in
              [('warehouse', 'curtain'), ('aperture', 'curtain'), ('hello', 'curtain'),
               ('t_maze', 'layers'), ('box_world', 'layers')]]
