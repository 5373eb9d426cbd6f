"""extraterrestrial_marauders levels of any shape marauders_step accepts, scripted rim
cases, and a record of which edges an oracle run went through.  Shared by
test_marauders.py (oracle vs reference) and test_gpu_marauders.py (device vs oracle).

The stock layout keeps the marauders in rows 0-4, away from column 0, the bunkers on
rows 11-13 and P on the last row, so nothing there reaches the board's rim.  Here:
  * the marauders 'X' move as one curtain: every max(1, count // 8.0000001) frames they
    shift by dx, and when any of them is in column 0 or W-1 they first reverse and roll
    down one row (np.roll on axis 0, so row H-1 wraps to row 0).  On a board of one or
    two columns every move is such a reversal.  A marauder in row 10 ends the episode;
  * the up bolts 'a'-'d' and the down bolts 'y', 'z' are unconfined MazeWalkers: a bolt
    that leaves the board is invisible and fires again.  A bolt fired by P in row 0
    starts at row -1; a down bolt fired below a marauder in row H-1 starts at row H;
  * the drapes and bolts read the stale board: only the top bolt of a cell is a hitter,
    a bolt hides the marauder under it, and a down bolt's column is np.random.choice of
    the columns that show an 'X'.  With none showing, choice raises ValueError;
  * P is confined: a push out of the board leaves it in place.
"""

import numpy as np

from oracle import games as ogames
from rim_sweep import repitch

UP = 'abcd'
DOWN = 'yz'
BOLTS = UP + DOWN
SPRITES = 'P' + BOLTS


def board(shape, cells):
  """The art of an H x W board of ' ' with `cells` {char: [(row, col), ...]} drawn in."""
  H, W = shape
  art = np.full((H, W), ord(' '), np.uint8)
  for ch, where in cells.items():
    for rc in where:
      assert art[rc] == ord(' '), (ch, rc)
      art[rc] = ord(ch)
  return [bytes(row).decode('ascii') for row in art]


def open_level(seed, shape, n_marauders, n_bunkers=0, x_rows=None, b_rows=None,
               p_cell=None):
  """`n_marauders` 'X' in rows `x_rows` (default: every row but 10, where the episode
  would end at once), `n_bunkers` 'B' in rows `b_rows` (default: any row), and P at
  `p_cell` (default: anywhere left), all drawn from RandomState(seed)."""
  rs = np.random.RandomState(seed)
  H, W = shape
  x_rows = [r for r in range(H) if r != 10] if x_rows is None else list(x_rows)
  b_rows = range(H) if b_rows is None else b_rows
  taken = {} if p_cell is None else {tuple(p_cell): 'P'}

  def place(ch, rows, n):
    free = [(r, c) for r in rows for c in range(W) if (r, c) not in taken]
    assert len(free) >= n, (shape, ch, n)
    for i in rs.permutation(len(free))[:n]:
      taken[free[i]] = ch
  place('X', x_rows, n_marauders)
  place('B', b_rows, n_bunkers)
  if p_cell is None:
    place('P', range(H), 1)
  cells = {}
  for rc, ch in taken.items():
    cells.setdefault(ch, []).append(rc)
  return board(shape, cells)


# The board shapes the GPU sweep steps (rows 11..32, columns 1..64): one and two columns,
# each side of 16, 32 and 48 columns, and the largest boards.
SHAPES = [(11, 1), (11, 2), (12, 3), (13, 16), (11, 17), (16, 31), (15, 32), (12, 33),
          (20, 48), (32, 39), (16, 64), (20, 63), (31, 63), (32, 64)]
COUNTS = (1, 8, 9, 16, 17, 30)


def sweep_level(shape, seed):
  """The open level of a board shape: a marauder count from COUNTS (at least 2, at most
  half the cells of their rows) in rows 0-4 and below row 10, where they have the longest way to
  row 10; a few bunkers, and P, anywhere."""
  H, W = shape
  k = H + W + seed
  x_rows = [r for r in range(H) if r < 5 or r > 10]
  n = max(2, min(COUNTS[k % len(COUNTS)], len(x_rows) * W // 2))
  return open_level(seed + 10 * k, shape, n, min(4 + k % 5, H * W // 5), x_rows=x_rows)


def lowered(art, pitch=None):
  """The lowered facade game of `art`, its backdrop re-padded to `pitch` columns."""
  from pycolab_b200 import lowering
  from pycolab_b200.games import extraterrestrial_marauders as marauders
  return repitch(lowering.lower(marauders.make_game(art)), pitch)


def make_world(art, rng):
  """An oracle world drawing from `rng`, the stand-in for NumPy's global generator."""
  return ogames.make_marauders(art, rng)


def random_actions(rs, T, B, quit_p=0.01):
  """West (0), east (1), fire (2), nothing (3) and a rare quit (4)."""
  rest = (1.0 - quit_p) / 4
  return rs.choice(5, size=(T, B), p=[rest] * 4 + [quit_p]).astype(np.int32)


# ------------------------------------------------------------------ rim cases
# Edges (Edges.seen):
#   reverse             the marauders reversed and rolled down
#   wrap_roll           ... with a marauder in row H-1, which the roll carries to row 0
#   both_sides          marauders in column 0 and column W-1 at once (W > 1)
#   row10               a marauder reached row 10 and the episode ended
#   last_x_shot         the last marauder was shot, and a down bolt flew on in that frame
#   fire_row0           P fired from row 0: the new up bolt sits at row -1
#   push_w / push_e     P pushed against column 0 / column W-1 and stayed
#   up_off_top          a visible up bolt left the board by row 0
#   down_off_bottom     a visible down bolt left the board by row H-1
#   drop_off_board      a down bolt fired below a marauder in row H-1: it starts at row H
#   hidden_flies_on     two bolts in one cell over 'B' or 'X': the top one hit, the hidden
#                       one flew on
#   up_under_down       an up bolt under a down bolt on an 'X': no hit, the up bolt flew on
#   bunker_and_x        one bolt on a 'B' under an 'X': -1 and +10 in one frame
#   bolt_on_p           a down bolt on P's cell ended the episode
#   choice_1            a down bolt drew from one column (no draw consumed)
#   choice_2k1          ... from 2^k + 1 columns (3, 5, 9, 17 or 33: most draws rejected)
#   count_N             the level starts with N marauders (1, 8, 9, 16, 17: cadences 1, 1,
#                       1, 1, 2)
#   raise               play() raised ValueError: no column shows an 'X', because
#   raise_last_hit      ... the last marauder was hit in that frame, or
#   raise_hidden        ... every marauder left is hidden under a bolt
RIM = {
    # One column: every move reverses and rolls down; P pushes out at both sides at once.
    'one_column': ([' ', ' ', ' ', ' ', ' ', 'B', 'X', 'P', ' ', ' ', ' ', ' ', 'X'],
                   [0, 1, 3, 1],
                   {'reverse', 'push_w', 'push_e', 'choice_1', 'row10'}),
    # Two columns: marauders in both at once; P in row 0 fires a bolt from row -1.
    'two_columns': (['PX', 'X ', '  ', ' X', '  ', '  ', '  ', '  ', 'X ', '  ', '  ', ' B',
                     '  '],
                    [2, 0, 3, 1, 1],
                    {'reverse', 'both_sides', 'push_w', 'push_e', 'fire_row0', 'row10'}),
    # A marauder below row 10 rolls from row 12 to row 0; a down bolt fired below the
    # last row starts at row H, and one leaves the board by the last row.
    'wrap_roll': (['    X ', '      ', ' P    ', '      ', '      ', '      ', '      ',
                   '      ', 'B     ', '      ', '      ', '  X   ', '      '],
                  [1, 1, 0, 0, 0],
                  {'wrap_roll', 'drop_off_board', 'down_off_bottom'}),
    # One marauder, shot while a down bolt flies on; an up bolt leaves by row 0 first.
    'last_x_shot': (['       ', '       ', '       ', '       ', '     P ', '       ',
                     '       ', '       ', '       ', '       ', '       ', '    X  '],
                    [3, 2, 2, 2, 2, 2, 1, 1, 2],
                    {'count_1', 'last_x_shot', 'up_off_top', 'choice_1', 'wrap_roll'}),
    # P on row 0 pushes out at both sides and fires from there.
    'p_top_row': ([' BP', '   ', '   ', '   ', '   ', '   ', '   ', '   ', ' X ', '   ',
                   '   '],
                  [0, 2, 0, 0, 0, 2, 1],
                  {'fire_row0', 'push_w', 'push_e', 'down_off_bottom', 'row10'}),
    # A down bolt lands on P's cell.
    'bolt_on_p': (['B    ', 'B    ', '     ', '   X ', '     ', '   P ', '     ', '     ',
                   '   B ', '  X  ', '     ', '     ', '     '],
                  [2, 1, 3, 0, 3, 2],
                  {'bolt_on_p', 'down_off_bottom'}),
    # Two bolts in one cell over 'B' or 'X', and an up bolt under a down bolt on an 'X'.
    'stacked': (['  B', '   ', '  X', '   ', 'BXB', '   ', 'XXX', 'X  ', '   ', ' B ', ' P ',
                 ' B '],
                [1, 1, 0, 1, 2, 2, 0],
                {'hidden_flies_on', 'up_under_down', 'choice_2k1', 'both_sides'}),
    # A marauder moves over a bunker above row 10; one bolt there scores -1 and +10.
    'bunker_and_x': (['  B X', '     ', '  X  ', '   B ', 'X  PX', '   X ', '     ', '     ',
                      '     ', '     ', '     ', '   X '],
                     [0, 1, 2, 0],
                     {'bunker_and_x', 'both_sides'}),
    # 8, 9, 16 and 17 marauders: the cadence is 1 up to 16 and 2 from 17; the down bolts
    # draw from 3, 5, 9 or 17 columns on the way.
    'count_8': (['  X      ', '    X    ', ' B       ', '   X     ', '     X X ', 'X       X',
                 '         ', '   X     ', '         ', '         ', '        P'],
                [1, 3, 0, 1, 2, 0, 2, 0, 0, 0, 0, 2, 1, 0, 0, 0, 2, 0, 2, 0],
                {'count_8', 'both_sides', 'reverse', 'row10'}),
    'count_9': (['  X       ', '      X   ', 'B     X   ', '  B       ', '          ',
                 '    XX    ', '          ', '   XPX    ', '      X   ', '   X      ',
                 '          '],
                [1, 0, 2, 0, 2, 0, 1, 2, 0, 3, 2, 2, 1, 3, 1, 0, 2, 0, 2, 2],
                {'count_9', 'choice_2k1', 'bolt_on_p', 'row10'}),
    'count_16': (['    X              ', '                   ', 'XX                 ',
                  '     X             ', '             X   X ', 'X         XX X     ',
                  'X        X         ', '                   ', '                 X ',
                  '                   ', '                   ', '    X   X  B     X ',
                  '             P     '],
                 [0, 0, 2, 0, 1, 0, 2, 2, 0, 1, 0, 2, 1, 1, 1, 1, 2, 2, 0, 2],
                 {'count_16', 'choice_2k1', 'wrap_roll', 'row10'}),
    'count_17': (['     XX           ', ' XX  X            ', '                  ',
                  '         X        ', '  X          XX   ', '           B      ',
                  '        X       X ', '     X            ', '    B             ',
                  ' XX  X   X  X     ', '                  ', '       B    P     '],
                 [1, 3, 2, 0, 1, 0, 1, 1, 0, 3, 1, 2, 2, 2, 1, 1, 3, 0, 1, 1],
                 {'count_17', 'choice_2k1', 'reverse', 'row10'}),
    # The last marauder is hit while a down bolt waits to fire: no column shows an 'X'.
    'raise_last_hit': ([' X ', '   ', '   ', '   ', '   ', '  X', '  B', '   ', '   ', '   ',
                        '   ', '  P', '   '],
                       [2, 2, 3, 1, 1, 1, 0],
                       {'raise', 'raise_last_hit'}),
    # 'y' fires at its_showtime onto the cell the marauder moves to; at the next frame
    # it hides the only marauder, and 'z' has no column to draw from.
    'raise_hidden': (['X'] + [' '] * 10 + ['P'], [3],
                     {'raise', 'raise_hidden', 'count_1'}),
}
# The index of the script action whose play() raises ValueError.
RAISES = {'raise_last_hit': 6, 'raise_hidden': 0}


def _snapshot(world, out):
  th = world.things
  return dict(sprites={ch: (th[ch].row, th[ch].col, bool(th[ch].visible), th[ch].vrow,
                            th[ch].vcol) for ch in SPRITES},
              X=th['X'].curtain.copy(), B=th['B'].curtain.copy(), dx=th['X'].aux['dx'],
              board=np.array(out[0]), shot=world.plot.store.get('last_marauder_shot'))


class Edges(object):
  """Which edges one oracle world went through, step by step (the names above)."""

  def __init__(self):
    self.seen = set()

  def start(self, world, out):
    self.prev = _snapshot(world, out)
    self.seen.add('count_%d' % int(world.things['X'].curtain.sum()))   # no hits at frame 0
    self._now(world, self.prev)

  def step(self, world, out, action):
    now = _snapshot(world, out)
    prev = self.prev
    H, W = world.rows, world.cols
    ps, ns = prev['sprites'], now['sprites']
    if now['dx'] != prev['dx']:
      self.seen.add('reverse')
      if prev['X'][H - 1].any():
        self.seen.add('wrap_roll')
    if world.game_over and now['X'][10].any():
      self.seen.add('row10')
    if prev['X'].any() and not now['X'].any():
      moved = [ch for ch in DOWN if ps[ch][2] and ns[ch][3] == ps[ch][3] + 1]
      if moved:
        self.seen.add('last_x_shot')
    p_prev = ps['P']
    if action == 0 and p_prev[1] == 0:
      self.seen.add('push_w')
    if action == 1 and p_prev[1] == W - 1:
      self.seen.add('push_e')
    for ch in UP:
      if not ps[ch][2] and not ns[ch][2] and ns[ch][3:] == (-1, p_prev[1]) and \
          ps[ch][3:] != ns[ch][3:] and p_prev[0] == 0:
        self.seen.add('fire_row0')
      if ps[ch][2] and ps[ch][0] == 0 and not ns[ch][2] and ns[ch][3] == -1 and \
          ns[ch][4] == ps[ch][4]:
        self.seen.add('up_off_top')
    for ch in DOWN:
      if ps[ch][2] and ps[ch][0] == H - 1 and not ns[ch][2] and ns[ch][3] == H:
        self.seen.add('down_off_bottom')
      if not ns[ch][2] and ns[ch][3] == H and ps[ch][3:] != ns[ch][3:]:
        self.seen.add('drop_off_board')
    # Bolts stacked on the stale board: the top one (last in z-order) is the hitter.
    cells = {}
    for ch in BOLTS:
      if ps[ch][2]:
        cells.setdefault(ps[ch][:2], []).append(ch)
    for rc, chs in cells.items():
      if len(chs) < 2:
        continue
      top, hidden = chs[-1], chs[:-1]
      target = prev['B'][rc] or (prev['X'][rc] and top in UP)
      if target and ns[top][3:] == (-1, -1) and any(ns[h][3:] != (-1, -1) for h in hidden):
        self.seen.add('hidden_flies_on')
      if prev['X'][rc] and not prev['B'][rc] and top in DOWN and \
          any(h in UP and ns[h][3] == ps[h][3] - 1 for h in hidden):
        self.seen.add('up_under_down')
    for ch in BOLTS:
      rc = ps[ch][:2]
      if ps[ch][2] and (rc not in cells or cells[rc][-1] == ch) and ch in UP and \
          prev['B'][rc] and prev['X'][rc] and not now['B'][rc] and out[1] is not None:
        self.seen.add('bunker_and_x')
    if world.game_over:
      for ch in DOWN:
        if ps[ch][2] and ps[ch][:2] == ns['P'][:2]:
          self.seen.add('bolt_on_p')
    if now['shot'] != prev['shot']:
      n = int(np.count_nonzero((prev['board'] == ord('X')).any(axis=0)))
      if n == 1:
        self.seen.add('choice_1')
      if n in (3, 5, 9, 17, 33):
        self.seen.add('choice_2k1')
    self.prev = now
    self._now(world, now)

  def on_raise(self, world):
    """play() raised ValueError: which way no column came to show an 'X'."""
    self.seen.add('raise_hidden' if world.things['X'].curtain.any() else 'raise_last_hit')

  def _now(self, world, snap):
    X = snap['X']
    if world.cols > 1 and X[:, 0].any() and X[:, -1].any():
      self.seen.add('both_sides')


# ------------------------------------------------ the block's shared memory
# Mirrors marauders.cu (s_rec, launch) and the bound pcl_create applies.
WARPS_PER_BLOCK = 4
STATIC_SMEM = WARPS_PER_BLOCK * 96 * 4      # s_rec: 96 record words per warp


def block_smem(H, pitch):
  """Static records plus one staged H x pitch tile per warp."""
  return STATIC_SMEM + WARPS_PER_BLOCK * H * pitch
