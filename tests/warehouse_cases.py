"""Warehouse levels that reach the board's rim, scripted rim cases, and a record of which
edges an oracle run went through.  Shared by test_warehouse.py (oracle vs reference) and
test_gpu_warehouse.py (device vs oracle).

The generated levels of `levels.warehouse_level` keep a '.' border and a '#' ring around
the floor, so no box or player ever reaches the rim.  The levels here have floor up to
the edge:
  * boxes and P are unconfined MazeWalkers: one that leaves the board is invisible and
    sits at position (0, 0), where the judge marks an off-board box ('X' on a goal);
  * every box at (0, 0) looks at the same neighbour of P, so several move at once;
  * BoxSprite.update reads layers['P'][row -+ 1, col -+ 1] with NumPy's index rules: a
    box on row 0 sees P on the last row (-1 wraps), and a box on the last row or
    column raises IndexError for action 0 or 2 wherever P is.
"""

import numpy as np

from oracle import games as ogames

BOX_ORDER = '1234567890'
# Box characters by count, with gaps in the update order ('3', '7', '0').
BOX_SETS = {1: '0', 2: '37', 3: '370', 7: '1345780', 10: '1234567890'}


def ceil16(x):
  return (x + 15) // 16 * 16


def open_level(seed, shape, boxes, num_goals=None, wall_density=0.06):
  """Floor up to the edge with scattered walls, a goal '_' at (0, 0) and `num_goals`
  more, and the boxes `boxes` and P in rows 1..H-2 and columns 1..W-2 (no box starts
  where its first look-up raises)."""
  rs = np.random.RandomState(seed)
  H, W = shape
  num_goals = len(boxes) + 1 if num_goals is None else num_goals
  art = np.full((H, W), ord(' '), np.uint8)
  art[rs.random_sample((H, W)) < wall_density] = ord('#')
  inner = [(r, c) for r in range(1, H - 1) for c in range(1, W - 1)]
  picks = [inner[i] for i in rs.permutation(len(inner))[:len(boxes) + 1]]
  for ch, rc in zip(boxes + 'P', picks):
    art[rc] = ord(ch)
  art[0, 0] = ord('_')
  free = np.argwhere((art == ord(' ')) | (art == ord('#')))
  for rc in free[rs.permutation(len(free))[:num_goals]]:
    art[tuple(rc)] = ord('_')
  return [bytes(row).decode('ascii') for row in art]


def lowered(art, beneath=' ', pitch=None):
  """The lowered facade game of `art`, its backdrop re-padded to `pitch` columns."""
  from pycolab_b200 import lowering
  from pycolab_b200.games import warehouse_manager
  low = lowering.lower(warehouse_manager.make_game(art, beneath))
  if pitch is not None:
    backdrop = np.zeros((low.rows, pitch), dtype=np.uint8)
    backdrop[:, :low.cols] = low.backdrop[:, :low.cols]
    low.backdrop, low.pitch = backdrop, pitch
  return low


def random_actions(rs, T, B, quit_p=0.02):
  """Walks and pushes (0-3), no-ops (4) and a rare quit (5)."""
  rest = (1.0 - quit_p - 0.05) / 4
  return rs.choice(6, size=(T, B), p=[rest] * 4 + [0.05, quit_p]).astype(np.int32)


# ------------------------------------------------------------------ rim cases
# name -> (art, what_lies_beneath, script, edges the script must reach).  Edges:
#   box_off       a box is off the board
#   x_off         an off-board box on the goal at (0, 0) is drawn as 'X'
#   multi_push    two or more boxes moved in one step
#   wrap_push     a box on row 0 (or column 0) was pushed by P on the last row (column)
#   shared_cell   two visible boxes stand in one cell
#   player_off    P is off the board
#   showtime_over the episode ended at its_showtime
#   raise         play() raised IndexError (a RAISES entry gives the step)
RIM = {
    # The issue's art: P pushes '1' off the board from the goal at (0, 0).
    'push_off_goal': (['_ 1  ', '  P  ', ' 2   ', '    _'], ' ',
                      [0, 3, 2, 1, 2, 0, 0, 1, 1, 3, 3], {'box_off', 'x_off', 'player_off'}),
    # '1' leaves from plain floor: nothing is drawn at (0, 0), P walks onto it, then
    # pushes the off-board box again from (1, 0).
    'push_off_walk_over': (['  1  ', '  P  ', ' 2  _', '     '], ' ',
                           [0, 2, 2, 1, 0, 1, 3, 3], {'box_off'}),
    # A box on row 0 and P on the last row: action 1 pushes the box south, P walks off.
    'wrap_push_rows': ([' 1  ', '    ', '_   ', ' P  '], ' ',
                       [1, 0, 1, 0, 2, 0], {'wrap_push', 'player_off'}),
    # The same across the columns: action 3 with the box in column 0, P in the last one.
    'wrap_push_cols': (['1   P', '    _', '     '], ' ',
                       [3, 2, 1, 2, 2, 0], {'wrap_push', 'player_off'}),
    # P leaves the board and comes back.
    'player_returns': (['  1 ', 'P   ', '   _'], ' ',
                       [2, 2, 3, 3, 0, 3, 1, 1, 1, 0], {'player_off'}),
    # Two boxes off the board at once, then both pushed back from the last row together.
    'two_off_back_together': (['1 2  ', 'P    ', '     ', '    _'], ' ',
                              [0, 1, 3, 3, 0, 1, 2, 2, 1, 1, 1, 0, 0],
                              {'box_off', 'multi_push', 'wrap_push', 'player_off'}),
    # Both boxes leave through one cell, so they share a virtual position: they come back
    # onto one cell together (the later box is drawn on top) and leave together again.
    'two_share_virtual_cell': (['  1  ', '  P  ', '     ', '  2  ', '    _'], ' ',
                               [0, 3, 1, 1, 1, 1, 2, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 1, 0,
                                0, 0, 0, 3, 3, 0],
                               {'box_off', 'multi_push', 'wrap_push', 'shared_cell',
                                'player_off'}),
    # Ten boxes: '6' and '5' leave, then P pushes '1' and both off-board boxes at once.
    'ten_boxes_top_row': (['1234567890 ', '     P     ', '_          '], ' ',
                          [0, 1, 2, 0, 1, 2, 2, 2, 2, 0, 1, 1], {'box_off', 'multi_push'}),
    # One box, '0', pushed off onto the goal at (0, 0) and left there.
    'one_box': (['_ 0  ', '  P  ', '    _'], ' ', [0, 1, 2, 2, 0, 0], {'box_off', 'x_off'}),
    # Boxes '3', '7' and '0' (gaps in the update order) on the rim.
    'gapped_boxes': (['3  7  ', ' P   _', '0     ', '     _'], ' ',
                     [2, 0, 1, 3, 3, 3, 0, 1, 2, 2, 2, 0], {'box_off', 'multi_push'}),
    # Every sprite stands on a goal: the judge ends the episode at its_showtime.
    'beneath_goal': (['  1 ', 'P   ', ' 2  '], '_', [0, 1, 2], {'showtime_over'}),
    # A box on the last row raises at the first action 0, wherever P is.
    'raise_last_row': (['    ', ' P  ', '_   ', ' 1  '], ' ', [3, 2, 0, 1], {'raise'}),
    # P pushes a box into the last column; the next action 2 raises.
    'raise_last_col': (['_   ', ' P1 ', '    '], ' ', [1, 0, 3, 2, 2], {'raise'}),
}
# The step (index into the script) whose action raises.
RAISES = {'raise_last_row': 2, 'raise_last_col': 3}


def rim_boxes(name):
  art = ''.join(RIM[name][0])
  return ''.join(c for c in BOX_ORDER if c in art)


def make_world(art, beneath=' '):
  return ogames.make_warehouse(art, beneath)


def _snapshot(world):
  return {ch: (w.row, w.col, bool(w.visible), w.vrow, w.vcol)
          for ch, w in world.things.items() if ch != 'X'}


class Edges(object):
  """Which edges one oracle world went through, step by step (`RIM`'s names)."""

  def __init__(self, boxes):
    self.boxes = boxes
    self.seen = set()

  def start(self, world):
    self.prev = _snapshot(world)
    if world.game_over:
      self.seen.add('showtime_over')
    self._now(world)

  def step(self, world, action):
    now = _snapshot(world)
    H, W = world.rows, world.cols
    moved = [b for b in self.boxes if now[b][3:] != self.prev[b][3:]]
    if len(moved) > 1:
      self.seen.add('multi_push')
    p = self.prev['P']
    for b in moved:
      row, col = self.prev[b][:2]
      if (action == 1 and row == 0 and p[2] and p[0] == H - 1) or (
          action == 3 and col == 0 and p[2] and p[1] == W - 1):
        self.seen.add('wrap_push')
    self.prev = now
    self._now(world)

  def _now(self, world):
    s = self.prev
    if not s['P'][2]:
      self.seen.add('player_off')
    off = [b for b in self.boxes if not s[b][2]]
    if off:
      self.seen.add('box_off')
      if world.backdrop[0, 0] == ord('_') and world.board[0, 0] == ord('X') and not any(
          s[b][2] and s[b][:2] == (0, 0) for b in self.boxes):
        self.seen.add('x_off')
    cells = [s[b][:2] for b in self.boxes if s[b][2]]
    if len(set(cells)) < len(cells):
      self.seen.add('shared_cell')


def oracle_run(art, beneath, actions, boxes):
  """Play `actions` on oracle worlds with auto-reset.  Returns (edges seen, restarts, the
  step whose action raised IndexError or None)."""
  edges = Edges(boxes)
  world = make_world(art, beneath)
  world.its_showtime()
  edges.start(world)
  restarts = 0
  for t, a in enumerate(actions):
    if world.game_over:
      restarts += 1
      world = make_world(art, beneath)
      world.its_showtime()
      edges.start(world)
      continue
    try:
      world.play(int(a))
    except IndexError:
      edges.seen.add('raise')
      return edges.seen, restarts, t
    edges.step(world, int(a))
  return edges.seen, restarts, None
