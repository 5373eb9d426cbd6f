"""Seeded synthetic level generators for the benchmark configurations.

The reference ships only small hand-drawn levels (scrolly_maze 10x30 board over
a 45x89 world, warehouse 11x10..11x13, marauders 16x39; see
examples/scrolly_maze.py:45-195, warehouse_manager.py:42-80,
extraterrestrial_marauders.py:40-55).  BASELINE.json's configs ask for 64x64 and
80x80 boards, so these generators produce ASCII art in the SAME vocabulary as
the reference art (same characters, same invariants) that feeds the reference,
the oracle and the device engine alike.  All randomness is
`numpy.random.RandomState(seed)` (stream frozen by NumPy policy).
"""

import numpy as np


def _to_art(arr):
  return [bytes(row).decode('ascii') for row in arr]


def scrolly_maze_level(seed, world_shape=(129, 129), board_shape=(64, 64),
                       coin_density=0.08, star_density=0.08, extra_doors=0.06):
  """A scrolly_maze level: (maze_art, board_art, what_lies_beneath_mark).

  Invariants kept from examples/scrolly_maze.py:45-60: solid outer wall (the
  player cannot escape), exactly one each of 'P', 'a', 'b', 'c' and '+', the
  board window anchored at '+' lies inside the world.  The maze is a spanning
  tree carved over the odd-coordinate lattice with a fraction `extra_doors` of
  the remaining interior walls knocked out so patrollers have room to roam.
  """
  rs = np.random.RandomState(seed)
  WH, WW = world_shape
  BH, BW = board_shape
  assert WH % 2 == 1 and WW % 2 == 1 and WH >= BH and WW >= BW
  art = np.full((WH, WW), ord('#'), dtype=np.uint8)
  nr, nc = WH // 2, WW // 2                 # lattice rooms at (2i+1, 2j+1)
  visited = np.zeros((nr, nc), dtype=bool)
  stack = [(int(rs.randint(nr)), int(rs.randint(nc)))]
  visited[stack[0]] = True
  art[2 * stack[0][0] + 1, 2 * stack[0][1] + 1] = ord(' ')
  steps = ((-1, 0), (1, 0), (0, -1), (0, 1))
  while stack:
    r, c = stack[-1]
    options = [(r + dr, c + dc, dr, dc) for dr, dc in steps
               if 0 <= r + dr < nr and 0 <= c + dc < nc
               and not visited[r + dr, c + dc]]
    if not options:
      stack.pop()
      continue
    r2, c2, dr, dc = options[int(rs.randint(len(options)))]
    visited[r2, c2] = True
    art[2 * r + 1 + dr, 2 * c + 1 + dc] = ord(' ')
    art[2 * r2 + 1, 2 * c2 + 1] = ord(' ')
    stack.append((r2, c2))
  # Extra doors: interior walls between two rooms (one odd, one even coord).
  rr, cc = np.meshgrid(np.arange(1, WH - 1), np.arange(1, WW - 1), indexing='ij')
  door = ((rr % 2) != (cc % 2)) & (art[1:-1, 1:-1] == ord('#'))
  door &= rs.random_sample(door.shape) < extra_doors
  art[1:-1, 1:-1][door] = ord(' ')

  # Board window: '+' sits on an (even, even) lattice point, always a wall.
  cr = 2 * int(rs.randint(0, (WH - BH) // 2 + 1))
  cc0 = 2 * int(rs.randint(0, (WW - BW) // 2 + 1))
  cr, cc0 = min(cr, WH - BH), min(cc0, WW - BW)
  cr -= cr % 2
  cc0 -= cc0 % 2

  floor = np.argwhere(art == ord(' '))
  def pick(pred):
    cand = floor[[bool(pred(r, c)) for r, c in floor]]
    r, c = cand[int(rs.randint(len(cand)))]
    return int(r), int(c)
  taken = set()
  def place(ch, pred):
    while True:
      pos = pick(pred)
      if pos not in taken:
        taken.add(pos)
        return pos
  # Player well inside the initial window; patrollers anywhere in the window's
  # neighbourhood (they may start off-board, as in the reference's Maze #0).
  inner = lambda r, c: (cr + BH // 4 <= r < cr + BH - BH // 4 and
                        cc0 + BW // 4 <= c < cc0 + BW - BW // 4)
  near = lambda r, c: (cr - 8 <= r < cr + BH + 8 and cc0 - 8 <= c < cc0 + BW + 8)
  spots = {'P': place('P', inner)}
  for ch in 'abc':
    spots[ch] = place(ch, near)
  coins = rs.random_sample(len(floor)) < coin_density
  for (r, c), is_coin in zip(floor, coins):
    if is_coin and (int(r), int(c)) not in taken:
      art[r, c] = ord('@')
  for ch, (r, c) in spots.items():
    art[r, c] = ord(ch)
  art[cr, cc0] = ord('+')

  stars = np.full((BH, BW), ord(' '), dtype=np.uint8)
  stars[rs.random_sample((BH, BW)) < star_density] = ord('.')
  return _to_art(art), _to_art(stars), '#'


def warehouse_level(seed, shape=(80, 80), num_boxes=10, num_goals=12,
                    wall_density=0.10):
  """A warehouse_manager level (art only; every sprite stands on ' ').

  Invariants from examples/warehouse_manager.py:42-80,203-226: a '.' border of
  width >= 1 around a '#' wall ring (so the BoxSprite's layers['P'][r±1, c±1]
  look-ups stay in bounds), boxes '0'..'9' each at most once, one 'P', goals
  '_' >= boxes so the puzzle is not trivially unsolvable by count.
  """
  rs = np.random.RandomState(seed)
  H, W = shape
  assert 1 <= num_boxes <= 10 and H >= 8 and W >= 8
  art = np.full((H, W), ord('.'), dtype=np.uint8)
  art[1:H - 1, 1:W - 1] = ord('#')
  art[2:H - 2, 2:W - 2] = ord(' ')
  inner = art[2:H - 2, 2:W - 2]
  inner[rs.random_sample(inner.shape) < wall_density] = ord('#')
  floor = np.argwhere(art == ord(' '))
  order = rs.permutation(len(floor))
  need = num_goals + num_boxes + 1
  assert len(floor) >= need
  picks = floor[order[:need]]
  k = 0
  for _ in range(num_goals):
    art[tuple(picks[k])] = ord('_'); k += 1
  for b in '1234567890'[:num_boxes]:
    art[tuple(picks[k])] = ord(b); k += 1
  art[tuple(picks[k])] = ord('P')
  return _to_art(art)


def marauders_level(rows=16, cols=39):
  """The marauders layout (extraterrestrial_marauders.py:40-55) generated
  procedurally: five staggered rows of 'X' every 4th column, four 4x3 bunkers
  on rows 11-13, the player two cells in on the last row."""
  assert rows >= 16 and cols >= 39
  art = np.full((rows, cols), ord(' '), dtype=np.uint8)
  for r in range(5):
    start = 4 if r % 2 == 0 else 5
    for i in range(8):
      art[r, start + 4 * i] = ord('X')
  for b in range(4):
    art[11:14, 4 + 9 * b: 8 + 9 * b] = ord('B')
  art[rows - 1, 2] = ord('P')
  return _to_art(art)


def classic_level(kind):
  """A second, larger level for each `examples/classics` game (the stock art is
  the only one the reference ships; the rules read only the board shape and,
  for four_rooms, the fixed goal cell (4, 3) — four_rooms.py:78)."""
  if kind == 'four_rooms':
    rows, cols = 15, 21
    a = np.full((rows, cols), ord(' '), dtype=np.uint8)
    a[0, :] = a[-1, :] = a[:, 0] = a[:, -1] = ord('#')
    a[:, 10] = ord('#')
    a[7, :] = ord('#')
    for r, c in ((3, 10), (11, 10), (7, 4), (7, 15)):   # doors
      a[r, c] = ord(' ')
    a[2, 7] = ord('P')
    return _to_art(a)
  if kind == 'cliff_walk':
    a = np.full((6, 20), ord('.'), dtype=np.uint8)
    a[5, 0] = ord('P')
    return _to_art(a)
  if kind == 'chain_walk':
    a = np.full((1, 40), ord('.'), dtype=np.uint8)
    a[0, 17] = ord('P')
    return _to_art(a)
  raise ValueError(kind)


def fluvial_level(rows=7, cols=40, seed=0):
  """A second river for `examples/fluvial_natation.py` (the rules flow rows 1..3
  whatever the size, fluvial_natation.py:106-110)."""
  rs = np.random.RandomState(seed)
  a = np.full((rows, cols), ord(' '), dtype=np.uint8)
  a[0, :] = a[-1, :] = ord('=')
  waves = rs.random_sample((rows - 2, cols)) < 0.15
  a[1:-1][waves] = rs.choice([ord(c) for c in '.,`:~'], size=int(waves.sum()))
  a[3, cols // 3] = ord('P')
  return _to_art(a)


def aperture_level():
  """A small `examples/aperture.py` level: an ooze moat between the player and
  the cranachan, special walls '@' on both sides to shoot apertures into."""
  return ['###############',
          '#@           @#',
          '#  A   ..     #',
          '#      ..     #',
          '#@     ..    @#',
          '#      ..  C  #',
          '###@###..##@###',
          '###############']


def shockwave_level(seed, height=12, width=15, safety_density=0.15):
  """A shockwave level in the vocabulary of examples/shockwave.py:40-88: a '^' safe row
  on top, ' ' exposed cells, '+' bunkers, '=' wall runs on non-adjacent interior rows
  (never the bottom row, always leaving gaps), one 'P' on the bottom row.  Same
  ingredients as the reference's `random_level`, drawn from a private
  RandomState(seed) (that function itself no longer runs: it uses `np.bool`)."""
  rs = np.random.RandomState(seed)
  level = np.full((height, width), ord(' '), dtype=np.uint8)
  level[rs.random_sample(level.shape) < safety_density] = ord('+')
  rows = set(range(1, height - 1))
  while rows:
    row = int(rs.choice(sorted(rows)))
    n_walls = int(rs.randint(2, max(3, width - 3)))
    mask = np.zeros((width,), dtype=bool)
    mask[:n_walls] = True
    rs.shuffle(mask)
    level[row, mask] = ord('=')
    rows -= {row - 1, row, row + 1}
  level[-1, int(rs.randint(0, width - 1))] = ord('P')
  level[0] = ord('^')
  return _to_art(level)


def t_maze_level(seed=0, shape=(77, 191)):
  """A research/lp-rnn/t_maze.py world: (maze_art, cue_art).

  The drapes hard-code where things are (t_maze.py:407-415), so the generator keeps those
  constants and draws the rest: the start room with the teleporter on row 4 and the board
  corner '+' at (3, 89) (the 7 x 11 board shows the room), the limbo cell (4, 140) walled
  in on all eight sides, and for every level L a T-maze whose hallway row 13 + 11 L lies
  dy = 11 L + 9 rows below the teleporter and the limbo cell, centred on column 94 = 140 - 46
  with goal pads 'l' / 'r' at the ends of two corridors.  The half-width of each level's
  hallway grows with L and is drawn from RandomState(seed); everything else is dirt '*'.
  The cue is 'Q' blocks in the bottom rows, on both sides of the board."""
  rs = np.random.RandomState(seed)
  rows, cols = shape
  assert rows >= 11 * 5 + 9 + 5 + 8 and cols >= 191
  art = np.full((rows, cols), ord('*'), dtype=np.uint8)
  art[:10] = ord(' ')
  art[3:8, 92:97] = ord('#')                        # start room, teleporter row 4
  art[4:7, 93:96] = ord(' ')
  art[4, 93:96] = ord('t')
  art[6, 94] = ord('P')
  art[3, 89] = ord('+')
  art[3:6, 139:142] = ord('#')                      # limbo cell (4, 140)
  art[4, 140] = ord(' ')
  centre = 140 - 46
  widths = (8, 13, 20, 33, 53, 88)
  for level, base in enumerate(widths):
    h = min(base + int(rs.randint(0, 4)), centre - 1, cols - centre - 2)
    y = 12 + 11 * level
    west, east = centre - h, centre + h
    art[y:y + 8, west:east + 1] = ord('#')
    art[y + 1:y + 3, west + 1:east] = ord(' ')      # the hallway
    art[y + 3:y + 6, west + 1:west + 4] = ord(' ')  # the corridors
    art[y + 3:y + 6, east - 3:east] = ord(' ')
    art[y + 6, west + 1:west + 4] = ord('l')
    art[y + 6, east - 3:east] = ord('r')
    art[y + 4:y + 7, west + 5:east - 4] = ord('*')
  cue = np.full((7, 11), ord(' '), dtype=np.uint8)
  block = 1 + int(rs.randint(0, 3))                 # 1-3 columns on each side
  first = 7 - (2 + int(rs.randint(0, 3)))
  cue[first:, :block] = ord('Q')
  cue[first:, 11 - block:] = ord('Q')
  return _to_art(art), _to_art(cue)


BOX_WORLD_KEYS = 'abcdefghijklmnopqrst'      # research/box_world: 20 colours, key 'a' opens 'A'
BOX_WORLD_LOCKS = BOX_WORLD_KEYS.upper()


def _box_world_problem(rand, solution_lengths, num_forward, num_backward, branch_length):
  """The box graph: solution length and (lock, key) id pairs.  Id 0 is "no lock" (the
  boxes on the floor), id -1 the gem; ids 1 .. n name colours of the shuffled palette.
  Rows past the solution length are distractor branches."""
  n = rand.choice(solution_lengths)
  forward = rand.choice(num_forward)
  backward = rand.choice(num_backward)
  pairs = [(i, i + 1) for i in range(n)] + [(n, -1)]
  for _ in range(forward):
    lock = rand.choice(range(1, n + 1))
    for _ in range(branch_length):
      key = None
      while key is None or key == lock:
        key = rand.choice(range(n + 1, len(BOX_WORLD_KEYS)))
      pairs.append((lock, key))
      lock = key
  for _ in range(backward):              # backward branches ignore branch_length
    key = rand.choice(range(1, n + 1))
    lock = rand.choice(range(n + 1, len(BOX_WORLD_KEYS)))
    pairs.append((lock, key))
  return n, pairs


def _box_world_attempt(rand, grid_size, solution_lengths, num_forward, num_backward,
                       branch_length, max_tries=200):
  """One generation attempt, or None when it ran out of placement tries."""
  n, pairs = _box_world_problem(rand, solution_lengths, num_forward, num_backward,
                                branch_length)
  palette = list(range(len(BOX_WORLD_KEYS)))
  rand.shuffle(palette)
  size = grid_size + 2
  art = np.full((size, size), ord(' '), dtype=np.uint8)
  art[0, :] = art[-1, :] = art[:, 0] = art[:, -1] = ord('#')
  distractors = []
  tries = 0

  def room_for_box(x, y):               # the box and its lock, with a free ring around both
    return (art[y - 1:y + 2, x - 1:x + 3] == ord(' ')).all()

  for i, (lock, key) in enumerate(pairs):
    while True:
      if tries > max_tries:
        return None
      x = rand.randint(0, grid_size - 3) + 1
      y = rand.randint(1, grid_size - 1) + 1
      if room_for_box(x, y):
        break
      tries += 1
    art[y, x] = ord('*') if key == -1 else ord(BOX_WORLD_KEYS[palette[key - 1]])
    if lock != 0:
      art[y, x + 1] = ord(BOX_WORLD_LOCKS[palette[lock - 1]])
      if i > n:
        distractors.append((x + 1, y))
  while True:
    if tries > max_tries:
      return None
    x = rand.randint(0, grid_size - 1) + 1
    y = rand.randint(1, grid_size - 1) + 1
    if art[y, x] == ord(' '):
      break
    tries += 1
  art[y, x] = ord('.')
  return _to_art(art), distractors


def box_world_level(seed, grid_size=12, solution_length=(1, 2, 3, 4),
                    num_forward=(0, 1, 2, 3, 4), num_backward=(0,), branch_length=1):
  """A research/box_world level: (art, distractors).

  `seed` is an int or a `np.random.RandomState`, which the generator continues.  It makes
  the draws of research/box_world/box_world.py's `make_game` in the same order — the
  problem's `choice`s, the `shuffle` of the 20 key / lock colours, the `randint`
  placements and both retry loops — so RandomState(s) gives the level that upstream
  builds from RandomState(s).  The art is (grid_size + 2)² with a '#' wall, the player
  '.', keys 'a'-'t', locks 'A'-'T' right of the box they close, and the gem '*';
  `distractors` lists the (column, row) of every lock that ends the episode."""
  rand = seed if isinstance(seed, np.random.RandomState) else np.random.RandomState(seed)
  for _ in range(200):
    level = _box_world_attempt(rand, grid_size, solution_length, num_forward, num_backward,
                               branch_length)
    if level is not None:
      return level
  raise RuntimeError('Could not generate game in MAX_GENERATION_TRIES tries.')


def cued_catch_art(rows=7, cols=12, player=(1, 3), balls=((1, 8), (2, 8)), cue_cells=()):
  """A research/lp-rnn/cued_catch.py board of `rows` x `cols` (the device takes up to
  32 x 64): the player 'P' and the balls 'a' / 'b' at the given cells, and 'Q' at
  `cue_cells`.  The defaults are the reference's 7 x 12 layout.  The player only moves
  between rows 1 and 2 (cued_catch.py:138-141), and a ball left of the player's column
  is put back at its start (:190-192)."""
  art = np.full((rows, cols), ord(' '), dtype=np.uint8)
  for r, c in cue_cells:
    art[r, c] = ord('Q')
  art[player] = ord('P')
  art[balls[0]] = ord('a')
  art[balls[1]] = ord('b')
  return _to_art(art)


def sequence_recall_art(rows=17, cols=21):
  """A research/lp-rnn/sequence_recall.py board of `rows` x `cols` (9 x 9 up to 32 x 64):
  a '#' ring, the player 'P' in the middle inside a 3 x 3 start box '%', and the four light
  pads, each one step past a free cell from the box: '2' above, '4' below, '1' left and '3'
  right of it.  Moving straight from the player's start enters a pad in three steps."""
  assert 9 <= rows and 9 <= cols
  cr, cc = rows // 2, cols // 2
  art = np.full((rows, cols), ord(' '), dtype=np.uint8)
  art[0, :] = art[-1, :] = art[:, 0] = art[:, -1] = ord('#')
  w = min(3, cc - 2)
  art[1:cr - 2, cc - w:cc + w + 1] = ord('2')
  art[cr + 3:rows - 1, cc - w:cc + w + 1] = ord('4')
  art[cr - 1:cr + 2, 1:cc - 2] = ord('1')
  art[cr - 1:cr + 2, cc + 3:cols - 1] = ord('3')
  art[cr - 1:cr + 2, cc - 1:cc + 2] = ord('%')
  art[cr, cc] = ord('P')
  return _to_art(art)
