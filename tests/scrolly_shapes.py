"""scrolly_maze at board shapes the generated levels cannot reach.

`levels.scrolly_maze_level` carves a lattice maze and puts the player in the inner half
of the first window, which needs boards of a few lattice cells each way.  The step
kernel's shared-memory layout changes with the board shape (segments per row, W
against 32 and 64, H against 32 and 64, pitch against ceil16(W)), down to a one-column
board, so these helpers build open levels of any shape, the facade game with any
scroll margins, and a Python model of the kernel's per-warp shared-memory layout.
"""

import numpy as np

from oracle import games as ogames
from rim_sweep import MAX_BLOCK_SMEM, ceil16, repitch


def open_level(seed, board_shape, world_shape, corner=None, wall_density=0.12,
               coin_density=0.15, star_density=0.1):
  """(maze_art, board_art, '#'): a walled world with sparse inner walls and coins, the
  board window's corner '+' at `corner` (default: random), the player inside the first
  window, patrollers anywhere on the floor."""
  rs = np.random.RandomState(seed)
  WH, WW = world_shape
  BH, BW = board_shape
  assert WH >= BH + 2 and WW >= BW + 2
  art = np.full((WH, WW), ord(' '), dtype=np.uint8)
  art[rs.random_sample((WH, WW)) < wall_density] = ord('#')
  art[0, :] = art[-1, :] = art[:, 0] = art[:, -1] = ord('#')
  if corner is None:
    corner = (int(rs.randint(1, WH - BH)), int(rs.randint(1, WW - BW)))
  cr, cc = corner
  assert 1 <= cr <= WH - BH - 1 and 1 <= cc <= WW - BW - 1
  taken = {(cr, cc)}

  def place(ch, r0, r1, c0, c1):
    while True:
      r, c = int(rs.randint(r0, r1)), int(rs.randint(c0, c1))
      if (r, c) not in taken:
        taken.add((r, c))
        art[r, c] = ord(ch)
        return

  place('P', cr, cr + BH, cc, cc + BW)
  for ch in 'abc':
    place(ch, 1, WH - 1, 1, WW - 1)
  floor = art == ord(' ')
  art[floor & (rs.random_sample((WH, WW)) < coin_density)] = ord('@')
  art[cr, cc] = ord('+')
  stars = np.full((BH, BW), ord(' '), dtype=np.uint8)
  stars[rs.random_sample((BH, BW)) < star_density] = ord('.')
  to_art = lambda a: [bytes(row).decode('ascii') for row in a]
  return to_art(art), to_art(stars), '#'


DEFAULT_MARGINS = ((2, 3), (2, 3))
NO_MARGINS = (None, None)

# (id, board shape, world shape, margins of '#' and '@'): the board shapes the kernel
# branches on.  1 segment per row (4x6 is the smallest board margins (2, 3) allow),
# 2 and 3 segments (row r's segment words land in the slot of row 3r/4), a partial
# high half (W = 49..63), narrow boards with a ragged last round of 32 rows and a third
# round, margins None on both drapes, different margins on '#' and '@' (the only way
# '@' issues its own order), and a one-column board.
SHAPES = [
    ('4x6', (4, 6), (15, 31), DEFAULT_MARGINS),
    ('5x16', (5, 16), (17, 45), DEFAULT_MARGINS),
    ('7x17', (7, 17), (19, 51), DEFAULT_MARGINS),
    ('11x33', (11, 33), (25, 81), DEFAULT_MARGINS),
    ('12x48', (12, 48), (25, 97), DEFAULT_MARGINS),
    ('13x49', (13, 49), (27, 99), DEFAULT_MARGINS),
    ('9x63', (9, 63), (21, 121), DEFAULT_MARGINS),
    ('33x63', (33, 63), (49, 101), DEFAULT_MARGINS),
    ('65x64', (65, 64), (81, 101), DEFAULT_MARGINS),
    ('20x20', (20, 20), (34, 61), DEFAULT_MARGINS),
    ('33x33', (33, 33), (45, 71), DEFAULT_MARGINS),
    ('11x33_nomargins', (11, 33), (25, 81), NO_MARGINS),
    ('12x24_walls_only', (12, 24), (22, 161), ((2, 3), None)),
    ('12x24_coins_only', (12, 24), (22, 161), (None, (2, 3))),
    ('9x1_nomargins', (9, 1), (25, 41), NO_MARGINS),
]
SHAPE = {case[0]: case[1:] for case in SHAPES}


def shape_level(name, seed, corner=None):
  board, world, _ = SHAPE[name]
  return open_level(seed, board, world, corner=corner)


def facade_game(maze, board, beneath, margins=DEFAULT_MARGINS, occlusion_in_layers=True):
  """pycolab_b200.games.scrolly_maze.make_game with scroll margins per drape ('#', '@')."""
  from pycolab_b200 import ascii_art
  from pycolab_b200.games import scrolly_maze as g
  from pycolab_b200.prefab_parts import drapes as prefab_drapes
  info = prefab_drapes.Scrolly.PatternInfo(maze, board, board_northwest_corner_mark='+',
                                           what_lies_beneath=beneath)
  sprites = {'P': ascii_art.Partial(g.PlayerSprite, info.virtual_position('P'))}
  for ch in 'abc':
    sprites[ch] = ascii_art.Partial(g.PatrollerSprite, info.virtual_position(ch))
  return ascii_art.ascii_art_to_game(
      board, what_lies_beneath=' ', sprites=sprites,
      drapes={'#': ascii_art.Partial(g.MazeDrape, scroll_margins=margins[0], **info.kwargs('#')),
              '@': ascii_art.Partial(g.CashDrape, scroll_margins=margins[1], **info.kwargs('@'))},
      update_schedule=[['#'], ['a', 'b', 'c', 'P'], ['@']],
      z_order='abc@#P', occlusion_in_layers=occlusion_in_layers)


def lowered(game, pitch=None, repack=False):
  """Lower a facade game; optionally widen its pitch (re-padding the backdrop) or re-pack
  its patterns at the smallest pattern_words pcl_create accepts."""
  from pycolab_b200 import lowering
  low = repitch(lowering.lower(game), pitch)
  if repack:
    words = min_pattern_words(low.cols, low.pattern_cols)
    low.patterns = {d: lowering.pack_rows(lowering.unpack_rows(p, low.pattern_cols), words)
                    for d, p in low.patterns.items()}
    low.pattern_words = words
  return low


def oracle_world(maze, board, beneath, margins=DEFAULT_MARGINS):
  """oracle.games.make_scrolly_maze with scroll margins per drape ('#', '@')."""
  return ogames.make_scrolly_maze(maze, board, '+', beneath, margins=margins)


# ----------------------------------------------- the kernel's shared-memory layout

# Mirrors scrolly_maze.cu (window_words, narrow_board, warp_smem_bytes) and the
# pattern_words rule of its check_spec, which pcl_create applies.
REC_WORDS = 64
WARPS_PER_BLOCK = 4
SEL_TABLE_BYTES = 512                  # one u16[256] selector table per warp (static)


def window_words(W):
  return 4 if W < 2 else 2 * ((63 + W + 63) // 64)


def warp_smem_bytes(H, W, pitch):
  narrow = pitch <= 64
  return (REC_WORDS * 4 + H * pitch + 2 * ceil16(H * window_words(W) * 4) +
          (0 if narrow else ceil16(H * (pitch >> 2))))


def min_pattern_words(W, PW):
  """The smallest pattern_words pcl_create accepts for a W-column board over PW columns."""
  need = max((((PW - W) >> 5) & ~1) + window_words(W), (PW + 31) // 32 + 1)
  return need + (need & 1)


def accepted_smem(H, W, pitch):
  """pcl_create's shared-memory test (UNSUPPORTED past it)."""
  return WARPS_PER_BLOCK * warp_smem_bytes(H, W, pitch) <= MAX_BLOCK_SMEM - WARPS_PER_BLOCK * SEL_TABLE_BYTES


def warp_accesses(H, W, pitch, corner_c, PW):
  """Every (byte offset, size) the kernel touches in one warp's region, for a window at
  pattern column corner_c; plus every pattern word index a staged row reads."""
  nw = window_words(W)
  narrow = pitch <= 64
  wall = REC_WORDS * 4 + H * pitch                  # byte offsets, as in the kernel
  coin = wall + 4 * ((H * nw + 3) & ~3)
  seg = wall if narrow else coin + 4 * ((H * nw + 3) & ~3)
  spr = pitch >> 4
  acc = [(0, REC_WORDS * 4), (REC_WORDS * 4, H * pitch)]
  e = (corner_c >> 5) & ~1
  words = set()
  if narrow:
    for i in range(2 * H):                          # two 8-byte halves per row
      acc += [(wall + 8 * i, 8), (coin + 8 * i, 8)]
      words |= {e + (i & 1) * 2, e + (i & 1) * 2 + 1}
    for r in range(H):                              # uint4 reads, segment words
      acc += [(wall + 16 * r, 16), (coin + 16 * r, 16), (seg + 4 * r * spr, 4 * spr)]
  else:
    for i in range(H * (nw >> 1)):
      acc += [(wall + 8 * i, 8), (coin + 8 * i, 8)]
    words |= set(range(e, e + nw))
    acc += [(wall, 4 * H * nw), (coin, 4 * H * nw), (seg, 4 * H * spr)]
  return acc, words
