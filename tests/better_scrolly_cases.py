"""better_scrolly_maze levels that reach the board's rim, scripted rim cases, a record of
which edges an oracle run went through, and a model of the step kernel's shared-memory
reads.  Shared by test_better_scrolly.py (oracle vs reference, the model) and
test_gpu_better_scrolly.py (device vs oracle).

The stock mazes keep a '#' ring around the floor, so no walker ever reaches the rim.
The levels here have floor up to the edge:
  * the patrollers 'a', 'b', 'c' and the player 'P' are unconfined MazeWalkers: one
    that leaves the board is invisible, sits at position (0, 0) and keeps moving from
    its virtual position;
  * a patroller looks up layers['#'][row, col -+ 1] on even frames (frame 0, its_showtime,
    included) with NumPy's index rules: at column 0 it reads the last column, so a wall
    there turns it east; at column W-1 it raises IndexError.  Off the board it looks
    around (0, 0);
  * a patroller whose position equals P's (P has not moved yet this frame) ends the
    episode, so two walkers off the board meet at (0, 0);
  * CashDrape reads the coin at P's position, (0, 0) for P off the board.
"""

import numpy as np

from oracle import games as ogames
from rim_sweep import MAX_BLOCK_SMEM, repitch

PATROLLERS = 'abc'


def open_level(seed, shape, n_coins, wall_density=0.08, fence=True):
  """Floor up to the edge with scattered '#', a coin at (0, 0) and `n_coins` - 1 more,
  the patrollers in columns 0..W-3 and P anywhere.  fence: a '#' in column W-2 of every
  patroller's row, east of it, so that no patroller can reach the last column (whose
  look-up raises); the patrollers still leave the board by column 0."""
  rs = np.random.RandomState(seed)
  H, W = shape
  assert W >= 4 and H * W >= 8, shape
  art = np.full((H, W), ord(' '), np.uint8)
  art[rs.random_sample((H, W)) < wall_density] = ord('#')
  west = [(r, c) for r in range(H) for c in range(W - 2) if (r, c) != (0, 0)]
  spots = [west[i] for i in rs.permutation(len(west))[:3]]
  for ch, rc in zip(PATROLLERS, spots):
    art[rc] = ord(ch)
    if fence:
      art[rc[0], W - 2] = ord('#')
  free = [tuple(rc) for rc in np.argwhere(art == ord(' ')) if tuple(rc) != (0, 0)]
  if not free:                                   # walls everywhere: clear one cell for P
    free = [tuple(rc) for rc in np.argwhere(art == ord('#')) if tuple(rc) != (0, 0)]
  art[free[rs.randint(len(free))]] = ord('P')
  if n_coins:
    art[0, 0] = ord('@')
    rest = np.argwhere(art == ord(' '))
    for rc in rest[rs.permutation(len(rest))[:n_coins - 1]]:
      art[tuple(rc)] = ord('@')
  else:
    art[0, 0] = ord(' ')
  return [bytes(row).decode('ascii') for row in art]


def lowered(art, pitch=None):
  """The lowered facade game of `art`, its backdrop re-padded to `pitch` columns."""
  from pycolab_b200 import lowering
  from pycolab_b200.games import better_scrolly_maze
  return repitch(lowering.lower(better_scrolly_maze.make_game(art)), pitch)


def make_world(art):
  return ogames.make_better_scrolly(art)


def random_actions(rs, T, B, quit_p=0.02):
  """Walks (0-3), no-ops (4) and a rare quit (5)."""
  rest = (1.0 - quit_p - 0.05) / 4
  return rs.choice(6, size=(T, B), p=[rest] * 4 + [0.05, quit_p]).astype(np.int32)


# ------------------------------------------------------------------ rim cases
# name -> (art, script, edges the script must reach).  'a' and 'c' start moving east,
# 'b' west.  Edges:
#   player_off_n/s/w/e  P left the board by its north, south, west or east side
#   player_return       P came back onto the board
#   p_off_coin          P, off the board, collected the coin at (0, 0)
#   patroller_off       a patroller is off the board
#   patroller_return    a patroller came back onto the board
#   wrap_turn           a patroller in column 0 turned east: a wall in the last column
#   origin_meet         a patroller off the board met P standing on (0, 0)
#   off_board_meet      the episode ended with P and a patroller both off the board
#   shared_cell         two visible patrollers stand in one cell
#   under_coin          a visible patroller stands under a coin
#   showtime_over       the episode ended at its_showtime
#   no_coins            a step left the board without coins and the episode went on
#   last_coin           P collected the last coin and the episode ended
#   raise               play() or its_showtime() raised IndexError
RIM = {
    # P leaves by the north, west, south and east sides, coming back each time; the
    # patrollers bounce in walled pockets.
    'player_off': (['      ', ' #a c#', '  P   ', ' #b  #', '      '],
                   [2, 2, 0, 0, 0, 1, 2, 3, 1, 1, 1, 1, 1, 0, 3, 3, 3, 3, 3, 3, 2],
                   {'player_off_n', 'player_off_s', 'player_off_w', 'player_off_e',
                    'player_return'}),
    # P steps off by the west side and, at (0, 0), collects the coin there; then the
    # other coin, the last, ends the episode.
    'p_off_coin': (['@     ', ' #a c#', 'P     ', ' #b  #', '    @ '],
                   [2, 3, 1, 1, 3, 3, 3, 3, 4, 4],
                   {'player_off_w', 'player_return', 'p_off_coin', 'last_coin'}),
    # 'b' leaves by column 0 and walks on west off the board; P walks onto (0, 0), where
    # the off-board 'b' meets it.
    'patroller_off': (['  P @ ', ' #a c#', ' b    ', '      '], [4, 4, 2, 2, 4, 4, 4, 4],
                      {'patroller_off', 'origin_meet'}),
    # 'b' leaves by column 0; off the board it looks up (0, W-1), a wall, turns east and
    # comes back in its own row, visible again; then it bounces off (2, 5) and leaves
    # again.
    'patroller_return': (['   @  #', ' #a c# ', ' b   # ', '  P    ', '       '],
                         [4] * 24,
                         {'patroller_off', 'patroller_return', 'wrap_turn'}),
    # 'b' starts in column 0 with a wall in the last column of its row: it turns east at
    # its_showtime, walks to the wall and back, and turns again.
    'wrap_turn': ([' #a c#', 'b    #', '  P @ ', '      '],
                  [4, 4, 4, 3, 4, 4, 2, 4, 4, 4, 4, 4, 4, 4, 4, 4, 4, 4],
                  {'wrap_turn'}),
    # P steps off by the west side; 'b' leaves by column 0 a frame later, and both sit at
    # (0, 0): the episode ends.
    'off_board_meet': (['       ', ' #a c# ', ' b     ', 'P  @   '],
                       [2, 4, 4, 4],
                       {'player_off_w', 'patroller_off', 'off_board_meet'}),
    # 'a' and 'c' meet in one cell of their pocket ('c' is drawn on top), and 'b' walks
    # onto a coin and back ('@' is drawn over it).
    'stacked': ([' #a c#', ' #@b #', '  P   ', '    @ '],
                [4, 4, 3, 4, 2, 4, 4, 4, 1, 4, 0, 4],
                {'shared_cell', 'under_coin'}),
    # 'b' moves onto P at its_showtime: every episode ends there.
    'showtime_over': ([' #a c#', ' Pb   ', '   @ #'], [4, 1, 3],
                      {'showtime_over'}),
    # No coins at all: neither side ever ends the episode on coins.
    'no_coins': ([' #a c#', '      ', '  P   ', ' #b  #'],
                 [3, 3, 1, 2, 2, 2, 0, 4, 4, 3, 3, 3, 3, 3],
                 {'no_coins', 'player_off_e'}),
    # One coin: its pick-up ends the episode.
    'one_coin': ([' #a c#', '  P @ ', ' #b  #'], [3, 3, 4],
                 {'last_coin'}),
    # 'a' reaches the last column at frame 2; its look-up at frame 4 raises.
    'raise_mid_run': (['   a  ', ' #b c#', '  P @ ', '      '], [3, 2, 1, 4, 4],
                      {'raise'}),
    # 'a' starts in the last column: its_showtime raises.
    'raise_at_showtime': (['     a', ' #b c#', '  P @ ', '      '], [4, 4],
                          {'raise'}),
}
# The index of the script action whose play() raises; None: its_showtime raises.
RAISES = {'raise_mid_run': 3, 'raise_at_showtime': None}


def _snapshot(world):
  out = {}
  for ch, w in world.things.items():
    if ch != '@':
      out[ch] = (w.row, w.col, bool(w.visible), w.vrow, w.vcol, w.aux.get('moving_east'))
  return out


class Edges(object):
  """Which edges one oracle world went through, step by step (`RIM`'s names)."""

  def __init__(self):
    self.seen = set()

  def start(self, world, out):
    self.prev = _snapshot(world)
    if world.game_over:
      self.seen.add('showtime_over')
    self._now(world, out)

  def step(self, world, out, action):
    now = _snapshot(world)
    H, W = world.rows, world.cols
    prev = self.prev
    p = now['P']
    if prev['P'][2] and not p[2]:
      self.seen.add('player_off_' + ('n' if p[3] < 0 else 's' if p[3] >= H else
                                     'w' if p[4] < 0 else 'e'))
    if p[2] and not prev['P'][2]:
      self.seen.add('player_return')
    if not p[2] and out[1] is not None:
      self.seen.add('p_off_coin')
    for ch in PATROLLERS:
      if now[ch][2] and not prev[ch][2]:
        self.seen.add('patroller_return')
      if prev[ch][1] == 0 and not prev[ch][5] and now[ch][5]:
        self.seen.add('wrap_turn')
    if world.game_over:
      off = [ch for ch in PATROLLERS if not now[ch][2]]
      if off and not p[2]:
        self.seen.add('off_board_meet')
      if off and p[2] and p[:2] == (0, 0):
        self.seen.add('origin_meet')
    if not world.things['@'].curtain.any():
      if not world.game_over:
        self.seen.add('no_coins')
      elif out[1] is not None:
        self.seen.add('last_coin')
    self.prev = now
    self._now(world, out)

  def _now(self, world, out):
    s = self.prev
    coins = world.things['@'].curtain
    cells = []
    for ch in PATROLLERS:
      if not s[ch][2]:
        self.seen.add('patroller_off')
      else:
        cells.append(s[ch][:2])
        if coins[s[ch][:2]]:
          self.seen.add('under_coin')
    if len(set(cells)) < len(cells):
      self.seen.add('shared_cell')


# ------------------------------------- the step kernel's shared-memory reads (render)

# Mirrors better_scrolly.cu (block_smem, the per-warp layout and the render loop) and
# the checks pcl_create applies to a better_scrolly spec.
REC_WORDS = 64
WARPS_PER_BLOCK = 4


def min_bits_words(W):
  """The bit-row width lowering gives a W-column board, the least pcl_create accepts."""
  return (W + 31) // 32 + 1


def warp_layout(H, pitch, BW):
  """Byte offsets of one warp's records, backdrop tile and coin bit rows, and its size."""
  tile = H * pitch
  bits = (H * BW * 4 + 15) & ~15
  return 0, REC_WORDS * 4, REC_WORDS * 4 + tile, REC_WORDS * 4 + tile + bits


def block_smem(H, pitch, BW):
  return WARPS_PER_BLOCK * warp_layout(H, pitch, BW)[3]


def accepted(H, W, pitch, BW=None):
  """pcl_create's verdict on the shape, as the model states it."""
  BW = min_bits_words(W) if BW is None else BW
  return (H > 0 and W > 0 and pitch >= W and pitch % 16 == 0 and BW >= min_bits_words(W)
          and block_smem(H, pitch, BW) <= MAX_BLOCK_SMEM)


def largest_rows(W, pitch, BW=None):
  """The most rows pcl_create accepts for a W-column board at `pitch` (0: none)."""
  lo, hi = 0, 1
  while accepted(hi, W, pitch, BW):
    lo, hi = hi, 2 * hi
  while hi - lo > 1:
    mid = (lo + hi) // 2
    lo, hi = (mid, hi) if accepted(mid, W, pitch, BW) else (lo, mid)
  return lo


def render_coin_reads(H, pitch, BW, bounded=True):
  """Every coin read of the render, as (lane, row, byte offset, size) in one warp's
  region: lane l walks segments l, l+32, ... of the H x pitch/16 segments, stepping its
  (row r, segment sg) as the kernel does, and reads half-word sg of bit row r.
  bounded: only for sg < 2*BW, as the kernel does; False models the unbounded read."""
  _, _, coin, _ = warp_layout(H, pitch, BW)
  spr = pitch >> 4
  total = H * spr
  dr, dsg = 32 // spr, 32 - (32 // spr) * spr
  reads = []
  for lane in range(32):
    r, sg = lane // spr, lane - (lane // spr) * spr
    for seg in range(lane, total, 32):
      assert (r, sg) == divmod(seg, spr), (H, pitch, lane, seg)
      if not bounded or sg < 2 * BW:
        reads.append((lane, r, coin + 4 * r * BW + 2 * sg, 2))
      r += dr
      sg += dsg
      if sg >= spr:
        sg -= spr
        r += 1
  return reads


def overreach(H, pitch, BW, bounded=True):
  """The coin reads that leave their own bit row (r*BW .. (r+1)*BW words) or the
  warp's region."""
  _, _, coin, end = warp_layout(H, pitch, BW)
  bad = []
  for lane, r, off, size in render_coin_reads(H, pitch, BW, bounded):
    lo, hi = coin + 4 * r * BW, coin + 4 * (r + 1) * BW
    if off < lo or off + size > hi or off + size > end:
      bad.append((lane, r, off))
  return bad
