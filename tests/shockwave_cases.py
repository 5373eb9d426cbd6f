"""shockwave levels of any shape shockwave_step accepts, at any ring width, scripted rim
cases, generator seeds that put the first impact where a case needs it, and a record of
which edges an oracle run went through.  Shared by test_shockwave.py (oracle vs
reference) and test_gpu_shockwave.py (device vs oracle).

The generated levels (levels.shockwave_level) keep a '^' row on top, P on the bottom row
and walls on interior rows; here '^', ' ', '+' and '=' go anywhere:
  * the ring is the cells at distance steps < d <= steps + width from the impact point,
    minus walls, so near a side of the board it is clipped there; with every ring cell on
    a wall the curtain is empty and the next frame draws a new impact;
  * an impact is np.random.randint(0, H * W): MT19937 outputs masked to the next power of
    two, and rejected above H * W - 1 (most of them for H * W = 2, 9 or 129);
  * P wins when the stale board shows '^' at its new position: neither the old ring nor
    P itself covered it.  P burns when it stands on ' ' under the new ring;
  * P is confined and stops at '='.
"""

import numpy as np

from oracle import games as ogames
from rim_sweep import repitch

ACTIONS = 5        # 0 north, 1 west, 2 east, 3 _stay(), 4 no call


def open_level(seed, shape, walls=0.15, safe=0.2, bunkers=0.2, p_cell=None):
  """An H x W art of ' ' with '=', '^' and '+' scattered at the given densities (at least
  one '='), and P at `p_cell` or on any cell but a wall."""
  rs = np.random.RandomState(seed)
  H, W = shape
  assert H * W >= 2, shape
  u = rs.random_sample((H, W))
  art = np.full((H, W), ord(' '), np.uint8)
  art[u < walls + safe + bunkers] = ord('+')
  art[u < walls + safe] = ord('^')
  art[u < walls] = ord('=')
  cells = [(r, c) for r in range(H) for c in range(W)]
  if p_cell is None:
    p_cell = cells[rs.randint(len(cells))]
  art[tuple(p_cell)] = ord('P')
  if not (art == ord('=')).any():
    others = [rc for rc in cells if rc != tuple(p_cell)]
    art[others[rs.randint(len(others))]] = ord('=')
  return [bytes(row).decode('ascii') for row in art]


# The board shapes the GPU sweep steps (up to 32 x 64): H * W = 2, 9 and 129 reject most
# MT19937 outputs of a draw, 2048 none; each side of 16, 32 and 48 columns.
SHAPES = [(1, 2), (2, 1), (1, 16), (3, 3), (3, 43), (2, 64), (5, 17), (7, 32), (9, 33),
          (12, 15), (12, 17), (12, 32), (17, 48), (31, 33), (31, 63), (32, 15), (32, 64)]
WIDTHS = (0, 1, 2, 5, 80, 1024)


def sweep_level(shape, seed):
  """The open level of a board shape, its densities varied with the seed."""
  k = sum(shape) + seed
  return open_level(seed + 10 * k, shape, walls=0.1 + 0.05 * (k % 3), safe=0.1 + 0.1 * (k % 2),
                    bunkers=0.1 + 0.1 * (k % 3))


def rim_cells(shape):
  """The four corners and a cell in the middle of each side."""
  H, W = shape
  return sorted({(0, 0), (0, W - 1), (H - 1, 0), (H - 1, W - 1), (0, W // 2),
                 (H - 1, W // 2), (H // 2, 0), (H // 2, W - 1)})


def make_game(art, width=2):
  """The facade game of `art` with a ring `width` cells thick."""
  from pycolab_b200 import ascii_art
  from pycolab_b200.games import shockwave
  return ascii_art.ascii_art_to_game(
      art, what_lies_beneath='+', sprites={'P': shockwave.PlayerSprite},
      drapes={'@': ascii_art.Partial(shockwave.ShockwaveDrape, width=width),
              ' ': shockwave.MinimalDrape, '^': shockwave.MinimalDrape},
      update_schedule=[' ', '^', 'P', '@'], z_order=[' ', '^', '@', 'P'])


def lowered(art, width=2, pitch=None):
  """The lowered facade game of `art`, its backdrop re-padded to `pitch` columns."""
  from pycolab_b200 import lowering
  return repitch(lowering.lower(make_game(art, width)), pitch)


def make_world(art, rng, width=2):
  return ogames.make_shockwave(art, rng, width)


def random_actions(rs, T, B, north=0.4):
  """Mostly north, as a player heading for the safe zone would, and the rest spread over
  west, east, _stay() and no call."""
  rest = (1.0 - north) / 4
  return rs.choice(ACTIONS, size=(T, B), p=[north] + [rest] * 4).astype(np.int32)


def impact_seed(shape, cell, start=0):
  """The least seed >= start whose RandomState's first randint(0, H * W) is `cell`."""
  H, W = shape
  k = cell[0] * W + cell[1]
  seed = start
  while np.random.RandomState(seed).randint(0, H * W) != k:
    seed += 1
  return seed


# ------------------------------------------------------------------ rim cases
# name -> (art, width, generator seed, script, edges the script must reach).  Edges:
#   clip_n/s/w/e        the ring reached past that side of the board
#   clip_all            ... past all four sides in one frame
#   wall_cut            a ring cell on '=' left out of the curtain
#   ring_on_walls       every ring cell on '=': an empty curtain, a new impact next frame
#   redraw              a frame drew a new impact (after the first)
#   push_n/w/e          P pushed out of the board by that side and stayed
#   push_wall           P pushed against '=' and stayed
#   stay / no_call      actions 3 (_stay()) and 4 (no call)
#   stay_on_safe        P stood on '^' and stayed there a frame: no win, as the stale board
#                       shows P there
#   return_win          P left a '^' it had stood on without winning and came back: a win
#   covered_safe        P stepped onto a '^' the old ring covered: no win that frame
#   win_off_row0        a win on a '^' off row 0
#   burn                P on ' ' under the new ring: -1
#   shelter             P on '+' under the new ring: nothing
#   no_safe / no_danger the level has no '^' / no ' '
RIM = {
    # P pushes out by the north, west and east sides; a ring clipped on all four sides.
    'clip_all': (['P +', '  +', ' ^=', '++ '], 2, 96,
                 [1, 2, 0, 3, 3, 1, 2, 2, 0, 0, 3, 2, 0, 2, 2],
                 {'clip_all', 'redraw', 'push_n', 'push_w', 'push_e', 'burn', 'wall_cut'}),
    # Mostly walls: a ring that lies wholly on '=' leaves the curtain empty, and the next
    # frame draws again; P pushes against a wall.
    'walls': (['= =', '===', '===', '^=P'], 1, 97, [0, 0, 0, 0],
              {'ring_on_walls', 'wall_cut', 'push_wall', 'redraw'}),
    # Width 0: the curtain stays empty, so every frame draws a new impact; a win on a '^'
    # off row 0.
    'width0': (['+ ', '=^', '==', 'P^'], 0, 525, [3, 2, 4, 2, 2, 3, 4],
               {'redraw', 'stay', 'no_call', 'win_off_row0'}),
    # Width 1: P burns on ' ', shelters on '+' and wins off row 0.
    'width1': ([' =^ ', '  ^ ', '+ P '], 1, 714, [0, 0, 4, 3, 1, 0, 0],
               {'burn', 'shelter', 'win_off_row0', 'clip_all', 'no_call'}),
    # Width 80, wider than the 32 x 64 board's diagonal: the first ring covers the board.
    'width80': ([' P^   ', '^^=+=+', ' ^  = ', '^+^ +^'], 80, 186, [0, 3, 0, 0, 1, 3],
                {'clip_all', 'burn', 'redraw', 'push_n'}),
    # Width 1024, the widest accepted; no ' ' on the board: P stands on a '^' the ring
    # covered, and stays there.
    'width1024': (['+=+', '+++', '^P^', '^++', '^+^'], 1024, 404, [2, 2, 2, 3, 4, 4, 0],
                  {'clip_all', 'shelter', 'covered_safe', 'stay_on_safe', 'no_danger'}),
    # P steps onto a '^' under the old ring (no win), stays (no win: the stale board
    # shows P), leaves and comes back: a win.
    'safe_return': ([' ^P^^', '^^^^^', ' ^   ', '^^==^'], 2, 944, [3, 0, 1, 0, 4, 2, 1],
                    {'covered_safe', 'stay_on_safe', 'return_win', 'push_n'}),
    # '^' everywhere off row 0 and under the ring.
    'covered_safe': (['^=+^', '^^^ ', '^^P+', '^+^ '], 2, 569, [1, 1, 1, 4, 0],
                     {'covered_safe', 'win_off_row0'}),
    # No '^': nobody wins.
    'no_safe': (['  + ', '  ++', 'P = '], 2, 586, [3, 0, 3, 2, 0, 0],
                {'no_safe', 'burn', 'redraw', 'shelter'}),
    # No ' ': nobody burns.
    'no_danger': (['+^+==+', '+^^+^+', '+++++^', '+P=+++'], 2, 198, [2, 4, 1, 0, 0],
                  {'no_danger', 'push_wall', 'shelter'}),
}


def _snapshot(world):
  th = world.things
  wave = th['@']
  return dict(p=th['P'].position, curtain=wave.curtain.copy(), steps=wave.aux['steps'],
              distance=wave.aux['distance'].copy(), width=wave.aux['width'])


class Edges(object):
  """Which edges one oracle world went through, step by step (the names above)."""

  def __init__(self):
    self.seen = set()

  def start(self, world, out):
    self.stood_on_safe = set()
    self.safe = world.things['^'].curtain.copy()
    self.danger = world.things[' '].curtain.copy()
    self.walls = world.backdrop == ord('=')
    if not self.safe.any():
      self.seen.add('no_safe')
    if not self.danger.any():
      self.seen.add('no_danger')
    self.prev = _snapshot(world)
    self._ring(self.prev, None)

  def step(self, world, out, action):
    now = _snapshot(world)
    prev = self.prev
    H, W = world.rows, world.cols
    p0, p1 = tuple(prev['p']), tuple(now['p'])
    if action == 3:
      self.seen.add('stay')
    if action == 4:
      self.seen.add('no_call')
    moves = {0: (-1, 0), 1: (0, -1), 2: (0, 1)}
    if action in moves and p0 == p1:
      r, c = p0[0] + moves[action][0], p0[1] + moves[action][1]
      if r < 0:
        self.seen.add('push_n')
      elif c < 0:
        self.seen.add('push_w')
      elif c >= W:
        self.seen.add('push_e')
      elif self.walls[r, c]:
        self.seen.add('push_wall')
    won = out[1] is not None and out[1] > 0
    burned = out[1] is not None and out[1] < 0
    if self.safe[p1] and p0 == p1 and not won:
      self.seen.add('stay_on_safe')
    if won and p1 in self.stood_on_safe:
      self.seen.add('return_win')
    if self.safe[p1] and not won:
      self.stood_on_safe.add(p1)
    if won and p1[0] != 0:
      self.seen.add('win_off_row0')
    if self.safe[p1] and p0 != p1 and prev['curtain'][p1] and not won:
      self.seen.add('covered_safe')
    if burned:
      self.seen.add('burn')
    if now['curtain'][p1] and not self.danger[p1] and not self.safe[p1] and not burned:
      self.seen.add('shelter')
    self.prev = now
    self._ring(now, prev)

  def _ring(self, now, prev):
    if now['steps'] == 1 and prev is not None:
      self.seen.add('redraw')
    d, s, w = now['distance'], now['steps'] - 1, now['width']
    band = (d > s) & (d <= s + w)
    if band.any() and not (band & ~self.walls).any():
      self.seen.add('ring_on_walls')
    if (band & self.walls).any() and (band & ~self.walls).any():
      self.seen.add('wall_cut')
    if not now['curtain'].any():
      return
    ir, ic = np.unravel_index(np.argmin(d), d.shape)
    hi = s + w
    H, W = d.shape
    sides = {'clip_n': ir - hi < 0, 'clip_s': ir + hi > H - 1,
             'clip_w': ic - hi < 0, 'clip_e': ic + hi > W - 1}
    for k, v in sides.items():
      if v:
        self.seen.add(k)
    if all(sides.values()):
      self.seen.add('clip_all')

