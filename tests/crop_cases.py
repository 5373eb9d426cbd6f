"""Synthetic frame sequences for the croppers, shared by the CPU and GPU tests.

No step program is involved: each frame gives, per env, the board (bytes; pad columns
non-zero), each sprite's (row, col, visible), each drape's curtain and the episode
counter.  Sprites random-walk, now and then jump (so a saccade fires) and toggle their
visibility; curtains are drawn from patterns chosen where the device's drape median can
go wrong (empty, one cell, even and odd counts, cells only in columns >= 32 / 64 / 96,
full rows, the whole board); some frames hide every tracked entity, so the corner must
stay put.

`CASES` is the grid: every board shape, window, margin kind, initial offset, saccade,
pad kind, tracking list, batch size and corner-state kind is taken at least once
against the others (pairwise by hand, not a full product).  A case is one frame
sequence seen by one or more croppers.
"""

import collections
import json
import os

import numpy as np

SPRITES = 'ABCD'
DRAPES = 'xyzw'
BACKDROP = ' .#'
PATTERNS = ('empty', 'one', 'even', 'odd', 'col32', 'col64', 'col96', 'rows', 'all')


def pitch(W):
  return (W + 15) // 16 * 16


def scroll(rows, cols, track, pad=None, margins=(2, 3), offset=None, saccade=True,
           state='own'):
  """A ScrollingCropper: `track` names entities ('s0' sprite 0, 'd1' drape 1), `pad` is
  None, 'backdrop' or 'sprite'; state 'own' (a caller-owned corner array) or 'plot' (the
  plot record's slot)."""
  return dict(kind='scroll', rows=rows, cols=cols, track=list(track), pad=pad,
              margins=margins, offset=offset, saccade=saccade, state=state)


def fixed(corner, rows, cols, pad=None):
  return dict(kind='fixed', rows=rows, cols=cols, corner=corner, pad=pad, state='own')


def case(name, H, W, croppers, B=5, S=2, D=2, T=16, bump=False):
  return dict(name=name, H=H, W=W, B=B, S=S, D=D, T=T, bump=bump, croppers=croppers,
              seed=sum(ord(c) * (i + 1) for i, c in enumerate(name)) % 100003)


CASES = [
    case('b1x1_w1x1', 1, 1, [scroll(1, 1, ['s0'], margins=(0, 0))], bump=True),
    case('b1x37_w1x5', 1, 37, [scroll(1, 5, ['d0'], margins=(0, None), saccade=False)],
         S=1, D=1),
    case('b37x1_w1x5_pad', 37, 1, [scroll(1, 5, ['s0', 'd0'], pad='backdrop',
                                          margins=(0, 2))], bump=True),
    case('b5x7_w3x5_b4099', 5, 7, [scroll(3, 5, ['d0', 's0', 'd1', 's1'], pad='sprite',
                                          margins=(1, 2), offset=(2, -3), saccade=False)],
         B=4099, T=10, bump=True),
    case('b5x7_w5x7_board', 5, 7, [scroll(5, 7, ['s0'], margins=(None, None),
                                          state='plot')], bump=True),
    case('b8x14_w4x6', 8, 14, [scroll(4, 6, ['s0', 'd0'], margins=(1, 2))], bump=True),
    case('b8x14_w10x16_pad', 8, 14, [scroll(10, 16, ['d1', 's1'], pad='backdrop',
                                            margins=(0, 0), offset=(2, -3))]),
    case('b31x33_w9x9_off', 31, 33, [scroll(9, 9, ['d0'], pad='backdrop',
                                            margins=(None, None), offset=(-45, 0))], S=1),
    case('b31x33_w1x5_b4099', 31, 33, [scroll(1, 5, ['s0'], margins=(0, 1))], B=4099, T=8,
         bump=True),
    case('b32x32_w5x7_plot', 32, 32, [scroll(5, 7, ['s0', 'd0'], margins=(2, 3),
                                             saccade=False, state='plot')], bump=True),
    case('b33x65_w9x9', 33, 65, [scroll(9, 9, ['d0', 's0'], margins=(4, 4))], bump=True),
    case('b64x64_w4x6_b1', 64, 64, [scroll(4, 6, ['s1', 'd1', 's0', 'd0'], pad='sprite',
                                           margins=(0, 0), offset=(2, -3))], B=1, T=24),
    case('b100x127_w9x9', 100, 127, [scroll(9, 9, ['d0'], margins=(None, None))], S=1,
         bump=True),
    case('b128x128_w5x7', 128, 128, [scroll(5, 7, ['d0', 'd1'], pad='backdrop',
                                            margins=(2, None), saccade=False)], T=12),
    case('b128x128_w255x257', 128, 128, [scroll(255, 257, ['s0'], pad='backdrop')],
         B=2, D=1, T=4),
    case('b32x32_two_croppers', 32, 32, [scroll(9, 9, ['s0'], margins=(None, None)),
                                         scroll(5, 7, ['d0', 's1'], pad='sprite',
                                                margins=(1, 2), state='plot')]),
    case('b8x14_fixed', 8, 14, [fixed((-2, -3), 5, 7, 'backdrop'),
                                fixed((6, 10), 5, 7, 'sprite'),
                                fixed((20, 30), 3, 5, 'backdrop'),
                                fixed((-9, 2), 4, 6, 'backdrop'),
                                fixed((1, 2), 3, 5)]),
    case('b1x1_fixed', 1, 1, [fixed((0, 0), 1, 1), fixed((-1, -1), 3, 3, 'backdrop')],
         S=1, D=1),
]

BY_NAME = dict((c['name'], c) for c in CASES)


def chars(c):
  """(sprite chars, drape chars) of a case."""
  return SPRITES[:c['S']], DRAPES[:c['D']]


def entity(c, name):
  s, d = chars(c)
  return (s if name[0] == 's' else d)[int(name[1:])]


def pad_char(c, cropper):
  return {None: None, 'backdrop': '.', 'sprite': SPRITES[0]}[cropper['pad']]


Frame = collections.namedtuple('Frame', 'boards sprites curtains episode')
# boards u8 [B, H, pitch]; sprites i32 [B, S, 3] (row, col, visible);
# curtains bool [B, D, H, W]; episode i32 [B]


def _curtain(rs, H, W):
  out = np.zeros((H, W), bool)
  kind = PATTERNS[rs.randint(len(PATTERNS))]
  if kind == 'one':
    out[rs.randint(H), rs.randint(W)] = True
  elif kind in ('even', 'odd'):
    n = min(H * W, 2 * rs.randint(1, 4) + (kind == 'odd'))
    out.reshape(-1)[rs.choice(H * W, n, replace=False)] = True
  elif kind.startswith('col'):
    c0 = min(int(kind[3:]), W - 1)
    n = min(H * (W - c0), rs.randint(1, 7))
    cells = rs.choice(H * (W - c0), n, replace=False)
    out[cells // (W - c0), c0 + cells % (W - c0)] = True
  elif kind == 'rows':
    out[rs.choice(H, min(H, rs.randint(1, 3)), replace=False)] = True
  elif kind == 'all':
    out[:] = True
  return out


def frames(c):
  """The case's T frames, seeded by its name."""
  rs = np.random.RandomState(c['seed'])
  B, H, W, S, D = c['B'], c['H'], c['W'], c['S'], c['D']
  pos = np.stack([rs.randint(0, H, (B, S)), rs.randint(0, W, (B, S))], -1)
  vis = np.ones((B, S), bool)
  episode = np.zeros(B, np.int32)
  curt = np.stack([[_curtain(rs, H, W) for _ in range(D)] for _ in range(B)]) if D else \
      np.zeros((B, 0, H, W), bool)
  out = []
  for t in range(c['T']):
    if t:
      pos += rs.randint(-1, 2, pos.shape)
      jump = rs.random_sample((B, S)) < 0.1
      pos[..., 0] = np.where(jump, rs.randint(0, H, (B, S)), pos[..., 0])
      pos[..., 1] = np.where(jump, rs.randint(0, W, (B, S)), pos[..., 1])
      pos[..., 0] = np.clip(pos[..., 0], 0, H - 1)
      pos[..., 1] = np.clip(pos[..., 1], 0, W - 1)
      vis ^= rs.random_sample((B, S)) < 0.15
      for e in range(B):
        for d in range(D):
          if rs.random_sample() < 0.4:
            curt[e, d] = _curtain(rs, H, W)
      if c['bump']:
        episode += (rs.random_sample(B) < 0.1).astype(np.int32)
    hidden = rs.random_sample(B) < 0.1                     # nothing to track: stay put
    v = vis & ~hidden[:, None]
    cu = curt & ~hidden[:, None, None, None]
    boards = rs.randint(128, 256, (B, H, pitch(W))).astype(np.uint8)
    codes = np.frombuffer(BACKDROP.encode(), np.uint8)
    boards[:, :, :W] = codes[rs.randint(0, len(codes), (B, H, W))]
    for d in range(D):
      boards[:, :, :W][cu[:, d]] = ord(DRAPES[d])
    for s in range(S):
      e = np.nonzero(v[:, s])[0]
      boards[e, pos[e, s, 0], pos[e, s, 1]] = ord(SPRITES[s])
    sprites = np.concatenate([pos, v[..., None]], -1).astype(np.int32)
    out.append(Frame(boards, sprites, cu.copy(), episode.copy()))
  return out


def layers(c, f, e):
  """Un-occluded layers of env e in frame f (what occlusion_in_layers=False gives)."""
  S, D = c['S'], c['D']
  board = f.boards[e, :, :c['W']]
  out = {ch: board == ord(ch) for ch in BACKDROP}
  for s in range(S):
    plane = np.zeros(board.shape, bool)
    if f.sprites[e, s, 2]:
      plane[f.sprites[e, s, 0], f.sprites[e, s, 1]] = True
    out[SPRITES[s]] = plane
  for d in range(D):
    out[DRAPES[d]] = f.curtains[e, d].copy()
  return out


# ---- the oracle over a case --------------------------------------------------------

class _Thing(object):
  pass


class World(object):
  """What oracle.engine_model.ScrollingCrop reads: rows, cols and things."""

  def __init__(self, c):
    self.rows, self.cols = c['H'], c['W']
    self.things = {}
    s_chars, d_chars = chars(c)
    for ch in s_chars + d_chars:
      self.things[ch] = _Thing()
      self.things[ch].is_sprite = ch in s_chars

  def show(self, c, f, e):
    s_chars, d_chars = chars(c)
    for s, ch in enumerate(s_chars):
      t = self.things[ch]
      t.row, t.col, t.visible = int(f.sprites[e, s, 0]), int(f.sprites[e, s, 1]), bool(
          f.sprites[e, s, 2])
    for d, ch in enumerate(d_chars):
      self.things[ch].curtain = f.curtains[e, d]


def oracle(c, cropper, seq, envs=None, with_layers=False):
  """Per frame: (crops u8 [n, rows, cols], corners i32 [n, 2][, layer dicts]) of the
  oracle for the envs `envs` (default all).  A new episode is a new engine."""
  from oracle import engine_model as em
  envs = range(c['B']) if envs is None else envs
  pad = pad_char(c, cropper)
  crops, worlds, out = {}, {}, []
  for f in seq:
    boards, corners, lays = [], [], []
    for e in envs:
      board = f.boards[e, :, :c['W']]
      lay = layers(c, f, e) if with_layers else None
      if cropper['kind'] == 'fixed':
        corner = cropper['corner']
        got = em.crop_window(board, corner, cropper['rows'], cropper['cols'], pad, lay)
      else:
        if e not in crops:
          crops[e] = em.ScrollingCrop(cropper['rows'], cropper['cols'],
                                      [entity(c, n) for n in cropper['track']], pad_char=pad,
                                      scroll_margins=cropper['margins'],
                                      initial_offset=cropper['offset'],
                                      saccade=cropper['saccade'])
        key = (e, int(f.episode[e]))
        if key not in worlds:
          worlds[key] = World(c)
        worlds[key].show(c, f, e)
        crops[e].set_engine(worlds[key])
        got = crops[e].crop(board, lay)
        corner = crops[e].corner
      if with_layers:
        boards.append(got[0])
        lays.append(got[1])
      else:
        boards.append(got)
      corners.append(corner)
    item = (np.stack(boards), np.array(corners, np.int32))
    out.append(item + (lays,) if with_layers else item)
  return out


# ---- the reference over a case (where it is installed) -----------------------------

Obs = collections.namedtuple('Obs', 'board layers')


class _RefSprite(object):
  def __init__(self, row, col, visible):
    self.position, self.visible = (row, col), visible


class _RefDrape(object):        # no `visible`: upstream's _centroid then takes the curtain
  def __init__(self, curtain):
    self.curtain = curtain


class _RefBackdrop(object):
  palette = BACKDROP


class RefEngine(object):
  """What the reference's croppers read of an Engine: rows, cols, things and the
  backdrop's palette."""

  def __init__(self, c):
    self.rows, self.cols = c['H'], c['W']
    self.backdrop = _RefBackdrop()
    self.things = {}

  def show(self, c, f, e):
    s_chars, d_chars = chars(c)
    for s, ch in enumerate(s_chars):
      self.things[ch] = _RefSprite(int(f.sprites[e, s, 0]), int(f.sprites[e, s, 1]),
                                   bool(f.sprites[e, s, 2]))
    for d, ch in enumerate(d_chars):
      self.things[ch] = _RefDrape(f.curtains[e, d])


def reference(cropping, c, cropper, seq, envs):
  """`oracle(..., with_layers=True)` computed by the reference's own croppers (module
  `cropping`); corners of a FixedCropper are its fixed corner."""
  pad = pad_char(c, cropper)
  per_env = []
  for e in envs:
    if cropper['kind'] == 'fixed':
      ref = cropping.FixedCropper(tuple(cropper['corner']), cropper['rows'], cropper['cols'],
                                  pad)
    else:
      ref = cropping.ScrollingCropper(cropper['rows'], cropper['cols'],
                                      [entity(c, n) for n in cropper['track']], pad_char=pad,
                                      scroll_margins=tuple(cropper['margins']),
                                      initial_offset=cropper['offset'],
                                      saccade=cropper['saccade'])
    engines, frames_e = {}, []
    for f in seq:
      ep = int(f.episode[e])
      if ep not in engines:                 # a new episode is a new Engine
        engines[ep] = RefEngine(c)
      engines[ep].show(c, f, e)
      ref.set_engine(engines[ep])
      got = ref.crop(Obs(f.boards[e, :, :c['W']], layers(c, f, e)))
      corner = cropper['corner'] if cropper['kind'] == 'fixed' else ref._corner
      frames_e.append((got.board.copy(), tuple(corner),
                       dict((ch, l.copy()) for ch, l in got.layers.items())))
    per_env.append(frames_e)
  return [(np.stack([p[t][0] for p in per_env]), np.array([p[t][1] for p in per_env], np.int32),
           [p[t][2] for p in per_env]) for t in range(len(seq))]


def crop_spec(c, cropper):
  """The pcl_crop_spec of a cropper, as the facade classes build it."""
  from pycolab_b200 import _lib
  from pycolab_b200 import batched
  pad = pad_char(c, cropper)
  if cropper['kind'] == 'fixed':
    r, col = cropper['corner']
    return _lib.CropSpec(cropper['rows'], cropper['cols'], -1, -1 if pad is None else ord(pad),
                         0, 0, r, col, 0)
  s_chars, d_chars = chars(c)
  track = []
  for n in cropper['track']:
    track.append(int(n[1:]) + 1 if n[0] == 's' else -(int(n[1:]) + 1))
  # a lone sprite goes through sprite_index with an empty list, as BatchedEngine.crop's
  # callers without a priority list pass it
  if len(track) == 1 and track[0] > 0:
    return batched.scrolling_crop_spec(cropper['rows'], cropper['cols'], track[0] - 1,
                                       pad_char=pad, scroll_margins=cropper['margins'],
                                       initial_offset=cropper['offset'],
                                       saccade=cropper['saccade'])
  return batched.scrolling_crop_spec(cropper['rows'], cropper['cols'], 0, pad_char=pad,
                                     scroll_margins=cropper['margins'],
                                     initial_offset=cropper['offset'],
                                     saccade=cropper['saccade'], track=track)


# ---- goldens: a few cases with the reference's own crops (tests/golden/cropgrid_*.npz) --

GOLDEN_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
GOLDEN_PREFIX = 'cropgrid_'
PAD_BYTE = 0xEE                  # the pad columns of a replayed board (any non-zero byte)


def layer_chars(c):
  s_chars, d_chars = chars(c)
  return ''.join(sorted(BACKDROP + s_chars + d_chars))


def golden_arrays(c, seq, per_cropper):
  """The npz arrays of a case: its inputs and, per cropper k, the crops, corners and
  layers `reference` returned (`per_cropper[k]`)."""
  W, lc = c['W'], layer_chars(c)
  out = dict(config=np.frombuffer(json.dumps(c).encode(), np.uint8),
             boards=np.stack([f.boards[:, :, :W] for f in seq]),
             sprites=np.stack([f.sprites for f in seq]),
             curtains=np.packbits(np.stack([f.curtains for f in seq]).reshape(-1)),
             episode=np.stack([f.episode for f in seq]))
  for k, frames_k in enumerate(per_cropper):
    out['crop%d' % k] = np.stack([x[0] for x in frames_k])
    out['corner%d' % k] = np.stack([x[1] for x in frames_k])
    planes = np.stack([[[lay[ch] for ch in lc] for lay in x[2]] for x in frames_k])
    out['layers%d' % k] = np.packbits(planes.reshape(-1))
  return out


def golden_names():
  import glob
  return sorted(os.path.basename(p)[:-4]
                for p in glob.glob(os.path.join(GOLDEN_DIR, GOLDEN_PREFIX + '*.npz')))


def load_golden(name):
  """(case, frames, [per cropper: per frame (crops, corners, layer dicts)])."""
  with np.load(os.path.join(GOLDEN_DIR, name + '.npz')) as z:
    g = dict((k, z[k]) for k in z.files)
  c = json.loads(bytes(g['config']).decode())
  for k in c['croppers']:
    for key in ('margins', 'offset', 'corner'):
      if k.get(key) is not None:
        k[key] = tuple(k[key])
  T, B, H, W, S, D = c['T'], c['B'], c['H'], c['W'], c['S'], c['D']
  curtains = np.unpackbits(g['curtains'])[:T * B * D * H * W].astype(bool).reshape(
      T, B, D, H, W)
  seq = []
  for t in range(T):
    boards = np.full((B, H, pitch(W)), PAD_BYTE, np.uint8)
    boards[:, :, :W] = g['boards'][t]
    seq.append(Frame(boards, g['sprites'][t], curtains[t], g['episode'][t]))
  lc = layer_chars(c)
  want = []
  for k, cropper in enumerate(c['croppers']):
    r, cc_ = cropper['rows'], cropper['cols']
    planes = np.unpackbits(g['layers%d' % k])[:T * B * len(lc) * r * cc_].astype(bool).reshape(
        T, B, len(lc), r, cc_)
    want.append([(g['crop%d' % k][t], g['corner%d' % k][t],
                  [dict((ch, planes[t, e, i]) for i, ch in enumerate(lc)) for e in range(B)])
                 for t in range(T)])
  return c, seq, want
