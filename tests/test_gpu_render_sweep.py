"""The stand-alone renderer (`pcl_render`, csrc/render.cu) vs the oracle.

Every `launch_render` instantiation, boards whose segment loop takes one to four
passes, sprites where NumPy's index rule (`board[tuple(position)]`,
rendering.py:139) wraps, paints nothing or never reaches (pad columns), curtain
bytes other than 0 / 1, shared and per-env backdrops, random per-env z-orders.
Then the facade `BaseObservationRenderer` against upstream's painting semantics.
"""

import ctypes as C

import numpy as np
import pytest

from oracle import engine_model as em

pytestmark = pytest.mark.gpu

SD = [(0, 0), (4, 2), (8, 2), (16, 2), (3, 3), (4, 8), (16, 8)]
BOARDS = [(1, 1), (1, 16), (3, 17), (64, 64), (65, 64), (200, 33), (128, 128)]
SPRITE_CHARS = 'ABCDEFGHIJKLMNOP'
DRAPE_CHARS = 'abcdefgh'


class _Ent(object):
  pass


def _sprite_positions(rs, B, S, H, W, pitch):
  """Rows / columns drawn from in range, negative in range, off the board either
  way, and the pad columns; a few sprites share one cell."""
  kinds = rs.randint(0, 5, size=(B, S, 2))
  rows = np.where(kinds[..., 0] == 0, rs.randint(-H, 0, size=(B, S)),
                  np.where(kinds[..., 0] == 1, H + rs.randint(0, 3, size=(B, S)),
                           np.where(kinds[..., 0] == 2, -H - 1 - rs.randint(0, 3, size=(B, S)),
                                    rs.randint(0, H, size=(B, S)))))
  cols = np.where(kinds[..., 1] == 0, rs.randint(-W, 0, size=(B, S)),
                  np.where(kinds[..., 1] == 1, W + rs.randint(0, pitch - W + 3, size=(B, S)),
                           np.where(kinds[..., 1] == 2, -W - 1 - rs.randint(0, 3, size=(B, S)),
                                    rs.randint(0, W, size=(B, S)))))
  if S >= 2:
    rows[:, 1], cols[:, 1] = rows[:, 0], cols[:, 0]          # two sprites on one cell
  return rows, cols


def _oracle(b, H, W, backdrop, curtains, sprites, z, S, D):
  """em.render with NumPy's index rule restated: a negative coordinate wraps once;
  a sprite outside [-H, H) x [-W, W) paints nothing."""
  things = {}
  for i, c in enumerate(SPRITE_CHARS[:S]):
    e = _Ent()
    r, col = int(sprites[b, i, 0]), int(sprites[b, i, 1])
    e.is_sprite, e.row, e.col = True, r, col
    e.visible = bool(sprites[b, i, 4] & 1) and -H <= r < H and -W <= col < W
    things[c] = e
  for i, c in enumerate(DRAPE_CHARS[:D]):
    e = _Ent()
    e.is_sprite, e.curtain = False, curtains[b, i, :, :W] != 0
    things[c] = e
  return em.render(H, W, backdrop[:, :W], [chr(c) for c in z[b, :S + D]], things)


@pytest.mark.parametrize('S,D', SD, ids=['S%dD%d' % sd for sd in SD])
@pytest.mark.parametrize('shape', BOARDS, ids=['%dx%d' % s for s in BOARDS])
def test_render_sweep(S, D, shape):
  import torch
  from pycolab_b200 import _lib
  lib = _lib.load()
  H, W = shape
  pitch = (W + 15) // 16 * 16
  k = BOARDS.index(shape) + SD.index((S, D))
  B = (1, 7, 1025)[k % 3]
  shared = k % 2 == 1
  rs = np.random.RandomState(1000 * k + H + W)
  spec = _lib.Spec()
  spec.abi_version, spec.program = _lib.ABI_VERSION, _lib.PROG_NONE
  spec.rows, spec.cols, spec.pitch, spec.n_sprites, spec.n_drapes = H, W, pitch, S, D
  for i, c in enumerate(SPRITE_CHARS[:S]):
    spec.sprite_char[i] = ord(c)
  for i, c in enumerate(DRAPE_CHARS[:D]):
    spec.drape_char[i] = ord(c)
  h = C.c_void_p()
  _lib.check(lib.pcl_create(C.byref(spec), B, 0, C.byref(h)), 'pcl_create')
  backdrop = np.zeros((1 if shared else B, H, pitch), np.uint8)
  backdrop[:, :, :W] = rs.randint(0, 256, size=(backdrop.shape[0], H, W))
  curtains = np.zeros((B, max(D, 1), H, pitch), np.uint8)
  curtains[:, :D, :, :W] = rs.choice([0, 0, 0, 1, 2, 255], size=(B, D, H, W))
  sprites = np.zeros((B, max(S, 1), _lib.SPRITE_WORDS), np.int32)
  if S:
    sprites[:, :S, _lib.S_ROW], sprites[:, :S, _lib.S_COL] = _sprite_positions(
        rs, B, S, H, W, pitch)
    sprites[:, :S, _lib.S_FLAGS] = rs.choice([0, 1, 1, 1], size=(B, S))
  chars = [ord(c) for c in SPRITE_CHARS[:S] + DRAPE_CHARS[:D]]
  z = np.stack([rs.permutation(chars) if chars else np.zeros(1, np.int64)
                for _ in range(B)]).astype(np.uint8)
  cuda = lambda a: torch.from_numpy(a).cuda()
  t_bd, t_cur, t_sp, t_z = cuda(backdrop), cuda(curtains), cuda(sprites), cuda(z)
  out = torch.full((B, H, pitch), 0xA5, dtype=torch.uint8, device='cuda')
  try:
    _lib.check(lib.pcl_render(h, t_bd.data_ptr(), 0 if shared else H * pitch,
                              t_cur.data_ptr(), t_sp.data_ptr(), t_z.data_ptr(),
                              out.data_ptr(), C.c_void_p(torch.cuda.current_stream().cuda_stream)),
               'pcl_render')
    torch.cuda.synchronize()
  finally:
    lib.pcl_destroy(h)
  got = out.cpu().numpy()
  envs = range(B) if B <= 7 else sorted(set(list(range(0, B, 41)) + [B - 2, B - 1]))
  for b in envs:
    want = _oracle(b, H, W, backdrop[0 if shared else b], curtains, sprites, z, S, D)
    np.testing.assert_array_equal(got[b, :, :W], want, err_msg='env %d' % b)
  assert not got[:, :, W:].any(), 'pad columns: a sprite or drape painted there'


# ---- the facade canvas -----------------------------------------------------------

def _upstream_paint(backdrop, calls):
  """BaseObservationRenderer (rendering.py:98-160) as NumPy does it."""
  board = backdrop.copy()
  for kind, ch, data in calls:
    if kind == 'sprite':
      board[tuple(data)] = ord(ch)
    else:
      board[data] = ord(ch)
  return board


def _random_calls(rs, n_sprites, n_drapes, H, W, chars):
  calls = [('sprite', None)] * n_sprites + [('drape', None)] * n_drapes
  out = []
  for i in rs.permutation(len(calls)):
    kind = calls[i][0]
    ch = chars[rs.randint(len(chars))]
    if kind == 'sprite':
      out.append((kind, ch, (int(rs.randint(-H, H)), int(rs.randint(-W, W)))))
    else:
      out.append((kind, ch, rs.random_sample((H, W)) < 0.2))
  return out


def _paint(renderer, backdrop, calls):
  renderer.clear()
  renderer.paint_all_of(backdrop)
  for kind, ch, data in calls:
    if kind == 'sprite':
      renderer.paint_sprite(ch, data)
    else:
      renderer.paint_drape(ch, data)
  return renderer.render()


@pytest.mark.parametrize('shape', [(5, 7), (65, 64), (33, 129)], ids=str)
def test_facade_many_paint_calls(shape):
  """24 sprites and 12 drapes: more than one launch holds, rendered as successive
  launches in paint order; characters painted several times keep their order."""
  from pycolab_b200 import rendering
  H, W = shape
  rs = np.random.RandomState(H * W)
  chars = 'PQRSxyz#. '
  r = rendering.BaseObservationRenderer(H, W, chars)
  for trial in range(3):
    backdrop = rs.choice([ord(c) for c in '#. '], size=(H, W)).astype(np.uint8)
    calls = _random_calls(rs, 24, 12, H, W, chars)
    obs = _paint(r, backdrop, calls)
    np.testing.assert_array_equal(obs.board, _upstream_paint(backdrop, calls),
                                  err_msg='trial %d' % trial)


def test_facade_high_backdrop_bytes():
  """Backdrop bytes 128..160 (paint_all_of takes any uint8 canvas) stay where no
  paint call lands; slot codes are taken from bytes the canvas does not use."""
  from pycolab_b200 import rendering
  H, W = 9, 40
  rs = np.random.RandomState(7)
  r = rendering.BaseObservationRenderer(H, W, 'Pab')
  backdrop = rs.randint(128, 161, size=(H, W)).astype(np.uint8)
  calls = _random_calls(rs, 5, 3, H, W, 'Pab')
  np.testing.assert_array_equal(_paint(r, backdrop, calls).board,
                                _upstream_paint(backdrop, calls))
  # a canvas using every byte value leaves no slot code
  full = np.arange(H * W, dtype=np.int64).reshape(H, W).astype(np.uint8)
  r.clear()
  r.paint_all_of(full)
  r.paint_sprite('P', (0, 0))
  with pytest.raises(ValueError):
    r.render()


def test_facade_off_board_sprite_raises():
  from pycolab_b200 import rendering
  r = rendering.BaseObservationRenderer(4, 6, 'P ')
  r.paint_all_of(np.full((4, 6), ord(' '), np.uint8))
  for pos in [(4, 0), (0, 6), (-5, 0), (0, -7), (10, 10)]:
    with pytest.raises(IndexError):
      r.paint_sprite('P', pos)
  r.paint_sprite('P', (-4, -6))                                  # wraps once: (0, 0)
  assert r.render().board[0, 0] == ord('P')
