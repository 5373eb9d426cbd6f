"""examples/hello_world.py on `csrc/hello.cu`."""

import numpy as np

from pycolab_b200 import _lib
from pycolab_b200.errors import NotLoweredError
from pycolab_b200.lowering import (LoweredGame, _common, _drape_record, _plot_record,
                                   _sprite_record, _update_order, pack_rows)


def lower(engine, roles):
  """examples/hello_world.py:58-118: up to four SlidingSprites (plain Sprites, each
  with one of four diagonal direction sets) and one RollingDrape, one update group."""
  th = engine.things
  sliders = [c for c in ''.join(_update_order(engine)) if roles[c] == 'hello.slider']
  rollers = [c for c, r in roles.items() if r == 'hello.roller']
  if not 1 <= len(sliders) <= 4 or len(rollers) != 1:
    raise NotLoweredError('hello_world program needs 1-4 SlidingSprites and one RollingDrape')
  game = LoweredGame()
  _common(engine, game, _lib.PROG_HELLO)
  if len(game.groups) != 1:
    raise NotLoweredError('hello_world entities share one update group')
  records = []
  for ch in sliders:
    sp = th[ch]
    sets = list(zip(type(sp)._DX, type(sp)._DY))
    try:
      k = sets.index((sp._dx, sp._dy))
    except ValueError:
      raise NotLoweredError('SlidingSprite {!r} uses an unknown direction set'.format(ch))
    records.append(_sprite_record(sp, aux0=k))
  game.sprite_chars = ''.join(sliders)
  game.impassable = [[0, 0, 0, 0]] * len(sliders)
  game.confined = [False] * len(sliders)
  game.egocentric = [False] * len(sliders)
  game.sprites = np.array(records, dtype=np.int32).reshape(len(sliders), _lib.SPRITE_WORDS)
  game.drape_chars = rollers[0]
  game.margins = [(-1, -1)]
  game.drapes = np.array([_drape_record()], dtype=np.int32)
  game.bits[0] = pack_rows(th[rollers[0]].curtain, game.bits_words)   # the un-rolled curtain
  game.plot = np.array(_plot_record(), dtype=np.int32)
  for k, ch in enumerate(game.z_order):          # the kernel paints in this order
    game.program_arg[k] = ord(ch)
  game.curtain = curtain
  return game


def curtain(eng, d):
  """RollingDrape: the reset curtain shifted by the record's (AUX0, AUX1) counters."""
  import torch
  rr = (torch.arange(eng.rows, device=eng.device)[None, :] -
        eng.drapes[:, d, _lib.D_AUX0].long()[:, None]) % eng.rows
  cc = (torch.arange(eng.cols, device=eng.device)[None, :] -
        eng.drapes[:, d, _lib.D_AUX1].long()[:, None]) % eng.cols
  out = torch.zeros((eng.batch, eng.rows, eng.pitch), dtype=torch.uint8, device=eng.device)
  out[:, :, :eng.cols] = eng.packed_bits(eng._keep_bits_init[d], rr, cc)
  return out
