"""examples/extraterrestrial_marauders.py on `csrc/marauders.cu`."""

import numpy as np

from pycolab_b200 import _lib
from pycolab_b200.errors import NotLoweredError
from pycolab_b200.lowering import (LoweredGame, _common, _drape_record, _plot_record,
                                   _set_sprites, _sprite_record, pack_rows)


def lower(engine, roles):
  th = engine.things
  want = {'P': 'marauders.player', 'B': 'marauders.bunker', 'X': 'marauders.marauder',
          'a': 'marauders.up_bolt', 'b': 'marauders.up_bolt', 'c': 'marauders.up_bolt',
          'd': 'marauders.up_bolt', 'y': 'marauders.down_bolt', 'z': 'marauders.down_bolt'}
  if roles != want:
    raise NotLoweredError('marauders program needs exactly {} (got {})'.format(want, roles))
  game = LoweredGame()
  _common(engine, game, _lib.PROG_MARAUDERS)
  sprites = [th[c] for c in 'Pabcdyz']
  _set_sprites(game, sprites, [_sprite_record(s) for s in sprites])
  game.drape_chars = 'BX'
  game.margins = [(-1, -1), (-1, -1)]
  game.bits = {0: pack_rows(th['B'].curtain, game.bits_words),
               1: pack_rows(th['X'].curtain, game.bits_words)}
  game.drapes = np.array([_drape_record(), _drape_record(aux0=th['X']._dx)], dtype=np.int32)
  game.plot = np.array(_plot_record(aux0=_lib.NEVER, aux1=_lib.NEVER), dtype=np.int32)
  game.rng_streams = ('numpy',)     # the global np.random (extraterrestrial_marauders.py:253)
  return game
