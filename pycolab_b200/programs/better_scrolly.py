"""examples/better_scrolly_maze.py on `csrc/better_scrolly.cu`."""

import numpy as np

from pycolab_b200 import _lib
from pycolab_b200.errors import NotLoweredError
from pycolab_b200.lowering import (LoweredGame, _common, _drape_record, _plot_record,
                                   _set_sprites, _sprite_record, pack_rows)


def lower(engine, roles):
  th = engine.things
  want = {'P': 'better.player', 'a': 'better.patroller', 'b': 'better.patroller',
          'c': 'better.patroller', '@': 'better.cash'}
  if roles != want:
    raise NotLoweredError('better_scrolly_maze program needs exactly {} (got {})'.format(
        want, roles))
  game = LoweredGame()
  _common(engine, game, _lib.PROG_BETTER_SCROLLY)
  sprites = [th[c] for c in 'Pabc']
  records = [_sprite_record(th['P'])]
  records += [_sprite_record(th[c], aux0=int(bool(th[c]._moving_east))) for c in 'abc']
  _set_sprites(game, sprites, records)
  game.drape_chars = '@'
  game.margins = [(-1, -1)]
  game.bits = {0: pack_rows(th['@'].curtain, game.bits_words)}
  game.drapes = np.array([_drape_record()], dtype=np.int32)
  game.plot = np.array(_plot_record(aux0=int(th['@'].curtain.sum())), dtype=np.int32)
  return game
