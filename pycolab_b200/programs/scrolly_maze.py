"""examples/scrolly_maze.py on `csrc/scrolly_maze.cu`."""

import numpy as np

from pycolab_b200 import _lib
from pycolab_b200.errors import NotLoweredError
from pycolab_b200.lowering import (LoweredGame, _common, _plot_record, _scrolly_record,
                                   _set_sprites, _sprite_record, pack_rows, round_up)


def lower(engine, roles):
  th = engine.things
  want = {'P': 'scrolly.player', 'a': 'scrolly.patroller', 'b': 'scrolly.patroller',
          'c': 'scrolly.patroller', '#': 'scrolly.maze', '@': 'scrolly.cash'}
  if roles != want:
    raise NotLoweredError('scrolly_maze program needs exactly {} (got {})'.format(want, roles))
  game = LoweredGame()
  _common(engine, game, _lib.PROG_SCROLLY_MAZE, never_reads_layers=True)
  sprites = [th[c] for c in 'Pabc']
  records = [_sprite_record(th['P'], aux0=0, aux1=_lib.NEVER)]
  records += [_sprite_record(th[c], aux0=int(bool(th[c]._moving_east))) for c in 'abc']
  _set_sprites(game, sprites, records)
  walls, coins = th['#'], th['@']
  for d in (walls, coins):
    if d._scrolling_group != '':
      raise NotLoweredError('only the default scrolling group is lowered')
    if d.whole_pattern.shape != walls.whole_pattern.shape:
      raise NotLoweredError('Scrolly patterns of different shapes')
    if tuple(d._board_shape) != (engine.rows, engine.cols):
      raise NotLoweredError('Scrolly board_shape differs from the Engine board')
  game.drape_chars = '#@'
  game.margins = [(-1, -1) if d._scroll_margins is None else tuple(d._scroll_margins)
                  for d in (walls, coins)]
  game.pattern_rows, game.pattern_cols = walls.whole_pattern.shape
  # zero-padded row: the kernel stages 2 * ceil((63 + W) / 64) words per window row
  # starting at an even word (4 words up to 64 columns).
  slack = 3 if engine.cols <= 64 else 2 * ((63 + engine.cols + 63) // 64) + 1
  game.pattern_words = round_up((game.pattern_cols + 31) // 32 + slack, 2)
  game.patterns = {0: pack_rows(walls.whole_pattern, game.pattern_words),
                   1: pack_rows(coins.whole_pattern, game.pattern_words)}
  game.pattern_mutable = {0: False, 1: True}
  game.drapes = np.array([_scrolly_record(walls), _scrolly_record(coins, -1, -1)],
                         dtype=np.int32)
  game.plot = np.array(_plot_record(aux0=int(coins.whole_pattern.sum())), dtype=np.int32)
  return game
