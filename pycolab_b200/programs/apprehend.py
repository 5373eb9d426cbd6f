"""examples/apprehend.py on `csrc/apprehend.cu`."""

import numpy as np

from pycolab_b200 import _lib
from pycolab_b200.errors import NotLoweredError
from pycolab_b200.lowering import (LoweredGame, _common, _plot_record, _set_sprites,
                                   _sprite_record, _update_order)


def _f64_words(x):
  """float64 -> (lo, hi) int32 words, as the kernels' __hiloint2double reads them."""
  lo, hi = np.array([x], dtype='<f8').view('<i4')
  return int(lo), int(hi)


def lower(engine, roles):
  """examples/apprehend.py:56-131: the catcher 'P' and the falling ball, one group
  [ball, catcher].  The ball's float64 slope (drawn when the Python sprite was built)
  and accumulator travel as bit patterns; `needs_rng` lets a BATCHED engine draw a new
  slope per episode on the device from per-env `random.Random` states."""
  th = engine.things
  players = [c for c, r in roles.items() if r == 'apprehend.player']
  balls = [c for c, r in roles.items() if r == 'apprehend.ball']
  if len(players) != 1 or len(balls) != 1 or len(roles) != 2:
    raise NotLoweredError('apprehend program needs one PlayerSprite and one BallSprite')
  game = LoweredGame()
  _common(engine, game, _lib.PROG_APPREHEND)
  pl, ball = th[players[0]], th[balls[0]]
  if _update_order(engine) != [balls[0], players[0]] or len(game.groups) != 1:
    raise NotLoweredError('apprehend program needs update_schedule [ball, player]')
  if game.z_order != balls[0] + players[0]:
    raise NotLoweredError('apprehend program draws the player over the ball')
  lo, hi = _f64_words(ball._dx)
  _set_sprites(game, [pl, ball], [_sprite_record(pl), _sprite_record(ball, aux0=lo, aux1=hi)])
  alo, ahi = _f64_words(ball._x_accumulator)
  game.drape_chars = ''
  game.margins = []
  game.drapes = np.zeros((0, _lib.DRAPE_WORDS), dtype=np.int32)
  game.plot = np.array(_plot_record(aux0=alo, aux1=ahi), dtype=np.int32)
  game.rng_streams = ('python',)    # the global `random` (apprehend.py:103)
  return game
