"""examples/shockwave.py on `csrc/shockwave.cu`."""

import numpy as np

from pycolab_b200 import _lib
from pycolab_b200.errors import NotLoweredError
from pycolab_b200.lowering import (LoweredGame, _common, _drape_record, _plot_record,
                                   _set_sprites, _sprite_record, _update_order, pack_rows)


def lower(engine, roles):
  """examples/shockwave.py:91-197: the player, the ShockwaveDrape and the two static
  MinimalDrapes the wave's update() names by character (' ' danger zone, '^' safe
  zone; walls are the backdrop's '=')."""
  th = engine.things
  by_role = {}
  for ch, role in roles.items():
    by_role.setdefault(role, []).append(ch)
  if (sorted(by_role) != ['shockwave.minimal', 'shockwave.player', 'shockwave.wave'] or
      len(by_role['shockwave.player']) != 1 or len(by_role['shockwave.wave']) != 1 or
      sorted(by_role['shockwave.minimal']) != [' ', '^']):
    raise NotLoweredError("shockwave program needs one PlayerSprite, one ShockwaveDrape and "
                          "MinimalDrapes ' ' and '^' (got {})".format(roles))
  p_ch, w_ch = by_role['shockwave.player'][0], by_role['shockwave.wave'][0]
  game = LoweredGame()
  _common(engine, game, _lib.PROG_SHOCKWAVE)
  order = _update_order(engine)
  if len(game.groups) != 1 or sorted(order[:2]) != [' ', '^'] or order[2:] != [p_ch, w_ch]:
    raise NotLoweredError("shockwave program needs update_schedule [' ', '^', P, wave]")
  if game.z_order != ' ^' + w_ch + p_ch:
    raise NotLoweredError("shockwave program needs z_order [' ', '^', wave, P]")
  pl, wave = th[p_ch], th[w_ch]
  if set(pl.impassable) != {'='}:
    raise NotLoweredError("the wave's update() stops at '=': the player must do the same")
  if '=' not in engine.backdrop.palette:
    raise NotLoweredError("the wave's update() reads layers['='], which holds only characters "
                          "of the backdrop: with no '=' in the art the reference raises "
                          "KeyError at its_showtime()")
  if engine.rows > 32 or engine.cols > 64:
    raise NotLoweredError('shockwave program: boards up to 32 x 64')
  _set_sprites(game, [pl], [_sprite_record(pl)])
  game.drape_chars = w_ch + ' ^'
  game.margins = [(-1, -1)] * 3
  recs = [_drape_record(aux1=wave._steps_since_impact), _drape_record(), _drape_record()]
  if wave.curtain.any() or np.any(wave._distance_from_impact):
    raise NotLoweredError('a ShockwaveDrape that is already burning is not lowered')
  game.drapes = np.array(recs, dtype=np.int32)
  for d, ch in enumerate(game.drape_chars):
    game.bits[d] = pack_rows(th[ch].curtain, game.bits_words)
  game.plot = np.array(_plot_record(), dtype=np.int32)
  game.program_arg[0] = int(wave._width)
  game.rng_streams = ('numpy',)     # np.random.randint, shockwave.py:133
  return game
