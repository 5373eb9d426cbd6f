"""examples/aperture.py on `csrc/aperture.cu`."""

import numpy as np

from pycolab_b200 import _lib
from pycolab_b200.errors import NotLoweredError
from pycolab_b200.lowering import (LoweredGame, _common, _drape_record, _plot_record,
                                   _set_sprites, _sprite_record)


def lower(engine, roles):
  """examples/aperture.py:188-196: sprite 'A' + the aperture drape.  The drape's
  state is its `_apertures` list (at most two cells) in the record's AUX words."""
  players = [c for c, r in roles.items() if r == 'aperture.player']
  drapes = [c for c, r in roles.items() if r == 'aperture.drape']
  if len(players) != 1 or len(drapes) != 1 or len(roles) != 2:
    raise NotLoweredError('aperture program needs one player and one aperture drape '
                          '(got {})'.format(roles))
  game = LoweredGame()
  _common(engine, game, _lib.PROG_APERTURE)
  player, drape = engine.things[players[0]], engine.things[drapes[0]]
  if game.z_order != drapes[0] + players[0] or game.groups != [players[0], drapes[0]]:
    raise NotLoweredError('aperture program needs update groups [[player], [drape]] and the '
                          'player drawn over the drape')
  if drape.curtain.any() or list(drape._apertures) != [None, None]:
    raise NotLoweredError('the aperture drape must start with no apertures')
  if game.rows * game.pitch > 8192:
    raise NotLoweredError('aperture boards are staged whole in shared memory (<= 8 KiB)')
  _set_sprites(game, [player], [_sprite_record(player)])
  game.drape_chars = drapes[0]
  game.margins = [(-1, -1)]
  game.drapes = np.array([_drape_record(aux0=-1, aux1=-1)], dtype=np.int32)
  game.plot = np.array(_plot_record(), dtype=np.int32)
  game.curtain = curtain
  game.sync = sync
  return game


def curtain(eng, d):
  """ApertureDrape curtain = the (at most two) cells of its `_apertures` list."""
  import torch
  out = torch.zeros((eng.batch, eng.rows, eng.pitch), dtype=torch.uint8, device=eng.device)
  for word in (_lib.D_AUX0, _lib.D_AUX1):
    cell = eng.drapes[:, d, word]
    b = torch.nonzero(cell >= 0, as_tuple=True)[0]
    out[b, (cell[b] >> 16).long(), (cell[b] & 0xffff).long()] = 1
  return out


def sync(engine):
  """ApertureDrape._apertures of env 0."""
  rec = engine.batched.drapes[0, 0].cpu().numpy()
  cells = [int(rec[_lib.D_AUX0]), int(rec[_lib.D_AUX1])]
  engine.things[engine.batched.drape_chars[0]]._apertures = [
      None if c < 0 else (c >> 16, c & 0xffff) for c in cells]
