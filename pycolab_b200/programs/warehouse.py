"""examples/warehouse_manager.py on `csrc/warehouse.cu`."""

import numpy as np

from pycolab_b200 import _lib
from pycolab_b200.errors import NotLoweredError
from pycolab_b200.lowering import (LoweredGame, _common, _drape_record, _plot_record,
                                   _set_sprites, _sprite_record)


def lower(engine, roles):
  th = engine.things
  groups = [[e.character for e in ents]
            for _, ents in sorted(engine._update_groups.items())]
  if len(groups) != 3 or groups[1] != ['X'] or groups[2] != ['P']:
    raise NotLoweredError('warehouse program needs update groups [boxes, [X], [P]]')
  boxes = groups[0]
  for ch in boxes:
    if roles.get(ch) != 'warehouse.box':
      raise NotLoweredError('unexpected entity {!r} in the box group'.format(ch))
  if roles.get('X') != 'warehouse.judge' or roles.get('P') != 'warehouse.player':
    raise NotLoweredError('warehouse program needs JudgeDrape X and PlayerSprite P')
  game = LoweredGame()
  _common(engine, game, _lib.PROG_WAREHOUSE)
  sprites = [th[c] for c in boxes] + [th['P']]
  _set_sprites(game, sprites, [_sprite_record(s) for s in sprites])
  judge = th['X']
  if judge.curtain.any():
    raise NotLoweredError("a pre-filled 'X' curtain is not lowered")
  game.drape_chars = 'X'
  game.margins = [(-1, -1)]
  game.drapes = np.array([_drape_record(aux0=judge._last_num_boxes_on_goals)], dtype=np.int32)
  game.plot = np.array(_plot_record(), dtype=np.int32)
  if '_' not in engine.backdrop.palette:
    raise NotLoweredError("warehouse backdrop has no goal character '_'")
  game.curtain = curtain
  return game


def curtain(eng, d):
  """JudgeDrape curtain = cells of boxes currently drawn as 'X'."""
  import torch
  out = torch.zeros((eng.batch, eng.rows, eng.pitch), dtype=torch.uint8, device=eng.device)
  nb = len(eng.sprite_chars) - 1
  rec = eng.sprites[:, :nb]
  on = rec[:, :, _lib.S_AUX0] != 0
  b, s = torch.nonzero(on, as_tuple=True)
  out[b, rec[b, s, _lib.S_ROW].long(), rec[b, s, _lib.S_COL].long()] = 1
  return out
