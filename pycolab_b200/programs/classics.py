"""examples/classics (four_rooms, cliff_walk, chain_walk) and fluvial_natation on
`csrc/classics.cu`."""

import numpy as np

from pycolab_b200 import _lib
from pycolab_b200.errors import NotLoweredError
from pycolab_b200.lowering import (LoweredGame, _common, _plot_record, _set_sprites,
                                   _sprite_record)


def lower(engine, roles):
  """examples/classics: one MazeWalker 'P', no drapes; the rule set rides in
  pcl_spec.program_arg (four_rooms.py:78 fixes the goal cell at (4, 3))."""
  if list(roles) != ['P']:
    raise NotLoweredError('classics programs have exactly one entity, P (got {})'.format(roles))
  game = LoweredGame()
  _common(engine, game, _lib.PROG_CLASSICS)
  rule = roles['P'].split('.')[1]
  game.program_arg[0] = {'four_rooms': _lib.CLASSIC_FOUR_ROOMS,
                         'cliff_walk': _lib.CLASSIC_CLIFF_WALK,
                         'chain_walk': _lib.CLASSIC_CHAIN_WALK,
                         'fluvial': _lib.CLASSIC_FLUVIAL}[rule]
  if rule == 'four_rooms':
    game.program_arg[1], game.program_arg[2] = 4, 3
  if (rule == 'fluvial') != (game.backdrop_role == 'river'):
    raise NotLoweredError('the river Backdrop and the swimmer are lowered only together')
  if rule == 'fluvial':
    game.program_arg[1], game.program_arg[2] = 1, 4      # curtain[1:4, :], fluvial_natation.py:110
  if game.rows * game.pitch > 8192:
    raise NotLoweredError('classics boards are staged whole in shared memory (<= 8 KiB)')
  player = engine.things['P']
  _set_sprites(game, [player], [_sprite_record(player)])
  if rule == 'fluvial' and any(game.impassable[0]):
    raise NotLoweredError('the river program needs a swimmer with no impassable characters')
  game.drapes = np.zeros((0, _lib.DRAPE_WORDS), dtype=np.int32)
  game.plot = np.array(_plot_record(), dtype=np.int32)
  game.reward_type = int if rule == 'fluvial' else float
  if rule == 'fluvial':
    game.sync = sync_river
  return game


def sync_river(engine):
  """RiverBackdrop.update as a rotation count: rows program_arg[1]:program_arg[2] of the
  lowered backdrop rolled west by the plot's AUX0."""
  b = engine.batched
  r0, r1 = b.game.program_arg[1], b.game.program_arg[2]
  engine.backdrop.curtain[r0:r1] = np.roll(b.game.backdrop[r0:r1, :b.cols],
                                           -int(b.plot[0, _lib.P_AUX0]), axis=1)
