"""The general program `csrc/fixture.cu`: MazeWalkers, Scrollys and plain Drapes of the
reference's test fixtures (`games/fixtures.py`), with Plot directives in the action row."""

import numpy as np

from pycolab_b200 import _lib
from pycolab_b200.errors import NotLoweredError
from pycolab_b200.lowering import (LoweredGame, _common, _drape_record, _plot_record,
                                   _scrolly_record, _set_sprites, _sprite_record, pack_rows,
                                   round_up)


def lower(engine, roles):
  th = engine.things
  game = LoweredGame()
  _common(engine, game, _lib.PROG_FIXTURE, never_reads_layers=True)
  order = ''.join(game.groups)
  sprite_chars = [c for c in order if roles[c] == 'fixture.walker']
  drape_chars = [c for c in order if roles[c] != 'fixture.walker']
  if len(sprite_chars) > _lib.MAX_SPRITES or len(drape_chars) > _lib.MAX_DRAPES:
    raise NotLoweredError('too many entities for the general device program')
  sprites = [th[c] for c in sprite_chars]
  _set_sprites(game, sprites, [_sprite_record(s, aux0=0, aux1=_lib.NEVER) for s in sprites],
               named_groups=True)
  # Scrolling groups (protocols/scrolling.py:198-241): one device record per name.
  names = []
  for ch in order:
    name = getattr(th[ch], '_scrolling_group', None)
    if name is not None and name not in names:
      names.append(name)
  names = names or ['']
  if len(names) > _lib.MAX_SCROLL_GROUPS:
    raise NotLoweredError('more than {} scrolling groups'.format(_lib.MAX_SCROLL_GROUPS))
  game.scroll_groups = names
  game.sprite_group = [names.index(th[c]._scrolling_group) for c in sprite_chars]
  game.drape_group = [names.index(getattr(th[c], '_scrolling_group', names[0]))
                      for c in drape_chars]
  game.group_records = np.zeros((_lib.MAX_SCROLL_GROUPS, _lib.GROUP_WORDS), dtype=np.int32)
  game.group_records[:, _lib.G_ORDER_FRAME] = _lib.NEVER
  game.drape_chars = ''.join(drape_chars)
  game.drape_kind, game.margins, recs = [], [], []
  shape = None
  for d, ch in enumerate(drape_chars):
    ent = th[ch]
    if roles[ch] == 'fixture.scrolly':
      if shape not in (None, ent.whole_pattern.shape):
        raise NotLoweredError('Scrolly patterns of different shapes')
      shape = ent.whole_pattern.shape
      game.drape_kind.append(1)
      game.margins.append((-1, -1) if ent._scroll_margins is None
                          else tuple(ent._scroll_margins))
      recs.append(_scrolly_record(ent))
    else:
      game.drape_kind.append(0)
      game.margins.append((-1, -1))
      recs.append(_drape_record())
      game.bits[d] = pack_rows(ent.curtain, game.bits_words)
  if shape is not None:
    game.pattern_rows, game.pattern_cols = shape
    game.pattern_words = round_up((shape[1] + 31) // 32 + 3, 2)
    for d, ch in enumerate(drape_chars):
      if game.drape_kind[d]:
        game.patterns[d] = pack_rows(th[ch].whole_pattern, game.pattern_words)
        game.pattern_mutable[d] = False
  game.drapes = np.array(recs, dtype=np.int32).reshape(len(drape_chars), _lib.DRAPE_WORDS)
  game.plot = np.array(_plot_record(), dtype=np.int32)
  game.dynamic_z = True
  # one motion word per entity, then (opcode, argument) pairs of Plot directives
  game.actions_per_env = (len(game.sprite_chars) + len(game.drape_chars) +
                          2 * _lib.FIXTURE_DIRECTIVES)
  game.action_row = action_row
  return game


_MOTION_NAMES = ('n', 'ne', 'e', 'se', 's', 'sw', 'w', 'nw')


def action_row(engine, actions):
  """General-program action row from the fixture conventions
  (tests/test_things.py:219-250): a direction string for everybody, or
  {char: direction}; unknown / missing = stay.  Directive keys '_reward',
  '_terminate', '_z' — or '_directives', an ordered list of Plot calls such as
  ('terminate_episode', 0.5) — stand in for post_update code injection."""
  from pycolab_b200.games import fixtures
  code = lambda d: _MOTION_NAMES.index(d) if d in _MOTION_NAMES else 8
  game = engine.batched.game
  order = ''.join(game.groups)
  if isinstance(actions, dict):
    motions = {ch: code(actions.get(ch)) for ch in order}
    return fixtures.action_rows(game, motions, actions.get('_reward'),
                                bool(actions.get('_terminate')), actions.get('_z'),
                                directives=actions.get('_directives'))
  return fixtures.action_rows(game, {ch: code(actions) for ch in order})
