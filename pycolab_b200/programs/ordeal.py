"""examples/ordeal.py on `csrc/ordeal.cu`."""

import numpy as np

from pycolab_b200 import _lib
from pycolab_b200 import things
from pycolab_b200.errors import NotLoweredError
from pycolab_b200.lowering import (LoweredGame, _common, _drape_record, _plot_record,
                                   _set_sprites, _sprite_record, pack_rows)

_CHAPTERS = {'castle': _lib.ORDEAL_CASTLE, 'cavern': _lib.ORDEAL_CAVERN,
             'kansas': _lib.ORDEAL_KANSAS}
_CHAPTER_NAMES = {v: k for k, v in _CHAPTERS.items()}


def lower(engine, roles):
  """examples/ordeal.py:74-266: one chapter of the Story.  Which chapter this Engine
  is comes from its entities (castle: P + D, cavern: P + S, kansas: P) and must agree
  with `the_plot.this_chapter`, which Story set before its_showtime()
  (storytelling.py:453-454).  The Plot entries the game code keeps in dict slots —
  `has_sword`, `last_position` — and the chapter bookkeeping enter the device plot
  record here and are mirrored back after every step (`sync`)."""
  th, plot = engine.things, engine.the_plot
  by_role = sorted(roles.values())
  chapter = {('ordeal.dragonduck', 'ordeal.player'): 'castle',
             ('ordeal.player', 'ordeal.sword'): 'cavern',
             ('ordeal.player',): 'kansas'}.get(tuple(by_role))
  if chapter is None:
    raise NotLoweredError('ordeal program: unknown chapter with entities {}'.format(roles))
  if plot.this_chapter is not None and plot.this_chapter != chapter:
    raise NotLoweredError('ordeal chapter {!r} is running under the Story key {!r}'.format(
        chapter, plot.this_chapter))
  if plot.prior_chapter is not None and plot.prior_chapter not in _CHAPTERS:
    raise NotLoweredError('ordeal chapter entered from an unknown chapter {!r}'.format(
        plot.prior_chapter))
  game = LoweredGame()
  _common(engine, game, _lib.PROG_ORDEAL)
  if len(game.groups) != 1:
    raise NotLoweredError('ordeal chapters have one update group')
  player = [c for c, r in roles.items() if r == 'ordeal.player'][0]
  sprites = [th[player]] + [th[c] for c, r in roles.items() if r == 'ordeal.dragonduck']
  if game.groups[0][0] != player:
    raise NotLoweredError('the ordeal player must update first')
  if game.rows * game.pitch > 8192:
    raise NotLoweredError('ordeal boards are staged whole in shared memory (<= 8 KiB)')
  _set_sprites(game, sprites, [_sprite_record(s) for s in sprites])
  game.program_arg[0] = _CHAPTERS[chapter]
  drapes = [c for c, r in roles.items() if r == 'ordeal.sword']
  game.drape_chars = ''.join(drapes)
  game.margins = [(-1, -1)] * len(drapes)
  game.drapes = np.array([_drape_record() for _ in drapes],
                         dtype=np.int32).reshape(len(drapes), _lib.DRAPE_WORDS)
  for d, ch in enumerate(drapes):
    game.bits[d] = pack_rows(th[ch].curtain, game.bits_words)
  last = plot.get('last_position')
  game.plot = np.array(_plot_record(
      aux0=1 if plot.get('has_sword') else 0,
      aux1=-1 if last is None else (int(last[0]) << 16) | int(last[1]),
      aux2=_lib.ORDEAL_NEXT_UNSET,
      aux3=_CHAPTERS.get(plot.prior_chapter, 0)), dtype=np.int32)
  game.dynamic_z = len(sprites) + len(drapes) == 2      # the kernel reads (castle: rewrites) it
  game.reward_type = float                              # ordeal.py pays 1.0 / -1.0
  game.sync = sync
  return game


def sync(engine):
  """The Plot's `has_sword`, `last_position` and next chapter from env 0's plot record."""
  p, words = engine.the_plot, engine.batched.plot[0].cpu().numpy()
  if words[_lib.P_AUX0]:
    p['has_sword'] = True
  if words[_lib.P_AUX1] >= 0:
    p['last_position'] = things.Sprite.Position(int(words[_lib.P_AUX1]) >> 16,
                                                int(words[_lib.P_AUX1]) & 0xffff)
  if words[_lib.P_AUX2] != _lib.ORDEAL_NEXT_UNSET:
    p.next_chapter = _CHAPTER_NAMES.get(int(words[_lib.P_AUX2]))   # 0 -> None: the story ends
