"""examples/research/box_world/box_world.py on `csrc/box_world.cu`.

The keys, locks and the gem are Drapes upstream, but never share a cell, so the device keeps
them as one per-env object grid (`pcl_state.d_bits[0]` as u8 [rows, pitch]: the character,
bit 7 on a distractor lock) and the spec has no drapes at all.  Levels of one grid size and
step limit therefore share one `signature()`, whichever key colours they use.  The grid's
characters are the lowered game's `object_chars`; the hooks below turn it back into
curtains, layers and the facade's Drapes.
"""

import numpy as np

from pycolab_b200 import _lib
from pycolab_b200 import levels
from pycolab_b200 import lowering
from pycolab_b200 import things
from pycolab_b200.errors import NotLoweredError
from pycolab_b200.lowering import (LoweredGame, _common, _plot_record, _set_sprites,
                                   _sprite_record)

KEYS, LOCKS = levels.BOX_WORLD_KEYS, levels.BOX_WORLD_LOCKS
DISTRACTOR = 0x80                # grid bit of a lock cell listed in PlayerSprite.distractors
OBJECTS = {'gem': '*', 'key': KEYS, 'lock': LOCKS}


def _check_box_thing(cls):
  """The objects' drapes run BoxThing.is_locked_at and where_player_over_me (box_world.py:
  205-229): a class outside this package must inherit them from a BoxThing whose source is
  the reference's."""
  for klass in cls.__mro__:
    if (klass.__module__.rsplit('.', 1)[-1], klass.__name__) == ('box_world', 'BoxThing'):
      if not lowering._is_known_implementation(klass, ('box_world', 'BoxThing')):
        raise NotLoweredError(
            'class {}.BoxThing is named like the lowered class box_world.BoxThing but its source '
            'differs from the implementation the device program restates'.format(klass.__module__))
      for name in ('is_locked_at', 'where_player_over_me'):
        if getattr(cls, name, None) is not getattr(klass, name, None):
          raise NotLoweredError('{} overrides BoxThing.{}'.format(cls.__name__, name))
      return
  raise NotLoweredError('box_world object class {} does not derive from BoxThing'.format(
      cls.__name__))


def lower(engine, roles):
  """box_world.py:127-271: the player '.' and one Drape per object character, in one update
  group ['.', sorted objects] and z-order sorted objects + '.'."""
  th = engine.things
  if roles.get('.') != 'box_world.player':
    raise NotLoweredError("box_world program needs its PlayerSprite on '.' (got {})".format(roles))
  objects = ''.join(sorted(ch for ch in roles if ch != '.'))
  for ch in objects:
    kind = roles[ch].split('.')[1]
    if kind not in OBJECTS or ch not in OBJECTS[kind]:
      raise NotLoweredError('box_world {} on {!r}: keys are a-t, locks A-T, the gem *'.format(
          kind, ch))
    _check_box_thing(type(th[ch]))
  game = LoweredGame()
  _common(engine, game, _lib.PROG_BOX_WORLD)
  if game.groups != ['.' + objects] or game.z_order != objects + '.':
    raise NotLoweredError("box_world program needs update groups ['.', sorted objects] and "
                          "z-order sorted objects + '.'")
  if engine.rows > 32 or engine.cols > 32:
    raise NotLoweredError('box_world program: boards up to 32 x 32 (one lane per row)')
  ring = np.concatenate([game.backdrop[0, :game.cols], game.backdrop[-1, :game.cols],
                         game.backdrop[:, 0], game.backdrop[:, game.cols - 1]])
  if engine.rows < 3 or engine.cols < 3 or (ring != ord('#')).any():
    raise NotLoweredError("box_world program needs a '#' wall around the board")
  player = th['.']
  _set_sprites(game, [player], [_sprite_record(player, aux0=player._step_counter)])
  if not game.confined[0] or game.egocentric[0]:
    raise NotLoweredError('box_world player: a confined, non-egocentric MazeWalker')
  grid = np.zeros((game.rows, game.pitch), dtype=np.uint8)
  for ch in objects:
    cells = np.asarray(th[ch].curtain, dtype=bool)
    if grid[:, :game.cols][cells].any():
      raise NotLoweredError('box_world objects share a cell ({!r})'.format(ch))
    grid[:, :game.cols][cells] = ord(ch)
  for x, y in player.distractors:
    if 0 <= y < game.rows and 0 <= x < game.cols and chr(grid[y, x]) in LOCKS:
      grid[y, x] |= DISTRACTOR
  game.z_order, game.groups = '.', ['.']
  game.object_chars = objects
  game.bits_words = game.pitch // 4
  game.bits = {0: grid.view('<u4').reshape(game.rows, game.bits_words)}
  game.drapes = np.zeros((0, _lib.DRAPE_WORDS), dtype=np.int32)
  over = engine.the_plot.get('over_this')
  char, at = 0, 0
  if over:
    char, (y, x) = ord(over[0]), over[1]
    at = int(y) << 16 | int(x)
  game.plot = np.array(_plot_record(aux0=char, aux1=at), dtype=np.int32)
  game.program_arg[0] = int(player._max_num_steps)
  game.reward_type = float
  game.curtain = curtain
  game.layers = layers
  game.sync = sync
  return game


def _objects(eng):
  """u8 [B, rows, pitch]: every env's object grid without the distractor bit."""
  import torch
  return eng.bits[0].view(torch.uint8).reshape(eng.batch, eng.rows, eng.pitch) & 0x7f


def curtain(eng, d):
  """Every object character's curtain is where the grid holds it."""
  import torch
  ch = (eng.drape_chars + eng.object_chars)[d]
  return _objects(eng).eq(ord(ch)).to(torch.uint8)


def layers(eng, chars):
  """Un-occluded layers: backdrop cells, grid cells and the player's cell of each char."""
  import torch
  backdrop = eng.backdrop[eng.level_rows(eng.backdrop), :, :eng.cols]
  grid = _objects(eng)[:, :, :eng.cols]
  rec = eng.sprites[:, 0].long()
  shown = torch.nonzero(rec[:, _lib.S_FLAGS] & 1, as_tuple=True)[0]
  planes = []
  for ch in chars:
    plane = backdrop.eq(ord(ch)) | grid.eq(ord(ch))
    if ch in eng.sprite_chars:
      plane[shown, rec[shown, _lib.S_ROW], rec[shown, _lib.S_COL]] = True
    planes.append(plane)
  return torch.stack(planes, dim=1)


def sync(engine):
  """Every object Drape's curtain, the player's `_step_counter` and the_plot['over_this'],
  from env 0."""
  b = engine.batched
  grid = _objects(b)[0, :, :b.cols].cpu().numpy()
  for ch in b.object_chars:
    np.copyto(engine.things[ch].curtain, grid == ord(ch))
  engine.things['.']._step_counter = int(b.sprites[0, 0, _lib.S_AUX0])
  words = b.plot[0].cpu().numpy()
  if words[_lib.P_AUX0]:
    at = int(words[_lib.P_AUX1])
    engine.the_plot['over_this'] = (chr(int(words[_lib.P_AUX0])),
                                    things.Sprite.Position(at >> 16, at & 0xffff))
  elif 'over_this' in engine.the_plot:
    del engine.the_plot['over_this']
