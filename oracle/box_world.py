"""Oracle restatement of examples/research/box_world/box_world.py:127-271.  TEST INFRASTRUCTURE ONLY.

Keys open the locks of their colour; a chain of boxes leads to the gem; a distractor lock
ends the episode.  Same shape as `oracle.games`: a builder (`make_box_world`) that turns a
level into an `engine_model.World` as `make_game` does — one plain drape per object
character, one update group ['.', sorted objects] — and a program (`box_world_program`) =
the `update()` of the entity that paints a character.  Rewards are Python floats.
"""

import numpy as np

from oracle import engine_model as em
from oracle.games import mask_position, split_art

KEYS = 'abcdefghijklmnopqrst'
LOCKS = KEYS.upper()
_MOTION = {0: em.M_N, 1: em.M_S, 2: em.M_W, 3: em.M_E}      # ACTION_MAP, :119-124


def make_box_world(art, distractors, max_num_steps=120):
  """box_world.py:380-415 from a generated level (`levels.box_world_level`): `distractors`
  lists the (column, row) of each distractor lock."""
  objects = sorted(set(''.join(art)) - set('.# '))
  backdrop, masks = split_art(art, objects + ['.'], ' ')
  shape = backdrop.shape
  things = {ch: em.PlainDrape(ch, masks[ch]) for ch in objects}
  player = em.Walker('.', shape, mask_position(masks['.']), impassable='#', confined=True)
  player.aux.update(steps=0, max_steps=max_num_steps,
                    distractors=[(int(x), int(y)) for x, y in distractors])
  things['.'] = player
  return em.World(shape[0], shape[1], backdrop, things, z_order=objects + ['.'],
                  groups=[['.'] + objects], program=box_world_program)


def _move(world, player, motion):
  em.walker_move(player, world.board, world.plot, motion)


def box_world_program(world, ch, actions):
  plot, store, board = world.plot, world.plot.store, world.board
  if ch == '.':                                   # PlayerSprite.update :163-202
    if actions not in range(4):
      return
    plot.add_reward(0.0)
    p, motion = world.things['.'], _MOTION[actions]
    dr, dc = em.MOTIONS[motion]
    y, x = p.row + dr, p.col + dc
    char = chr(board[y, x])
    thing = None if char == '#' else world.things.get(char)
    held = chr(board[0, 0])
    if not thing:
      _move(world, p, motion)
    else:
      is_lock = char in LOCKS
      if is_lock and held == KEYS[LOCKS.index(char)]:
        _move(world, p, motion)
      locked = any(c in LOCKS and world.things[c].curtain[y, x + 1] for c in world.things)
      if not is_lock and not locked:
        _move(world, p, motion)
    p.aux['steps'] += 1
    if p.aux['steps'] > p.aux['max_steps']:
      plot.terminate_episode()
    if thing:
      store['over_this'] = (char, (p.row, p.col))
    return
  ent = world.things[ch]                          # BoxThing.where_player_over_me :221-229
  over = store.get('over_this')
  if not over:
    return
  char, (y, x) = over
  if char != ch or not ent.curtain[y, x]:
    return
  held = chr(board[0, 0])
  if ch == '*':                                   # GemDrape :235-238
    plot.add_reward(10.0)
    plot.terminate_episode()
  elif ch in KEYS:                                # KeyDrape :244-251
    if held in KEYS:
      world.things[held].curtain[0, 0] = False
    ent.curtain[y, x] = False
    ent.curtain[0, 0] = True
  else:                                           # LockDrape :261-271
    ent.curtain[y, x] = False
    world.things[held].curtain[0, 0] = False
    if (x, y) in world.things['.'].aux['distractors']:
      plot.add_reward(-1.0)
      plot.terminate_episode()
    else:
      plot.add_reward(1.0)


def over_this(world):
  """the_plot['over_this'] of an oracle world, or None."""
  return world.plot.store.get('over_this')
