"""Oracle restatement of examples/research/lp-rnn/t_maze.py:180-505.  TEST INFRASTRUCTURE ONLY.

A cue, a teleporter into limbo and then into the hallway of the level, two goal pads.  Every
Scrolly "teleports" by np.roll of its own pattern at the start of its own update; rewards are
Python floats.  Same shape as `oracle.games`: a builder (`make_t_maze`) that turns the art
into an `engine_model.World` the way `make_game` does, and a program (`t_maze_program`) =
the `update()` of the entity that paints a character.
"""

import numpy as np

from oracle import engine_model as em
from oracle.games import art_to_array, mask_position, split_art

T_MAZE_LIMBO = (4, 140)           # TeleporterDrape._limbo_row / _limbo_col, :408-409
T_MAZE_DX = -46                   # :412


def make_t_maze(maze_art, cue_art, level, cue_after_teleport, timeout_frames=-1,
                teleport_delay=0, limbo_time=10, rng=None, np_rng=None):
  """t_maze.py:180-217 with Scrolly.PatternInfo inlined.  `rng` stands for Python's `random`
  module (the cue side, :262), `np_rng` for NumPy's global RandomState (the speckle, :365);
  either may be None for a template without that draw (cue 'left', speckle left whole)."""
  world_art = art_to_array(maze_art)
  marks = np.argwhere(world_art == ord('+'))
  assert len(marks) == 1
  corner = (int(marks[0][0]), int(marks[0][1]))
  world_art[corner] = ord(' ')
  board_shape = (len(cue_art), len(cue_art[0]))
  backdrop, masks = split_art(cue_art, ['Q'], ' ')
  things = {}
  for ch in '#*tlr':
    things[ch] = em.Scrolly(ch, board_shape, world_art == ord(ch), corner, margins=None)
  if np_rng is not None:                                               # SpeckleDrape :365
    dirt = things['*']
    dirt.pattern[np_rng.rand(*dirt.pattern.shape) < 0.4] = False
    em.scrolly_refresh(dirt)
  tele = things['t']
  tele.aux.update(delay=teleport_delay, countdown=limbo_time, in_limbo=False,
                  dy=11 * level + 9)
  if teleport_delay > 0:                                               # :397-400
    tele.aux['saved'] = tele.pattern.copy()
    tele.pattern[:] = False
    em.scrolly_refresh(tele)
  if tele.aux['dy'] + 5 > tele.pattern.shape[0]:
    raise ValueError('There is no {} difficulty level.'.format(level))
  for ch, name in (('l', 'left'), ('r', 'right')):
    things[ch].aux['name'] = name
  cue = em.PlainDrape('Q', masks['Q'])
  cue.aux['which_goal'] = 'left' if (rng is None or rng.random() < 0.5) else 'right'
  if cue.aux['which_goal'] == 'left':                                  # :263-266
    cue.curtain[:, 6:] = False
  else:
    cue.curtain[:, :6] = False
  cue.aux['cue_after_teleport'] = bool(cue_after_teleport)
  things['Q'] = cue
  where = np.argwhere(world_art == ord('P'))
  assert len(where) == 1
  p = em.Walker('P', board_shape, mask_position(np.zeros(board_shape, dtype=bool)),
                impassable='#', egocentric=True)                       # :223-227
  em.walker_teleport(p, int(where[0][0]) - corner[0], int(where[0][1]) - corner[1])
  things['P'] = p
  world = em.World(board_shape[0], board_shape[1], backdrop, things, z_order='*#ltrQP',
                   groups=[['Q', '#', '*'], ['P'], ['l', 't', 'r']], program=t_maze_program)
  world.plot.store['timeout_frames'] = float('inf') if timeout_frames < 0 else timeout_frames
  return world


def _t_maze_staying(plot):
  """0 <= frame - teleportation_order_frame <= 1 (:232 and every drape)."""
  return 0 <= plot.frame - plot.store.get('teleportation_order_frame', -1) <= 1


_T_MAZE_MOTION = {1: em.M_N, 2: em.M_S, 3: em.M_W, 4: em.M_E, 5: em.M_STAY}


def t_maze_program(world, ch, actions):
  plot, store, ent = world.plot, world.plot.store, world.things[ch]
  frame = plot.frame
  if ch == 'Q':                                   # CueDrape.update :271-283
    if not ent.aux['cue_after_teleport'] and store.get('yo_we_have_teleported'):
      del store['yo_we_have_teleported']
      ent.curtain[:] = False
    if frame >= store['timeout_frames']:
      plot.terminate_episode()
    elif frame > 1:
      plot.add_reward(-0.001)
    return
  if ch == 'P':                                   # PlayerSprite.update :229-245
    if _t_maze_staying(plot):
      em.walker_move(ent, world.board, plot, em.M_STAY)
    elif actions in _T_MAZE_MOTION:
      em.walker_move(ent, world.board, plot, _T_MAZE_MOTION[actions])
    elif actions in (0, 6):
      store['timeout_frames'] = frame + 1
    return
  # PseudoTeleportingScrolly.update :315-320: obey an order placed for this frame
  if store.get('teleportation_order_frame', -1) == frame:
    rows, cols = store['teleportation_order']
    ent.pattern[:] = np.roll(ent.pattern, -rows, axis=0)
    ent.pattern[:] = np.roll(ent.pattern, -cols, axis=1)
    ent.aux['rolled'] = True
  if ch in 'lr':                                  # GoalDrape.update :480-492
    ppos = em.scrolly_prescroll(ent, world.things['P'].position, plot)
    if ent.pattern[ppos] and frame < store['timeout_frames']:
      plot.add_reward(1.0 if ent.aux['name'] == world.things['Q'].aux['which_goal'] else -1.0)
      store['timeout_frames'] = frame + 1
  if ch == 't' and ent.aux['delay'] > 0:          # :425-428
    ent.aux['delay'] -= 1
    if ent.aux['delay'] <= 0:
      assert not ent.aux.get('rolled'), 'the teleporter rolled before it was shown'
      ent.pattern[:] = ent.aux['saved']
  if _t_maze_staying(plot):
    motion = em.M_STAY
  else:
    motion = _T_MAZE_MOTION.get(actions, em.M_STAY if ch == 't' else None)
  if motion is not None:
    em.scrolly_move(ent, world, motion)
  if ch != 't':
    return
  aux, p = ent.aux, world.things['P']             # TeleporterDrape :446-468
  if not store.get('yo_we_have_teleported'):
    ppos = em.scrolly_postscroll(ent, p.position, plot)
    if ent.pattern[ppos]:
      store['yo_we_have_teleported'] = True
      if aux['countdown'] <= 0:
        _t_maze_order(plot, aux['dy'], 0)
      else:
        aux['in_limbo'] = True
        _t_maze_order(plot, T_MAZE_LIMBO[0] - ppos[0], T_MAZE_LIMBO[1] - ppos[1])
  if aux['in_limbo']:
    aux['countdown'] -= 1
    if aux['countdown'] == 0:
      aux['in_limbo'] = False
      _t_maze_order(plot, aux['dy'], T_MAZE_DX)


def _t_maze_order(plot, rows, cols):              # place_teleportation_order :322-331
  plot.store['teleportation_order_frame'] = plot.frame + 1
  plot.store['teleportation_order'] = (rows, cols)
