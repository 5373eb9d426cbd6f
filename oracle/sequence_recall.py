"""Oracle restatement of examples/research/lp-rnn/sequence_recall.py:107-317.  TEST
INFRASTRUCTURE ONLY.

Four light pads flash a sequence while the player is held in the start box '%', then the
player must visit them in order.  Same shape as `oracle.t_maze`: a builder
(`make_sequence_recall`) and a program (`sequence_recall_program`).  `rng` stands for
Python's `random` module (the sequence, drawn by `make_program` as _make_program does).
The mask's `curtain -= mask` (NumPy 1 boolean subtraction, an XOR) always finds the light
covered, so it is restated as and-not.
"""

import numpy as np

from oracle import engine_model as em
from oracle.games import mask_position, split_art

LIGHTS = '1234'


def make_program(sequence_length, on, off, pause, rng):
  """_make_program (:160-188), states as their names."""
  sequence = [rng.choice(LIGHTS) for _ in range(sequence_length)]
  program = []
  for g in sequence:
    program += [('OFF', off), ('ON', on, g)]
  program.append(('OFF', max(1, pause)))
  for g in sequence:
    program += [('SEEK', g), ('EXIT',)]
  program[-1] = ('QUIT',)
  return program


def make_sequence_recall(art, sequence_length=4, demo_light_on_frames=60,
                         demo_light_off_frames=30, pause_frames=30, timeout_frames=-1, rng=None):
  """make_game (:130-157)."""
  program = make_program(sequence_length, demo_light_on_frames, demo_light_off_frames,
                         pause_frames, rng)
  backdrop, masks = split_art(art, ['P', 'M', '%'], ' ')
  shape = backdrop.shape
  player = em.Walker('P', shape, mask_position(masks['P']), impassable='#', confined=True)
  mask = em.PlainDrape('M', masks['M'])
  mask.aux['light'] = {g: backdrop == ord(g) for g in LIGHTS}       # _set_up_masks :206-211
  mask.aux['all_off'] = np.isin(backdrop, [ord(g) for g in LIGHTS])
  world = em.World(shape[0], shape[1], backdrop,
                   {'P': player, 'M': mask, '%': em.PlainDrape('%', masks['%'])},
                   z_order='MP%', groups=[['P', 'M', '%']], program=sequence_recall_program)
  store = world.plot.store
  store['program'] = program
  store['frames_in_state'] = 0
  store['timeout_frames'] = float('inf') if timeout_frames < 0 else timeout_frames
  return world


_MOTION = {1: em.M_N, 2: em.M_S, 3: em.M_W, 4: em.M_E, 5: em.M_STAY}


def sequence_recall_program(world, ch, actions):
  plot, store, ent = world.plot, world.plot.store, world.things[ch]
  state = store['program'][0]
  if ch == 'P':                                   # PlayerSprite.update :288-317
    if actions in (0, 6):
      store['timeout_frames'] = 1
    elif state[0] in ('SEEK', 'EXIT') and actions in _MOTION:
      em.walker_move(ent, world.board, plot, _MOTION[actions])
    if store['timeout_frames'] <= 0:
      plot.terminate_episode()
    else:
      if plot.frame > 1:
        plot.add_reward(-0.005)
      store['timeout_frames'] -= 1
    return
  if ch == '%':                                   # WaitForSeekDrape.update :268-271
    if store['frames_in_state'] == 1 and state[0] == 'SEEK' and ent.curtain.any():
      ent.curtain[:] = False
    return
  aux = ent.aux                                   # MaskDrape.update :213-262
  pos = world.things['P'].position
  store['frames_in_state'] += 1
  fis = store['frames_in_state']

  def pop():
    store['program'].pop(0)
    store['frames_in_state'] = 0
  if state[0] == 'QUIT':
    if fis == 1:
      store['timeout_frames'] = 1
  elif state[0] == 'OFF':
    if fis == 1:
      ent.curtain[:] |= aux['all_off']
    elif fis >= state[1]:
      pop()
  elif state[0] == 'ON':
    if fis == 1:
      ent.curtain[:] &= ~aux['light'][state[2]]
    elif fis >= state[1]:
      pop()
  elif state[0] == 'SEEK':
    above = chr(world.backdrop[pos])
    if above != ' ':
      ent.curtain[:] &= ~aux['light'][above]
      plot.add_reward(1.0 if above == state[1] else 0.0)
      pop()
  else:                                           # EXIT
    if chr(world.backdrop[pos]) == ' ':
      ent.curtain[:] |= aux['all_off']
      pop()
