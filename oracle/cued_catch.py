"""Oracle restatement of examples/research/lp-rnn/cued_catch.py:96-317.  TEST INFRASTRUCTURE ONLY.

The catcher 'P' moves between rows 1 and 2, the balls 'a' / 'b' approach from the right once
the cue drape 'Q' has shown the four cue->ball pairings, and every frame pays.  Same shape as
`oracle.t_maze`: a builder (`make_cued_catch`) and a program (`cued_catch_program`).  `rng`
stands for Python's `random` module: the pairings (random.sample), every trial's cue
(random.randrange) and the reward noise (random.normalvariate) are CPython's own draws.
Where upstream compares None with ints, Python 2's order (None below everything) is kept.
"""

import numpy as np

from oracle import engine_model as em
from oracle.games import mask_position, split_art

NUM_CUES = 4


class Ball(object):
  """A plain Sprite (things.py:265-391) that remembers its start (cued_catch.py:170-179)."""
  is_sprite = True

  def __init__(self, char, position):
    self.char = char
    self.row, self.col = position
    self.start = position
    self.visible = False
    self.aux = {}

  @property
  def position(self):
    return (self.row, self.col)


def make_cued_catch(art, initial_cue_duration, cue_duration, num_trials,
                    always_show_ball_symbol=False, reward_sigma=0.0, reward_free_trials=0,
                    rng=None, pairings=None):
  """cued_catch.py:96-113 and the constructors; the pairings are rng.sample(...) unless
  given (a template whose drape drew them already)."""
  backdrop, masks = split_art(art, ['P', 'a', 'b', 'Q'], ' ')
  shape = backdrop.shape
  player = em.Walker('P', shape, mask_position(masks['P']), impassable='', confined=True)
  player.aux.update(sigma=reward_sigma, ttr=reward_free_trials, rng=rng)
  cue = em.PlainDrape('Q', masks['Q'])
  if pairings is None:
    pairings = rng.sample(['top'] * (NUM_CUES // 2) + ['bottom'] * (NUM_CUES // 2), NUM_CUES)
  cue.aux.update(icd=initial_cue_duration, cd=cue_duration, trials_left=num_trials,
                 always=always_show_ball_symbol, pairings=list(pairings), phase='first',
                 tick1=NUM_CUES * initial_cue_duration, choice=-1, tick2=-1,
                 last_reset=-float('inf'), rng=rng)
  things = {'P': player, 'a': Ball('a', mask_position(masks['a'])),
            'b': Ball('b', mask_position(masks['b'])), 'Q': cue}
  return em.World(shape[0], shape[1], backdrop, things, z_order='PabQ', groups=[['P', 'a', 'b', 'Q']],
                  program=cued_catch_program)


def _band(curtain, rows, cols=None):
  curtain[rows, :] = False
  if cols is not None:
    curtain[rows, cols] = True


def cued_catch_program(world, ch, actions):
  plot, store, ent = world.plot, world.plot.store, world.things[ch]
  if ch == 'P':                                   # PlayerSprite.update :136-167
    if actions == 1 and ent.vrow > 1:
      em.walker_move(ent, world.board, plot, em.M_N)
    elif actions == 2 and ent.vrow < 2:
      em.walker_move(ent, world.board, plot, em.M_S)
    elif actions in (0, 4):
      plot.terminate_episode()
    else:
      em.walker_move(ent, world.board, plot, em.M_STAY)
    ball = world.things['a' if store.get('which_ball') == 'top' else 'b']
    aux = ent.aux
    if aux['sigma']:
      if ent.col == ball.col and aux['ttr'] <= 0:
        plot.add_reward(float(ent.position == ball.position) +
                        aux['rng'].normalvariate(mu=0, sigma=aux['sigma']))
      else:
        plot.add_reward(0)
    else:
      plot.add_reward(int(ent.position == ball.position and aux['ttr'] <= 0))
    if ent.col == ball.col and aux['ttr'] > 0:
      aux['ttr'] -= 1
    return
  if ch in 'ab':                                  # BallSprite.update :181-194
    if not store.get('programming_complete'):
      return
    ent.visible = True
    if ent.col < world.things['P'].col:
      ent.row, ent.col = ent.start
      store['last_ball_reset'] = plot.frame
    else:
      ent.col -= 1
    return
  aux, c = ent.aux, ent.curtain                   # CueDrape.update :247-317
  _band(c, slice(1, 3))                           # _show_phase_cue
  if aux['phase'] == 'first':
    c[1:3, 0:2] = True
    c[1:3, -2:] = True

  def show_ball_symbol(ball):
    _band(c, slice(3, 5), slice(0, 6) if ball == 'top' else slice(-6, None)
          if ball == 'bottom' else None)

  def show_cue(cue):
    c[-2:, :] = False
    if cue is not None and 0 <= cue < NUM_CUES:   # None < 0 in Python 2
      width = c.shape[1] // NUM_CUES
      c[-2:, cue * width:cue * width + width] = True

  def second_phase_reset():
    aux['choice'] = aux['rng'].randrange(NUM_CUES)
    store['which_ball'] = aux['pairings'][aux['choice']]
    aux['tick2'] = aux['cd']
    aux['last_reset'] = plot.frame
    if aux['trials_left'] <= 0:
      plot.terminate_episode()
    aux['trials_left'] -= 1

  if aux['phase'] == 'first':
    aux['tick1'] -= 1
    cue = aux['tick1'] // aux['icd']
    show_ball_symbol(aux['pairings'][cue])
    show_cue(cue)
    if aux['tick1'] <= 0:
      aux['phase'] = 'second'
      store['programming_complete'] = True
      second_phase_reset()
  else:
    show_ball_symbol('neither')
    if store.get('last_ball_reset', -float('inf')) > aux['last_reset']:
      second_phase_reset()
    if aux['tick2'] > 0:
      show_cue(aux['choice'])
      if aux['always']:
        show_ball_symbol(aux['pairings'][aux['choice']])
    else:
      show_cue(None)
      show_ball_symbol(None)
    aux['tick2'] -= 1
