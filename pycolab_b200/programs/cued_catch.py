"""examples/research/lp-rnn/cued_catch.py on `csrc/cued_catch.cu`."""

import random

import numpy as np

from pycolab_b200 import _lib
from pycolab_b200.errors import NotLoweredError
from pycolab_b200.lowering import (LoweredGame, _common, _drape_record, _plot_record,
                                   _sprite_record, _walker_meta, pack_rows)
from pycolab_b200.programs.apprehend import _f64_words

_WHICH = {None: 0, 'top': 1, 'bottom': 2}


def _frame_word(x):
  """A frame number of the game, or -inf / None (never), as an int32 word."""
  if x is None or x == -float('inf'):
    return _lib.NEVER
  if not isinstance(x, (int, np.integer)) or not -2 ** 31 < x < 2 ** 31:
    raise NotLoweredError('cued_catch frame {!r} is not an int32 frame'.format(x))
  return int(x)


def _int32(x, what):
  if isinstance(x, bool) or not isinstance(x, (int, np.integer)) or not -2 ** 31 <= x < 2 ** 31:
    raise NotLoweredError('cued_catch {} must be an int32 integer (got {!r})'.format(what, x))
  return int(x)


def lower(engine, roles):
  """examples/research/lp-rnn/cued_catch.py:96-317: the catcher 'P', the balls 'a' / 'b' and
  the cue 'Q', one update group [P a b Q].  The pairings the Python CueDrape drew are in the
  template; update() draws from Python's `random` (slot 0), which a batched engine also uses
  to draw new pairings at every restart, and which the single-env facade continues from the
  global generator (`rng_from_globals`, `template_draws`)."""
  th, plot = engine.things, engine.the_plot
  want = {'P': 'cued_catch.player', 'a': 'cued_catch.ball', 'b': 'cued_catch.ball',
          'Q': 'cued_catch.cue'}
  if roles != want:
    raise NotLoweredError('cued_catch program needs exactly {} (got {})'.format(want, roles))
  game = LoweredGame()
  _common(engine, game, _lib.PROG_CUED_CATCH)
  if game.groups != ['PabQ'] or game.z_order != 'PabQ':
    raise NotLoweredError("cued_catch program needs update_schedule ['P', 'a', 'b', 'Q'] and "
                          "z-order 'PabQ'")
  if engine.rows > 32 or engine.cols > 64:
    raise NotLoweredError('cued_catch program: boards up to 32 x 64')
  player, cue = th['P'], th['Q']
  impassable, confined, egocentric = _walker_meta(player)
  if any(impassable) or not confined or egocentric:
    raise NotLoweredError('cued_catch player is confined and passes everything')
  icd = _int32(cue._initial_cue_duration, 'initial_cue_duration')
  if icd < 1:        # upstream divides by it (cued_catch.py:261)
    raise NotLoweredError('cued_catch initial_cue_duration must be >= 1 (got %d)' % icd)
  if icd > 1 << 28:
    raise NotLoweredError('cued_catch initial_cue_duration above 2^28')
  sigma = player._reward_sigma
  if isinstance(sigma, bool) or not isinstance(sigma, (int, float, np.floating, np.integer)):
    raise NotLoweredError('cued_catch reward_sigma must be a number')
  sigma = float(sigma)
  if sorted(cue._cues_to_balls) != ['bottom', 'bottom', 'top', 'top'] or cue._NUM_CUES != 4:
    raise NotLoweredError('cued_catch pairs four cues with two top and two bottom balls')
  if cue._phase not in ('first', 'second'):
    raise NotLoweredError('cued_catch cue phase {!r}'.format(cue._phase))
  game.sprite_chars = 'Pab'
  game.impassable = [impassable, [0] * 4, [0] * 4]
  game.confined = [True, False, False]
  game.egocentric = [False, False, False]
  recs = [_sprite_record(player, aux0=_int32(player._trials_till_reward, 'reward_free_trials'))]
  for ch in 'ab':
    ball = th[ch]
    start = ball._start_position
    recs.append([int(ball.position[0]), int(ball.position[1]), int(start[0]), int(start[1]),
                 1 if ball.visible else 0, 0, 0, 0])
  game.sprites = np.array(recs, dtype=np.int32)
  game.drape_chars = 'Q'
  game.margins = [(-1, -1)]
  pairs = sum(1 << k for k, ball in enumerate(cue._cues_to_balls) if ball == 'top')
  rec = _drape_record(aux0=_int32(cue._num_trials_left, 'num_trials'), aux1=pairs)
  rec[_lib.D_CORNER_R] = 0 if cue._phase == 'first' else 1
  rec[_lib.D_CORNER_C] = _int32(cue._first_phase_tick, 'first-phase tick')
  rec[_lib.D_PRE_R] = _int32(cue._second_phase_cue_choice, 'cue choice')
  rec[_lib.D_PRE_C] = _int32(cue._second_phase_tick, 'second-phase tick')
  rec[_lib.D_LAST_FRAME] = _frame_word(cue._second_phase_last_reset)
  game.drapes = np.array([rec], dtype=np.int32)
  game.bits = {0: pack_rows(cue.curtain, game.bits_words)}
  which = plot.get('which_ball')
  if which not in _WHICH:
    raise NotLoweredError('cued_catch which_ball {!r}'.format(which))
  game.plot = np.array(_plot_record(
      aux0=1 if plot.get('programming_complete') else 0, aux1=_WHICH[which],
      aux2=_frame_word(plot.get('last_ball_reset'))), dtype=np.int32)
  noisy = sigma != 0.0 or sigma != sigma
  s_lo, s_hi = _f64_words(sigma)
  m_lo, m_hi = _f64_words(random.NV_MAGICCONST)
  game.program_arg[:8] = [1 if noisy else 0, icd, _int32(cue._cue_duration, 'cue_duration'),
                          1 if cue._always_show_ball_symbol else 0, s_lo, s_hi, m_lo, m_hi]
  game.rng_streams = ('python',)
  game.rng_from_globals = True
  game.template_draws = (3, 2)
  game.float_reward = noisy
  if noisy:
    game.python_reward = python_reward
  game.sync = sync
  return game


def python_reward(engine, value):
  """A step's reward as upstream types it: float(caught) + normalvariate(...) is a float, the
  `add_reward(0)` of the other frames an int (cued_catch.py:149-156)."""
  return float(value) if int(engine.batched.plot[0, _lib.P_AUX3]) else int(value)


def sync(engine):
  """CueDrape's privates, the player's reward-free trials left and the Plot's
  programming_complete / which_ball / last_ball_reset, from env 0."""
  p, b = engine.the_plot, engine.batched
  words = b.plot[0].cpu().numpy()
  q = b.drapes[0, 0].cpu().numpy()
  cue, player = engine.things['Q'], engine.things['P']
  cue._phase = 'first' if q[_lib.D_CORNER_R] == 0 else 'second'
  cue._first_phase_tick = int(q[_lib.D_CORNER_C])
  cue._second_phase_cue_choice = int(q[_lib.D_PRE_R])
  cue._second_phase_tick = int(q[_lib.D_PRE_C])
  last = int(q[_lib.D_LAST_FRAME])
  cue._second_phase_last_reset = -float('inf') if last == _lib.NEVER else last
  cue._num_trials_left = int(q[_lib.D_AUX0])
  cue._cues_to_balls = ['top' if (int(q[_lib.D_AUX1]) >> k) & 1 else 'bottom' for k in range(4)]
  player._trials_till_reward = int(b.sprites[0, 0, _lib.S_AUX0])
  if int(words[_lib.P_AUX0]):
    p['programming_complete'] = True
  which = int(words[_lib.P_AUX1])
  if which:
    p['which_ball'] = 'top' if which == 1 else 'bottom'
  if int(words[_lib.P_AUX2]) != _lib.NEVER:
    p['last_ball_reset'] = int(words[_lib.P_AUX2])
