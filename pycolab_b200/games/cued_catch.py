"""Cued Catch set-up (reference `pycolab/examples/research/lp-rnn/cued_catch.py:96-317`): four
cues are shown with the ball each one names, then in every trial a cue says which of two
approaching balls to catch.

Set-up only; per-step logic is csrc/cued_catch.cu.  As upstream, CueDrape draws the four
cue->ball pairings from Python's global `random` when it is BUILT, and update() keeps drawing
from it (a trial's cue, the reward noise): the single-env Engine hands that generator to the
device and takes it back after every step.  A batched engine with auto-reset draws the
pairings on the device at every restart from per-env `random.Random(seed)` states instead.

No art ships with this module: `make_game` takes one (`levels.cued_catch_art()` builds
them at any accepted size).
"""

import random

from pycolab_b200 import ascii_art
from pycolab_b200 import levels
from pycolab_b200 import things as plab_things
from pycolab_b200.prefab_parts import sprites as prefab_sprites


def make_game(initial_cue_duration, cue_duration, num_trials, always_show_ball_symbol=False,
              reward_sigma=0.0, reward_free_trials=0, art=None):
  """cued_catch.py:96-113; `art` defaults to `levels.cued_catch_art()`."""
  return ascii_art.ascii_art_to_game(
      art=levels.cued_catch_art() if art is None else art,
      what_lies_beneath=' ',
      sprites={'P': ascii_art.Partial(PlayerSprite, reward_sigma=reward_sigma,
                                      reward_free_trials=reward_free_trials),
               'a': BallSprite,
               'b': BallSprite},
      drapes={'Q': ascii_art.Partial(CueDrape, initial_cue_duration, cue_duration, num_trials,
                                     always_show_ball_symbol)},
      update_schedule=['P', 'a', 'b', 'Q'])


def _device(self, *unused_args, **unused_kwargs):
  raise NotImplementedError('runs on the device: csrc/cued_catch.cu')


class PlayerSprite(prefab_sprites.MazeWalker):
  """The catcher: up or down one row, paid for standing on the correct ball (:116-167)."""

  def __init__(self, corner, position, character, reward_sigma=0.0, reward_free_trials=0):
    super(PlayerSprite, self).__init__(
        corner, position, character, impassable='', confined_to_board=True)
    self._reward_sigma = reward_sigma
    self._trials_till_reward = reward_free_trials

  update = _device


class BallSprite(plab_things.Sprite):
  """A ball that approaches the player once the cues were shown (:170-194)."""

  def __init__(self, corner, position, character):
    super(BallSprite, self).__init__(corner, position, character)
    self._start_position = position
    self._visible = False

  update = _device


class CueDrape(plab_things.Drape):
  """Programs the player with the pairings, then shows a cue per trial (:197-317)."""

  _NUM_CUES = 4

  def __init__(self, curtain, character, initial_cue_duration, cue_duration, num_trials,
               always_show_ball_symbol):
    super(CueDrape, self).__init__(curtain, character)
    self._initial_cue_duration = initial_cue_duration
    self._cue_duration = cue_duration
    self._num_trials_left = num_trials
    self._always_show_ball_symbol = always_show_ball_symbol
    self._cues_to_balls = random.sample(
        ['top'] * (self._NUM_CUES // 2) + ['bottom'] * (self._NUM_CUES // 2), self._NUM_CUES)
    self._phase = 'first'
    self._first_phase_tick = self._NUM_CUES * self._initial_cue_duration
    self._second_phase_cue_choice = -1
    self._second_phase_tick = -1
    self._second_phase_last_reset = -float('inf')

  update = _device
