"""Sequence Recall set-up (reference `pycolab/examples/research/lp-rnn/sequence_recall.py:
107-317`): four pads light up in a drawn sequence while the player is held in the middle,
then the player must visit them in the same order.

Set-up only; per-step logic is csrc/sequence_recall.cu.  As upstream, the sequence is drawn
from Python's global `random` in `make_game` (`_make_program`), so seeding it and calling
make_game() builds the same game here and there.  A batched engine with auto-reset redraws
the sequence on the device at every restart from per-env `random.Random(seed)` states.

No art ships with this module: `make_game` takes one (`levels.sequence_recall_art()` builds
them at any accepted size).
"""

import enum
import random

from pycolab_b200 import ascii_art
from pycolab_b200 import levels
from pycolab_b200 import things as plab_things
from pycolab_b200.prefab_parts import sprites as prefab_sprites

# The start box looks like the walls (:90-93).
REPAINT_MAPPING = {'%': '#'}


class _State(enum.Enum):
  """States of the game's state machine (:107-127)."""
  OFF = 0
  ON = 1
  SEEK = 2
  EXIT = 3
  QUIT = 4


def make_game(sequence_length=4, demo_light_on_frames=60, demo_light_off_frames=30,
              pause_frames=30, timeout_frames=-1, art=None):
  """sequence_recall.py:130-157; `art` defaults to `levels.sequence_recall_art()`."""
  program = _make_program(sequence_length, demo_light_on_frames, demo_light_off_frames,
                          pause_frames)
  engine = ascii_art.ascii_art_to_game(
      levels.sequence_recall_art() if art is None else art, what_lies_beneath=' ',
      sprites={'P': PlayerSprite},
      drapes={'M': MaskDrape, '%': WaitForSeekDrape},
      update_schedule=['P', 'M', '%'],
      z_order='MP%')
  engine.the_plot['program'] = program
  engine.the_plot['frames_in_state'] = 0
  engine.the_plot['timeout_frames'] = float('inf') if timeout_frames < 0 else timeout_frames
  return engine


def _make_program(sequence_length, demo_light_on_frames, demo_light_off_frames, pause_frames):
  """The state machine program of one episode (:160-188)."""
  sequence = [random.choice('1234') for _ in range(sequence_length)]
  program = []
  for g in sequence:
    program.extend([
        (_State.OFF, demo_light_off_frames),
        (_State.ON, demo_light_on_frames, g),
    ])
  program.append(
      (_State.OFF, max(1, pause_frames)),
  )
  for g in sequence:
    program.extend([
        (_State.SEEK, g),
        (_State.EXIT,),
    ])
  program[-1] = (_State.QUIT,)
  return program


def _device(self, *unused_args, **unused_kwargs):
  raise NotImplementedError('runs on the device: csrc/sequence_recall.cu')


class MaskDrape(plab_things.Drape):
  """Covers the lights, runs the state machine and pays for pads (:191-262)."""

  def __init__(self, curtain, character):
    super(MaskDrape, self).__init__(curtain, character)
    self._all_off_mask = None
    self._mask_for_light = {g: None for g in '1234'}

  update = _device


class WaitForSeekDrape(plab_things.Drape):
  """The start box, gone when the first SEEK begins (:265-271)."""

  update = _device


class PlayerSprite(prefab_sprites.MazeWalker):
  """Held until the sequence is shown; -0.005 per frame and the timeout (:274-317)."""

  def __init__(self, corner, position, character):
    super(PlayerSprite, self).__init__(
        corner, position, character, impassable='#', confined_to_board=True)

  update = _device
