"""oracle/sampled_check.lockstep on the CPU, driven by a stand-in for BatchedEngine.

The stand-in replays, per env, the frames `trajectory.run_trajectory` records for the same
actions from the same oracle worlds, as CPU torch tensors laid out as the device's.  So
lockstep passing on it shows that lockstep rebuilds worlds in run_trajectory's auto-reset
sequence, and corrupting one field of one frame shows that lockstep compares that field.
"""

import numpy as np
import pytest
import torch

import trajectory as tj
from oracle import engine_model as em
from oracle import games as ogames
from oracle import sampled_check as sc
from pycolab_b200 import levels

ART = levels.scrolly_maze_level(7, world_shape=(33, 41), board_shape=(12, 20))
B, T, PITCH = 5, 60, 32
SPRITES, DRAPES = 'Pabc', '#@'
CROP = (7, 9, ['P'], ' ', (None, None))        # rows, cols, to_track, pad_char, margins


def make_world(e):
  return ogames.make_scrolly_maze(ART[0], ART[1], '+', ART[2])


def make_cropper():
  rows, cols, track, pad, margins = CROP
  return em.ScrollingCrop(rows, cols, track, pad_char=pad, scroll_margins=margins)


def _actions():
  rs = np.random.RandomState(2)
  actions = rs.choice(6, size=(T, B), p=[.22, .22, .22, .22, .04, .08])
  return actions.astype(np.int32)


class StandIn(object):
  """The attributes and methods of BatchedEngine that lockstep reads, on the CPU."""
  device = 'cpu'
  sprite_chars = SPRITES

  def __init__(self, actions, float_reward=False):
    self.actions = actions
    frames = [self._record(e, actions[:, e]) for e in range(B)]
    self.cols = len(ART[1][0])
    self.frames = {k: torch.from_numpy(np.stack([f[k] for f in frames], axis=1))
                   for k in frames[0]}
    if float_reward:
      self.frames['reward'] = self.frames['reward'].double()
    self.t = 0

  @staticmethod
  def _record(e, actions):
    cropper = make_cropper()
    rec = {k: [] for k in ('board', 'reward', 'has_reward', 'discount', 'done', 'sprites',
                           'curtains', 'crop')}

    def on_frame(world, out):
      board = np.zeros((world.rows, PITCH), np.uint8)
      board[:, :world.cols] = out[0]
      rec['board'].append(board)
      rec['reward'].append(0 if out[1] is None else out[1])
      rec['has_reward'].append(out[1] is not None)
      rec['discount'].append(out[2])
      rec['done'].append(world.game_over)
      rec['sprites'].append([list(sc.sprite_words(world.things[ch])) + [0, 0, 0]
                             for ch in SPRITES])
      rec['curtains'].append([world.things[ch].curtain.copy() for ch in DRAPES])
      cropper.set_engine(world)
      rec['crop'].append(cropper.crop(out[0]).copy())
    tj.run_trajectory(lambda: make_world(e), actions.tolist(), on_frame=on_frame)
    dtypes = dict(board=np.uint8, reward=np.int32, has_reward=np.uint8, discount=np.float32,
                  done=np.uint8, sprites=np.int32, curtains=bool, crop=np.uint8)
    return {k: np.array(v, dtype=dtypes[k]) for k, v in rec.items()}

  def play(self, actions):
    assert actions.tolist() == self.actions[self.t].tolist()
    self.t += 1

  def __getattr__(self, name):
    key = {'_board': 'board', 'reward': 'reward', 'has_reward': 'has_reward',
           'discount': 'discount', 'done': 'done', 'sprites': 'sprites'}.get(name)
    if key is None:
      raise AttributeError(name)
    return self.frames[key][self.t]

  @property
  def board(self):
    return self._board[:, :, :self.cols]

  def curtain(self, ch):
    return self.frames['curtains'][self.t][:, DRAPES.index(ch)]

  def crop(self, spec, state=None):
    assert spec == CROP and state == 'state'
    return self.frames['crop'][self.t]


def _lockstep(eng, actions, **kw):
  return sc.lockstep(eng, make_world, range(B), actions, crop=(CROP, 'state', make_cropper),
                     curtains=DRAPES, sprites=SPRITES, pad_columns=True, **kw)


@pytest.mark.parametrize('float_reward', [False, True])
def test_unchanged_stand_in_passes(float_reward):
  actions = _actions()
  eng = StandIn(actions, float_reward)
  assert int(eng.frames['done'].sum()) > B               # auto-resets happen on the way
  seen = []
  n = _lockstep(eng, actions, on_step=lambda t, e, worlds, outs: seen.append(t))
  assert n == B * (T + 1) and seen == list(range(T + 1))


def test_auto_reset_sequence_equals_run_trajectory():
  """The worlds lockstep holds after each step are those run_trajectory steps to."""
  actions = _actions()
  boards = []
  sc.lockstep(StandIn(actions), make_world, range(B), actions,
              on_step=lambda t, e, worlds, outs: boards.append([outs[k][0] for k in range(B)]))
  for e in range(B):
    want = tj.run_trajectory(lambda: make_world(e), actions[:, e].tolist())
    np.testing.assert_array_equal(np.array(boards)[:, e], want['boards'])


def _flip(x, bit=1):
  """x with one value changed: another bit pattern of the same dtype."""
  if x.dtype == torch.float64:
    return torch.nextafter(x, x + 1)          # the same value to int()
  if x.dtype == torch.float32:
    return x + 0.5
  return ~x if x.dtype == torch.bool else x ^ bit


CORRUPTIONS = {                     # frame field, index within one env, field lockstep names
    'board': ('board', (3, 4), 'board'),
    'reward': ('reward', (), 'reward'),
    'reward_float64': ('reward', (), 'reward'),
    'has_reward': ('has_reward', (), 'reward'),
    'discount': ('discount', (), 'discount'),
    'done': ('done', (), 'game_over'),
    'crop': ('crop', (3, 4), 'crop'),
    'curtain': ('curtains', (1, 2, 2), 'curtain @'),
    'sprite_row': ('sprites', (0, 0), 'sprite P'),
    'sprite_col': ('sprites', (1, 1), 'sprite a'),
    'sprite_vrow': ('sprites', (2, 2), 'sprite b'),
    'sprite_vcol': ('sprites', (3, 3), 'sprite c'),
    'sprite_visible': ('sprites', (0, 4), 'sprite P'),
    'sprite_prior_visible': ('sprites', (1, 4), 'sprite a'),
    'pad_columns': ('board', (0, PITCH - 1), 'pad columns'),
}


@pytest.mark.parametrize('what', sorted(CORRUPTIONS))
def test_one_corrupted_field_is_named(what):
  actions = _actions()
  eng = StandIn(actions, float_reward=what == 'reward_float64')
  key, at, name = CORRUPTIONS[what]
  t, e = 17, 3
  frame = eng.frames[key][t, e]
  frame[at] = _flip(frame[at], bit=2 if what == 'sprite_prior_visible' else 1)
  with pytest.raises(sc.Mismatch) as err:
    _lockstep(eng, actions)
  msg = str(err.value)
  assert msg.startswith(name + ' differ') and 'at step %d env %d' % (t, e) in msg, msg
