"""examples/research/lp-rnn/sequence_recall.py on `csrc/sequence_recall.cu`."""

import sys

import numpy as np

from pycolab_b200 import _lib
from pycolab_b200.errors import NotLoweredError
from pycolab_b200.lowering import (LoweredGame, _common, _drape_record, _is_known_implementation,
                                   _plot_record, _set_sprites, _sprite_record, pack_rows)

LIGHTS = '1234'


def _program_shape(program):
  """(sequence, on, off, pause) of a list _make_program built (sequence_recall.py:160-188),
  or None for any other list."""
  try:
    names = [s[0].name for s in program]
  except (AttributeError, IndexError, TypeError):
    return None
  L = names.count('ON')
  if L < 1 or len(program) != 4 * L + 1:
    return None
  seq = [program[2 * k + 1][2] for k in range(L)]
  off, on, pause = program[0][1], program[1][1], program[2 * L][1]
  want = []
  for g in seq:
    want += [('OFF', off), ('ON', on, g)]
  want.append(('OFF', pause))
  for g in seq:
    want += [('SEEK', g), ('EXIT',)]
  want[-1] = ('QUIT',)
  got = [(names[i],) + tuple(s[1:]) for i, s in enumerate(program)]
  if got != want or any(g not in LIGHTS or not isinstance(g, str) for g in seq):
    return None
  for x in (on, off, pause):
    if isinstance(x, bool) or not isinstance(x, (int, np.integer)) or not -2 ** 31 <= x < 2 ** 31:
      return None
  return seq, int(on), int(off), int(pause)


def lower(engine, roles):
  """examples/research/lp-rnn/sequence_recall.py:107-317: 'P', the mask 'M' and the start box
  '%', one update group [P M %].  the_plot['program'] becomes a program counter over the
  fixed shape `_make_program` builds (whose source must be the reference's: the device's
  restart draw restates it) and the sequence, which a batched engine redraws at every
  restart from per-env `random.Random` states (slot 0)."""
  th, plot = engine.things, engine.the_plot
  want = {'P': 'sequence_recall.player', 'M': 'sequence_recall.mask',
          '%': 'sequence_recall.wait'}
  if roles != want:
    raise NotLoweredError('sequence_recall program needs exactly {} (got {})'.format(want, roles))
  module = sys.modules.get(type(th['M']).__module__)
  make_program = getattr(module, '_make_program', None)
  if make_program is None or not _is_known_implementation(
      make_program, ('sequence_recall', '_make_program')):
    raise NotLoweredError('sequence_recall: the module\'s _make_program differs from the one '
                          'the device restates')
  game = LoweredGame()
  _common(engine, game, _lib.PROG_SEQUENCE_RECALL)
  if game.groups != ['PM%'] or game.z_order != 'MP%':
    raise NotLoweredError("sequence_recall program needs update_schedule ['P', 'M', '%'] and "
                          "z-order 'MP%'")
  if engine.rows > 32 or engine.cols > 64:
    raise NotLoweredError('sequence_recall program: boards up to 32 x 64')
  chars = set(np.unique(engine.backdrop.curtain).tolist())
  if not chars <= set(map(ord, ' #' + LIGHTS)):
    raise NotLoweredError("sequence_recall backdrop characters other than ' #1234' (upstream "
                          "raises KeyError when the player stands on one)")
  if th['M'].curtain.any():
    raise NotLoweredError("sequence_recall art with 'M' cells")
  shape = _program_shape(plot.get('program'))
  if shape is None:
    raise NotLoweredError('sequence_recall: the_plot[\'program\'] is not a whole program as '
                          '_make_program builds it')
  seq, on, off, pause = shape
  if not 1 <= len(seq) <= 16:
    raise NotLoweredError('sequence_recall program: sequence_length 1 to 16 (got %d)' % len(seq))
  if pause < 1:
    raise NotLoweredError('sequence_recall pause state of %d frames' % pause)
  timeout = plot['timeout_frames']
  if timeout == float('inf'):
    timeout = _lib.SEQUENCE_RECALL_NO_TIMEOUT
  elif (isinstance(timeout, bool) or not isinstance(timeout, (int, np.integer)) or
        not -2 ** 31 <= timeout < _lib.SEQUENCE_RECALL_NO_TIMEOUT):
    raise NotLoweredError('sequence_recall timeout_frames {!r}'.format(timeout))
  fis = plot['frames_in_state']
  if isinstance(fis, bool) or not isinstance(fis, (int, np.integer)) or not 0 <= fis < 2 ** 31:
    raise NotLoweredError('sequence_recall frames_in_state {!r}'.format(fis))
  _set_sprites(game, [th['P']], [_sprite_record(th['P'])])
  game.drape_chars = 'M%'
  game.margins = [(-1, -1)] * 2
  game.drapes = np.array([_drape_record(aux0=0), _drape_record(aux0=0)], dtype=np.int32)
  game.bits = {0: pack_rows(th['M'].curtain, game.bits_words),
               1: pack_rows(th['%'].curtain, game.bits_words)}
  seq_word = sum(LIGHTS.index(g) << (2 * k) for k, g in enumerate(seq))
  game.plot = np.array(_plot_record(aux0=0, aux1=int(fis), aux2=int(timeout),
                                    aux3=np.int64(seq_word).astype(np.uint32).view(np.int32)),
                       dtype=np.int32)
  game.program_arg[:4] = [len(seq), on, off, pause]
  game.rng_streams = ('python',)
  game.reward_type = float
  game.float_reward = True
  state_enum = type(plot['program'][0][0])
  game.sync = lambda eng: sync(eng, state_enum)
  return game


def remaining_program(state_enum, pc, seq, on, off, pause):
  """the_plot['program'] after `pc` states were popped."""
  full = []
  for g in seq:
    full += [(state_enum.OFF, off), (state_enum.ON, on, g)]
  full.append((state_enum.OFF, pause))
  for g in seq:
    full += [(state_enum.SEEK, g), (state_enum.EXIT,)]
  full[-1] = (state_enum.QUIT,)
  return full[pc:]


def sync(engine, state_enum):
  """the_plot's remaining program, frames_in_state and timeout_frames, from env 0."""
  p, b = engine.the_plot, engine.batched
  words = b.plot[0].cpu().numpy()
  L, on, off, pause = (int(x) for x in b.game.program_arg[:4])
  seq_word = int(np.int32(words[_lib.P_AUX3]).view(np.uint32))
  seq = [LIGHTS[(seq_word >> (2 * k)) & 3] for k in range(L)]
  p['program'][:] = remaining_program(state_enum, int(words[_lib.P_AUX0]), seq, on, off, pause)
  p['frames_in_state'] = int(words[_lib.P_AUX1])
  t = int(words[_lib.P_AUX2])
  p['timeout_frames'] = float('inf') if t == _lib.SEQUENCE_RECALL_NO_TIMEOUT else t
