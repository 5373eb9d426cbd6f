"""examples/research/lp-rnn/t_maze.py on `csrc/t_maze.cu`."""

import numpy as np

from pycolab_b200 import _lib
from pycolab_b200.errors import NotLoweredError
from pycolab_b200.lowering import (LoweredGame, _common, _drape_record, _plot_record,
                                   _scrolly_record, _set_sprites, _sprite_record, pack_rows,
                                   round_up)


def lower(engine, roles):
  """examples/research/lp-rnn/t_maze.py:180-505: 'P', the cue 'Q' and five
  PseudoTeleportingScrollys (drapes 'Q#*ltr' on the device).  What the constructors drew —
  the cue side, the speckle — is in the templates; with an RNG bound a batched engine redraws
  both at every restart from the UN-speckled '*' pattern (`pattern_redraw`) and the full cue
  (`bits[0]`, halved on the device)."""
  th, plot = engine.things, engine.the_plot
  want = {'P': 't_maze.player', 'Q': 't_maze.cue', '#': 't_maze.maze', '*': 't_maze.speckle',
          't': 't_maze.teleporter', 'l': 't_maze.goal', 'r': 't_maze.goal'}
  if roles != want:
    raise NotLoweredError('t_maze program needs exactly {} (got {})'.format(want, roles))
  game = LoweredGame()
  _common(engine, game, _lib.PROG_T_MAZE)
  if game.groups != ['Q#*', 'P', 'ltr'] or game.z_order != '*#ltrQP':
    raise NotLoweredError("t_maze program needs update groups [Q # *] [P] [l t r] and z-order "
                          "'*#ltrQP'")
  if engine.rows > 32 or engine.cols > 16:
    raise NotLoweredError('t_maze program: boards up to 32 x 16')
  if th['l']._name != 'left' or th['r']._name != 'right':
    raise NotLoweredError("t_maze program needs the 'left' goal on 'l' and the 'right' on 'r'")
  player = th['P']
  _set_sprites(game, [player], [_sprite_record(player, aux0=0, aux1=_lib.NEVER)])
  scrollys = '#*ltr'
  shape = th['#'].whole_pattern.shape
  for ch in scrollys:
    d = th[ch]
    if d._scrolling_group != '' or d._scroll_margins is not None:
      raise NotLoweredError('t_maze Scrollys have margins None in the default scrolling group')
    if d.whole_pattern.shape != shape or tuple(d._board_shape) != (engine.rows, engine.cols):
      raise NotLoweredError('t_maze Scrolly patterns of different shapes')
  tele = th['t']
  level = (tele._dy - 9) // 11
  if (11 * level + 9 != tele._dy or (tele._limbo_row, tele._limbo_col, tele._dx) != (4, 140, -46)
      or tele._in_limbo):
    raise NotLoweredError('t_maze teleporter with other limbo constants')
  # TeleporterDrape lands the player in the level's hallway: that cell must exist and be free.
  hall = (tele._limbo_row + tele._dy, tele._limbo_col + tele._dx)
  if not (0 <= hall[0] < shape[0] and 0 <= hall[1] < shape[1]) or th['#'].whole_pattern[hall]:
    raise NotLoweredError('t_maze level {} has no hallway at {}'.format(level, hall))
  game.drape_chars = 'Q' + scrollys
  game.margins = [(-1, -1)] * 6
  game.pattern_rows, game.pattern_cols = shape
  game.pattern_words = round_up((shape[1] + 31) // 32 + 1, 2)
  tele_pattern = tele._saved_whole_pattern if tele._teleport_delay > 0 else tele.whole_pattern
  for d, ch in enumerate(scrollys, 1):
    game.patterns[d] = pack_rows(tele_pattern if ch == 't' else th[ch].whole_pattern,
                                 game.pattern_words)
    game.pattern_mutable[d] = ch == '*'
  game.pattern_redraw[2] = pack_rows(th['*']._pattern_at_init, game.pattern_words)
  cue = th['Q']
  full_cue = engine._drape_prefills['Q']
  if cue.which_goal not in ('left', 'right'):
    raise NotLoweredError('t_maze cue names no goal')
  game.bits = {0: pack_rows(full_cue, game.bits_words)}
  recs = [_drape_record(aux0=0 if cue.which_goal == 'left' else 1,
                        aux1=1 if plot.get('yo_we_have_teleported') else 0)]
  for ch in scrollys:
    recs.append(_scrolly_record(th[ch]))
  recs[4][_lib.D_AUX1] = int(tele._teleport_delay)
  recs[4][_lib.D_AUX2] = int(tele._limbo_countdown)
  game.drapes = np.array(recs, dtype=np.int32)
  timeout = plot['timeout_frames']
  order = plot.get('teleportation_order', (0, 0))
  game.plot = np.array(_plot_record(
      aux0=_lib.T_MAZE_NO_TIMEOUT if timeout == float('inf') else int(timeout),
      aux1=plot.get('teleportation_order_frame', -1), aux2=order[0], aux3=order[1]),
      dtype=np.int32)
  game.program_arg[:5] = [level, 1 if cue._cue_after_teleport else 0,
                          _lib.T_MAZE_NO_TIMEOUT if timeout == float('inf') else int(timeout),
                          int(tele._teleport_delay), int(tele._limbo_countdown)]
  # t_maze.py:262 and :365: slot 0 continues random.Random (the cue side), slot 1 NumPy's
  # RandomState (the speckle field)
  game.rng_streams = ('python', 'numpy')
  game.reward_type = float
  game.float_reward = True
  game.curtain = curtain
  game.layers = layers
  game.sync = sync
  return game


def _rolled(eng, d, rows, cols):
  """u8 [B, R, C]: each env's pattern of Scrolly `d` after its np.roll, read at pattern rows
  `rows` [B, R] and columns `cols` [B, C] of the rolled pattern.  The record's AUX0 holds the
  cumulative roll (rows << 16 | cols); the teleporter is empty while its delay (AUX1) lasts
  (t_maze.py:397-428)."""
  import torch
  rec = eng.drapes[:, d].long()
  roll = rec[:, _lib.D_AUX0]
  bits = eng.packed_bits(eng.patterns[d], (rows + (roll >> 16)[:, None]) % eng.game.pattern_rows,
                         (cols + (roll & 0xffff)[:, None]) % eng.game.pattern_cols)
  if eng.drape_chars[d] == 't':
    bits = bits * (rec[:, _lib.D_AUX1] <= 0).to(torch.uint8)[:, None, None]
  return bits


def curtain(eng, d):
  """The Scrollys' curtains: the board window at the drape's corner onto the rolled pattern.
  The cue (drape 0) is a plain curtain the device exports."""
  import torch
  if d == 0:
    return None
  rec = eng.drapes[:, d].long()
  rows = torch.arange(eng.rows, device=eng.device)[None, :] + rec[:, _lib.D_CORNER_R, None]
  cols = torch.arange(eng.cols, device=eng.device)[None, :] + rec[:, _lib.D_CORNER_C, None]
  out = torch.zeros((eng.batch, eng.rows, eng.pitch), dtype=torch.uint8, device=eng.device)
  out[:, :, :eng.cols] = _rolled(eng, d, rows, cols)
  return out


def layers(eng, chars):
  """Rolled Scrolly patterns: each layer is the backdrop's cells plus its owner's curtain."""
  import torch
  backdrop = eng.backdrop[eng.level_rows(eng.backdrop), :, :eng.cols]
  planes = []
  for ch in chars:
    plane = backdrop.eq(ord(ch))
    if ch in eng.drape_chars:
      plane |= eng.curtain(ch)
    elif ch in eng.sprite_chars:
      rec = eng.sprites[:, eng.sprite_chars.index(ch)].long()
      b = torch.nonzero(rec[:, _lib.S_FLAGS] & 1, as_tuple=True)[0]
      plane[b, rec[b, _lib.S_ROW], rec[b, _lib.S_COL]] = True
    planes.append(plane)
  return torch.stack(planes, dim=1)


def sync(engine):
  """The Plot's timeout and teleportation entries, the cue's `which_goal` and every Scrolly's
  rolled `whole_pattern`, from env 0."""
  import torch
  p, b = engine.the_plot, engine.batched
  words = b.plot[0].cpu().numpy()
  p['timeout_frames'] = (float('inf') if int(words[_lib.P_AUX0]) == _lib.T_MAZE_NO_TIMEOUT
                         else int(words[_lib.P_AUX0]))
  if int(words[_lib.P_AUX1]) >= 0:
    p['teleportation_order_frame'] = int(words[_lib.P_AUX1])
    p['teleportation_order'] = (int(words[_lib.P_AUX2]), int(words[_lib.P_AUX3]))
  q = b.drapes[0, 0].cpu().numpy()
  if q[_lib.D_AUX1]:
    p['yo_we_have_teleported'] = True
  elif 'yo_we_have_teleported' in p:
    del p['yo_we_have_teleported']
  engine.things['Q'].which_goal = 'left' if q[_lib.D_AUX0] == 0 else 'right'
  rows = torch.arange(b.game.pattern_rows, device=b.device).expand(b.batch, -1)
  cols = torch.arange(b.game.pattern_cols, device=b.device).expand(b.batch, -1)
  for d in range(1, len(b.drape_chars)):
    np.copyto(engine.things[b.drape_chars[d]].whole_pattern,
              _rolled(b, d, rows, cols)[0].cpu().numpy().astype(bool))
