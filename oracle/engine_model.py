"""CPU restatement of pycolab's per-step hot path.  TEST INFRASTRUCTURE ONLY.

This module is the *oracle* for the H100 step engine: a plain Python/NumPy
restatement of what `Engine.play()` does in the reference, written as explicit
register structs + free functions (the same shape the CUDA kernels have) instead
of the reference's class hierarchy.  Nothing under `pycolab_b200/` may import
it; only `tests/`, `__graft_entry__.smoke()` and `bench.py`'s CPU-baseline legs
do.

Parity status: PINNED.  `tests/golden/*.npz` hold trajectories produced by the
real reference (imported from /root/reference by `tests/golden/make_golden.py`);
`tests/test_oracle_golden.py` replays them through this module bit-exactly, and
`tests/test_oracle_vs_reference.py` runs live differential checks whenever
/root/reference is present.

Reference sections restated here (file:line in /root/reference/pycolab):
  engine.py:583-639    Engine.play                       -> `World.play`
  engine.py:698-735    Engine._update_and_render         -> `World.play`
  engine.py:737-759    Engine._render                    -> `render`
  engine.py:761-847    Engine._apply_and_clear_plot      -> `World._apply_plot`
  rendering.py:98-179  BaseObservationRenderer           -> `render`
  plot.py:69-104,136-260  Plot engine directives         -> `PlotRegs`
  prefab_parts/sprites.py:223-550  MazeWalker            -> `Walker` + walker_*
  prefab_parts/drapes.py:293-695   Scrolly               -> `Scrolly` + scrolly_*
  protocols/scrolling.py:287-569   scrolling protocol    -> `ScrollRegs` + fns
  cropping.py:118-227,393-598      ScrollingCropper      -> `ScrollingCrop`
"""

import numpy as np

# Motion codes shared with the CUDA side (include/pcl.h: PCL_MOTION_*).
# (drow, dcol); index 8 = stay.  sprites.py:140-150, drapes.py (same constants).
MOTIONS = ((-1, 0), (-1, 1), (0, 1), (1, 1), (1, 0), (1, -1), (0, -1), (-1, -1),
           (0, 0))
M_N, M_NE, M_E, M_SE, M_S, M_SW, M_W, M_NW, M_STAY = range(9)
MOTION_OF_NAME = {'n': M_N, 'ne': M_NE, 'e': M_E, 'se': M_SE, 's': M_S,
                  'sw': M_SW, 'w': M_W, 'nw': M_NW, 'stay': M_STAY}
NO_MOTION = -1          # "no motion helper was called this frame"

EDGE = -1               # obstruction code for the board edge (sprites.py:137)


# --------------------------------------------------------------------------
# Plot registers (plot.py:69-104) and scrolling-protocol registers
# (protocols/scrolling.py:198-241).
# --------------------------------------------------------------------------

class ScrollRegs(object):
  """Blackboard of one scrolling group (scrolling.py:198-241)."""

  def __init__(self):
    self.order = None          # (drow, dcol) or None
    self.order_frame = None    # frame the order was issued at
    self.ego = []              # chars of egocentric entities (a set upstream)
    self.permit_frame = {}     # char -> frame the permit is valid AT
    self.permits = {}          # char -> set of motion tuples


class PlotRegs(object):
  """Per-env Plot state the engine consults (plot.py:69-104, 274-341)."""

  def __init__(self):
    self.frame = -1            # plot.py:110
    self.update_group = None
    self.scroll = {}           # scrolling group name -> ScrollRegs
    self.store = {}            # game-specific messages (the dict part of Plot)
    self.clear_directives()

  def clear_directives(self):  # plot.py:343
    self.z_updates = []
    self.reward = None         # None until somebody calls add_reward
    self.game_over = False
    self.discount = 1.0

  def add_reward(self, r):     # plot.py:201-214
    self.reward = r if self.reward is None else self.reward + r

  def terminate_episode(self, discount=0.0):   # plot.py:176-199
    self.game_over = True
    self.discount = discount

  def change_z_order(self, move_this, in_front_of_that):  # plot.py:136-174
    self.z_updates.append((move_this, in_front_of_that))

  def group(self, name):
    return self.scroll.setdefault(name, ScrollRegs())


def scroll_get_order(plot, group):
  """scrolling.py:339-370: an order counts only in the frame it was issued."""
  regs = plot.group(group)
  if regs.order_frame != plot.frame:
    return None
  return regs.order


def scroll_permit(plot, group, char, motions):
  """scrolling.py:373-434: permits issued now are valid at frame + 1."""
  regs = plot.group(group)
  assert char in regs.ego, 'permit() by a non-egocentric entity'
  valid_at = plot.frame + 1
  mine = regs.permits.setdefault(char, set())
  if regs.permit_frame.setdefault(char, valid_at) != valid_at:
    regs.permit_frame[char] = valid_at
    mine.clear()
  mine.update(motions)


def scroll_is_possible(plot, group, motion):
  """scrolling.py:437-482."""
  regs = plot.group(group)
  for char in regs.ego:
    if regs.permit_frame.get(char) != plot.frame:
      return False
    if tuple(motion) not in regs.permits.get(char, ()):
      return False
  return True


def scroll_order(plot, group, motion):
  """scrolling.py:485-531 with check_possible=False (the only mode the
  prefabs use, drapes.py:621,656)."""
  regs = plot.group(group)
  if regs.order_frame == plot.frame:
    raise RuntimeError('second scrolling order in one frame')
  regs.order_frame = plot.frame
  regs.order = tuple(motion)


# --------------------------------------------------------------------------
# MazeWalker (prefab_parts/sprites.py).
# --------------------------------------------------------------------------

class Walker(object):
  """Registers of one MazeWalker sprite (sprites.py:153-205; things.py:339-391)."""
  is_sprite = True

  def __init__(self, char, board_shape, position, impassable='',
               confined=False, egocentric=False, group=''):
    self.char = char
    self.rows, self.cols = board_shape       # Sprite.corner
    self.row, self.col = position            # true position
    self.vrow, self.vcol = position          # virtual position
    self.visible = True                      # things.py:355
    self.prior_visible = None                # sprites.py:205
    self.impassable = frozenset(ord(c) for c in impassable)
    self.confined = confined
    self.egocentric = egocentric
    self.group = group
    self.aux = {}                            # game-specific registers
    self.last_result = None                  # last motion-helper return value

  @property
  def position(self):
    return (self.row, self.col)

  @property
  def virtual_position(self):
    return (self.vrow, self.vcol)


def _on_board(w, r, c):                      # sprites.py:548-550
  return 0 <= r < w.rows and 0 <= c < w.cols


def walker_teleport(w, vr, vc):
  """sprites.py:315-352 (+ exit/enter hooks :223-275)."""
  was_on = _on_board(w, w.vrow, w.vcol)
  now_on = _on_board(w, vr, vc)
  if was_on and not now_on:                  # _on_board_exit
    w.prior_visible = w.visible
    w.visible = False
  w.vrow, w.vcol = vr, vc
  if now_on:
    w.row, w.col = vr, vc
  else:
    w.row, w.col = 0, 0
  if (not was_on) and now_on:                # _on_board_enter
    w.visible = w.prior_visible


def walker_check(w, board, motion):
  """sprites.py:479-546.  Returns None when `motion` is legal, else the
  obstruction: an int cell code (cardinal) or a 3-tuple of codes (diagonal)."""
  dr, dc = MOTIONS[motion]
  if dr == 0 and dc == 0:
    return None

  def at(ddr, ddc):
    r, c = w.vrow + ddr, w.vcol + ddc
    if not _on_board(w, r, c):
      return EDGE
    return int(board[r, c])

  def blocked(code):
    return (w.confined and code == EDGE) or (code in w.impassable)

  if dr != 0 and dc != 0:
    # Diagonal: flank sharing the row first for west-going ... the reference
    # hard-codes the triples (sprites.py:519-534); order matters only for the
    # returned tuple: (a, diagonal, b) going clockwise from the motion's
    # counter-clockwise neighbour.
    if motion == M_NW:
      trio = (at(0, -1), at(-1, -1), at(-1, 0))
    elif motion == M_NE:
      trio = (at(-1, 0), at(-1, 1), at(0, 1))
    elif motion == M_SE:
      trio = (at(0, 1), at(1, 1), at(1, 0))
    else:  # M_SW
      trio = (at(1, 0), at(1, -1), at(0, -1))
    if blocked(trio[1]):
      return trio
    if blocked(trio[0]) and blocked(trio[2]):
      return trio
    return None
  code = at(dr, dc)
  return code if blocked(code) else None


def walker_move(w, board, plot, motion):
  """sprites.py:356-389 `_move`: obey order, check, move, publish permits."""
  # _obey_scrolling_order, sprites.py:413-454
  if w.egocentric:
    regs = plot.group(w.group)
    if w.char not in regs.ego:
      regs.ego.append(w.char)
  order = scroll_get_order(plot, w.group)
  if order is not None:
    walker_teleport(w, w.vrow - order[0], w.vcol - order[1])
    dr, dc = MOTIONS[motion]
    if w.egocentric and order[0] != dr and order[1] != dc:
      raise RuntimeError('scroll order shares no component with motion')
  result = walker_check(w, board, motion)
  if result is None:                         # _raw_move, sprites.py:391-411
    dr, dc = MOTIONS[motion]
    walker_teleport(w, w.vrow + dr, w.vcol + dc)
  # _update_scroll_permissions, sprites.py:456-477
  if w.egocentric:
    legal = [MOTIONS[M_STAY]]
    for m in (M_N, M_NE, M_E, M_SE, M_S, M_SW, M_W, M_NW):
      if walker_check(w, board, m) is None:
        legal.append(MOTIONS[m])
    scroll_permit(plot, w.group, w.char, legal)
  w.last_result = result
  return result


# --------------------------------------------------------------------------
# Scrolly (prefab_parts/drapes.py).
# --------------------------------------------------------------------------

class PlainDrape(object):
  """A Drape that is just a bool curtain (things.py:146-217)."""
  is_sprite = False

  def __init__(self, char, curtain):
    self.char = char
    self.curtain = np.array(curtain, dtype=bool)
    self.aux = {}


class Scrolly(PlainDrape):
  """Registers of one Scrolly drape (drapes.py:293-376)."""

  def __init__(self, char, board_shape, whole_pattern, corner,
               margins=(2, 3), group=''):
    PlainDrape.__init__(self, char, np.zeros(board_shape, dtype=bool))
    self.board_shape = tuple(board_shape)
    self.pattern = np.array(whole_pattern, dtype=bool)
    self.corner = (int(corner[0]), int(corner[1]))
    self.group = group
    self.limit = (self.pattern.shape[0] - board_shape[0],
                  self.pattern.shape[1] - board_shape[1])
    assert min(self.limit) >= 0
    self.margins = None if margins is None else tuple(margins)
    if self.margins is not None:             # drapes.py:352-364
      self.m_north = margins[0] - 1
      self.m_south = board_shape[0] - margins[0]
      self.m_west = margins[1] - 1
      self.m_east = board_shape[1] - margins[1]
      assert self.m_west < self.m_east and self.m_north < self.m_south
    scrolly_refresh(self)
    self.last_move_frame = None              # -inf upstream (drapes.py:371)
    self.prescroll = self.corner


def scrolly_refresh(d):                      # drapes.py:689-695
  r, c = d.corner
  d.curtain[...] = d.pattern[r:r + d.board_shape[0], c:c + d.board_shape[1]]


def _stale(d, plot):
  return d.last_move_frame is None or d.last_move_frame < plot.frame


def scrolly_prescroll(d, vpos, plot):        # drapes.py:378-411
  if _stale(d, plot):
    d.prescroll = d.corner
  return (vpos[0] + d.prescroll[0], vpos[1] + d.prescroll[1])


def scrolly_postscroll(d, vpos, plot):       # drapes.py:413-441
  if _stale(d, plot):
    raise RuntimeError('postscroll queried before the Scrolly moved')
  return (vpos[0] + d.corner[0], vpos[1] + d.corner[1])


def scrolly_move(d, world, motion):
  """drapes.py:487-659 `_maybe_move`."""
  plot = world.plot
  if _stale(d, plot):
    d.last_move_frame = plot.frame
    d.prescroll = d.corner
  dr, dc = MOTIONS[motion]

  order = scroll_get_order(plot, d.group)
  if order:                                  # somebody already ordered a scroll
    if dr != order[0] and dc != order[1]:
      raise RuntimeError('fresh scroll order shares no component with motion')
    d.corner = (d.corner[0] + order[0], d.corner[1] + order[1])
    scrolly_refresh(d)
    return

  if dr == 0 and dc == 0:
    scrolly_refresh(d)
    return

  if d.margins is None:                      # drapes.py:598-623
    if scroll_is_possible(plot, d.group, (dr, dc)):
      ok_v = 0 <= d.corner[0] + dr <= d.limit[0]
      ok_h = 0 <= d.corner[1] + dc <= d.limit[1]
      issued = (dr if ok_v else 0, dc if ok_h else 0)
      d.corner = (d.corner[0] + issued[0], d.corner[1] + issued[1])
      scroll_order(plot, d.group, issued)
    scrolly_refresh(d)
    return

  # Margin mode, drapes.py:625-659.  "Vertical" means the row component.
  want_v = want_h = False
  for ch in plot.group(d.group).ego:
    ent = world.things[ch]
    if not ent.is_sprite:
      continue
    nr, nc = ent.row + dr, ent.col + dc      # TRUE position (drapes.py:676)
    want_v |= ((ent.row > nr and nr <= d.m_north) or
               (ent.row < nr and nr >= d.m_south))
    want_h |= ((ent.col > nc and nc <= d.m_west) or
               (ent.col < nc and nc >= d.m_east))
  if not (want_v or want_h):
    scrolly_refresh(d)
    return
  issued = (dr if want_v else 0, dc if want_h else 0)
  cand = (d.corner[0] + issued[0], d.corner[1] + issued[1])
  can = (0 <= cand[0] <= d.limit[0]) and (0 <= cand[1] <= d.limit[1])
  # NB the permit test uses the full requested motion, not `issued`
  # (drapes.py:650-651).
  can = can and scroll_is_possible(plot, d.group, (dr, dc))
  if can:
    d.corner = cand
    scroll_order(plot, d.group, issued)
  scrolly_refresh(d)


# --------------------------------------------------------------------------
# Renderer + Engine.
# --------------------------------------------------------------------------

def render(rows, cols, backdrop, z_order, things):
  """engine.py:737-759 + rendering.py:98-160: backdrop, then every entity in
  z-order; visible sprites paint one cell, drapes paint their mask."""
  board = np.array(backdrop, dtype=np.uint8, copy=True)
  for ch in z_order:
    ent = things[ch]
    if ent.is_sprite:
      if ent.visible:
        board[ent.row, ent.col] = ord(ch)
    else:
      board[ent.curtain] = ord(ch)
  return board


def layers_of(board, chars):
  """rendering.py:177-178: occluded layers are `board == ord(c)`."""
  return {c: board == ord(c) for c in chars}


def unoccluded_layers_of(backdrop, things, chars):
  """rendering.py:187-301 (`BaseUnoccludedObservationRenderer`): every layer is
  painted on its own — backdrop characters where the backdrop has them, a visible
  sprite's cell on top of that, a drape's whole curtain in place of it (paint_drape
  copies the curtain over the layer, :278) — so several layers may be set at one
  position."""
  layers = {c: np.asarray(backdrop) == ord(c) for c in chars}
  for ch, ent in things.items():
    if ent.is_sprite:
      layer = np.zeros_like(layers[ch])
      if ent.visible:
        layer[ent.row, ent.col] = True
      layers[ch] = layers[ch] | layer
    else:
      layers[ch] = np.array(ent.curtain, dtype=bool)
  return layers


class World(object):
  """One environment = one reference `Engine` (engine.py:38-246)."""

  def __init__(self, rows, cols, backdrop, things, z_order, groups, program):
    self.rows, self.cols = rows, cols
    self.backdrop = np.array(backdrop, dtype=np.uint8)
    self.things = dict(things)
    self.z_order = list(z_order)
    self.groups = [list(g) for g in groups]
    self.program = program          # callable(world, char, actions)
    self.backdrop_program = None    # callable(world, actions): Backdrop.update, engine.py:718-721
    self.plot = PlotRegs()
    self.board = None               # last render (engine._board.board)
    self.game_over = False
    self.staged = []                # boards after each group render, last step
    self.chars = sorted(set(self.things) |
                        set(chr(c) for c in np.unique(self.backdrop)))

  def _render(self):
    self.board = render(self.rows, self.cols, self.backdrop, self.z_order,
                        self.things)

  def its_showtime(self):           # engine.py:520-581
    self._render()
    return self.play(None)

  def play(self, actions):          # engine.py:583-639, 698-735
    if self.game_over:
      raise RuntimeError('play() after the episode terminated')
    plot = self.plot
    plot.frame += 1
    plot.update_group = None
    self.staged = []
    if self.backdrop_program is not None:      # before any entity, on the stale board
      self.backdrop_program(self, actions)
    for gi, group in enumerate(self.groups):
      plot.update_group = gi
      for ch in group:
        self.program(self, ch, actions)
      self._render()
      self.staged.append(self.board)
    reward, discount, rerender = self._apply_plot()
    if rerender:
      self._render()
    return self.board, reward, discount

  def _apply_plot(self):            # engine.py:761-847
    plot = self.plot
    rerender = False
    for move_this, in_front_of in plot.z_updates:
      rerender = True
      rest = [c for c in self.z_order if c != move_this]
      if in_front_of is None:
        self.z_order = [move_this] + rest
      else:
        k = rest.index(in_front_of)
        self.z_order = rest[:k + 1] + [move_this] + rest[k + 1:]
    self.game_over = plot.game_over
    reward, discount = plot.reward, plot.discount
    plot.clear_directives()
    return reward, discount, rerender

  @property
  def layers(self):
    return layers_of(self.board, self.chars)


# --------------------------------------------------------------------------
# ScrollingCropper (cropping.py:229-598), board and (optionally) a layer dict.
# --------------------------------------------------------------------------

class ScrollingCrop(object):
  """cropping.py:313-598 restated for a single tracked-entity list.  The engine is any
  object with `rows`, `cols` and `things`: {char: entity with `is_sprite` and either
  `row`, `col`, `visible` (a sprite) or a bool `curtain` (a drape)}."""

  def __init__(self, rows, cols, to_track, pad_char=None,
               scroll_margins=(2, 3), initial_offset=None, saccade=True):
    self.rows, self.cols = rows, cols
    self.to_track = list(to_track)
    self.pad = pad_char
    m0 = rows // 2 if scroll_margins[0] is None else scroll_margins[0]
    m1 = cols // 2 if scroll_margins[1] is None else scroll_margins[1]
    assert 2 * m0 < rows and 2 * m1 < cols
    self.margins = (m0, m1)
    self.offset = initial_offset if initial_offset is not None else (0, 0)
    self.saccade = saccade
    self.corner = None
    self.world = None

  def set_engine(self, world):
    if world is not self.world:
      self.corner = None
    self.world = world

  def _centroid(self):              # cropping.py:544-598
    for ch in self.to_track:
      ent = self.world.things[ch]
      if ent.is_sprite:
        if ent.visible:
          return (ent.row, ent.col)
      elif ent.curtain.any():
        rr, cc = ent.curtain.nonzero()
        return (int(np.median(rr)), int(np.median(cc)))
    return None

  def _rectify(self):               # cropping.py:533-542
    r, c = self.corner
    r = max(0, r) - max(0, r + self.rows - self.world.rows)
    c = max(0, c) - max(0, c + self.cols - self.world.cols)
    self.corner = (r, c)

  def _initialise(self, centroid, offset):   # cropping.py:438-458
    if centroid is None:
      self.corner = (0, 0)
      return
    self.corner = (centroid[0] - offset[0], centroid[1] - offset[1])
    if self.pad is None:
      self._rectify()

  def _can_pan_to(self, centroid):  # cropping.py:460-505
    crow, ccol = centroid
    wrow, wcol = self.corner
    mrow, mcol = self.margins
    can_v = (mrow - 1) <= (crow - wrow) <= (self.rows - mrow)
    can_h = (mcol - 1) <= (ccol - wcol) <= (self.cols - mcol)
    if self.pad is None:
      if not can_v:
        if wrow <= 0:
          can_v = crow <= mrow
        elif wrow >= self.world.rows - self.rows:
          can_v = crow >= wrow + self.rows - mrow
      elif not can_h:
        if wcol <= 0:
          can_h = ccol <= mcol
        elif wcol >= self.world.cols - self.cols:
          can_h = ccol >= wcol + self.cols - mcol
    return can_v and can_h

  def _pan_to(self, centroid):      # cropping.py:507-531
    crow, ccol = centroid
    wrow, wcol = self.corner
    mrow, mcol = self.margins
    drow = min(0, crow - wrow - mrow)
    dcol = min(0, ccol - wcol - mcol)
    if drow == 0:
      drow += max(0, crow - wrow - self.rows + mrow + 1)
    if dcol == 0:
      dcol += max(0, ccol - wcol - self.cols + mcol + 1)
    self.corner = (wrow + drow, wcol + dcol)
    if self.pad is None:
      self._rectify()

  def crop(self, board, layers=None):   # cropping.py:393-426 + 118-227
    """The cropped board; with `layers`, (board, layers) as `crop_window` returns."""
    centroid = self._centroid()
    if self.corner is None:
      self._initialise(centroid, (self.rows // 2 + self.offset[0],
                                  self.cols // 2 + self.offset[1]))
    elif centroid is not None:
      if self._can_pan_to(centroid):
        self._pan_to(centroid)
      elif self.saccade:
        self._initialise(centroid, (self.rows // 2, self.cols // 2))
    return crop_window(board, self.corner, self.rows, self.cols, self.pad, layers)


# --------------------------------------------------------------------------
# Observation post-processors (rendering.py:304-661), board-only restatements.
# --------------------------------------------------------------------------

def observation_to_array(board, value_mapping, dtype=None, permute=None):
  """rendering.py:409-542: any dtype; a value is stored by masked assignment, one
  vector component at a time, as upstream stores it."""
  first = next(iter(value_mapping.values()))
  dtype = dtype if dtype is not None else np.array(first).dtype
  try:
    depth, is_3d = len(first), True
  except TypeError:
    depth, is_3d = 1, False
  out = np.zeros((depth,) + board.shape, dtype=dtype)
  for code in np.unique(board):
    if chr(code) not in value_mapping:
      raise RuntimeError('character %r outside the value mapping' % chr(code))
    mask = board == code
    if is_3d:
      for layer, component in enumerate(value_mapping[chr(code)]):
        out[layer, mask] = component
    else:
      out[:, mask] = value_mapping[chr(code)]
  result = out if is_3d else out[0]
  return result if permute is None else np.transpose(result, permute)


def observation_repaint(board, character_mapping):
  """rendering.py:304-406 (board part): upstream repaints through an
  ObservationToArray of the 128 ASCII codes, so a byte >= 128 raises."""
  if board.size and int(board.max()) > 127:
    raise RuntimeError('byte %d outside the ASCII repaint mapping' % int(board.max()))
  lut = np.arange(256, dtype=np.uint8)
  for src, dst in character_mapping.items():
    lut[ord(src)] = ord(dst)
  return lut[board]


def observation_to_feature_array(board, layers, permute=None, observation_layers=None):
  """rendering.py:545-661.  `observation_layers` is the observation's layer dict,
  copied as upstream copies it (a zero plane where a character is missing); None
  means occluded layers of every character, `board == ord(c)`."""
  if observation_layers is None:
    observation_layers = {c: board == ord(c) for c in layers}
  out = np.zeros((len(layers),) + board.shape, dtype=np.float32)
  for index, character in enumerate(layers):
    if character in observation_layers:
      np.copyto(out[index], observation_layers[character])
  return out if permute is None else np.transpose(out, permute)


def crop_window(board, corner, rows, cols, pad_char, layers=None):
  """cropping.py:118-227 `_do_crop`.  With `layers` ({char: bool [H, W]}) returns
  (board, layers): each layer cut at the same window, its pad cells `pad_char == char`."""
  top, left = corner
  H, W = board.shape
  if pad_char is None:
    assert top >= 0 and left >= 0 and top + rows <= H and left + cols <= W
    out = np.zeros((rows, cols), dtype=np.uint8)
  else:
    out = np.full((rows, cols), ord(pad_char), dtype=np.uint8)
  fr0, fc0 = max(0, top), max(0, left)
  fr1 = max(0, min(H, top + rows))
  fc1 = max(0, min(W, left + cols))
  tr0, tc0 = max(0, -top), max(0, -left)
  tr1 = min(rows, max(0, H - top))
  tc1 = min(cols, max(0, W - left))
  out[tr0:tr1, tc0:tc1] = board[fr0:fr1, fc0:fc1]
  if layers is None:
    return out
  cut = {}
  for char, layer in layers.items():
    cut[char] = np.full((rows, cols), pad_char == char, dtype=bool)
    cut[char][tr0:tr1, tc0:tc1] = layer[fr0:fr1, fc0:fc1]
  return out, cut
