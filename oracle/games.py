"""Oracle restatement of the configured example games.  TEST INFRASTRUCTURE ONLY.

Each game is (a) a builder that turns ASCII art into an `engine_model.World`
the way `ascii_art.ascii_art_to_game` + the example's `make_game` do, and (b) a
"program": `program(world, char, actions)` = the `update()` of the entity that
paints `char`.  Reference (under /root/reference/pycolab/):

  examples/scrolly_maze.py:212-364            -> make_scrolly_maze / scrolly_maze_program
  examples/warehouse_manager.py:139-295       -> make_warehouse / warehouse_program
  examples/extraterrestrial_marauders.py:91-256 -> make_marauders / marauders_program
  tests/test_things.py:153-295 (fixtures)     -> make_fixture_world / fixture_program
  examples/better_scrolly_maze.py:209-324     -> make_better_scrolly / better_scrolly_program
  examples/classics/four_rooms.py:45-85, cliff_walk.py:39-86,
  chain_walk.py:37-73                         -> make_classic / classics_program
  examples/fluvial_natation.py:53-110         -> make_fluvial / fluvial_program
  examples/aperture.py:118-196                -> make_aperture / aperture_program
  ascii_art.py:31-292                         -> split_art
"""

import numpy as np

from oracle import engine_model as em


def art_to_array(art):
  """ascii_art.py:295-328."""
  return np.vstack([np.frombuffer(line.encode('ascii'), dtype=np.uint8)
                    for line in art]).copy()


def split_art(art, entity_chars, what_lies_beneath):
  """ascii_art.py:241-289: masks/positions per entity char + the backdrop that
  remains once every entity char is replaced by what lies beneath it."""
  art = art_to_array(art)
  if isinstance(what_lies_beneath, str):
    beneath = np.full_like(art, ord(what_lies_beneath))
  else:
    beneath = art_to_array(what_lies_beneath)
  masks = {}
  for ch in entity_chars:
    mask = art == ord(ch)
    masks[ch] = mask
    art[mask] = beneath[mask]
  return art, masks


def mask_position(mask):
  """ascii_art.py:262-268: a sprite absent from the art sits at (0, 0)."""
  rr, cc = np.where(mask)
  assert len(rr) <= 1
  return (int(rr[0]), int(cc[0])) if len(rr) else (0, 0)


# ==========================================================================
# scrolly_maze
# ==========================================================================

def make_scrolly_maze(maze_art, board_art, corner_mark='+', beneath='#',
                      margins=((2, 3), (2, 3))):
  """examples/scrolly_maze.py:212-242 with Scrolly.PatternInfo
  (drapes.py:166-291) inlined.  margins: scroll margins of '#' and '@' (the example
  keeps the Scrolly default (2, 3) for both)."""
  world_art = art_to_array(maze_art)
  marks = np.argwhere(world_art == ord(corner_mark))
  assert len(marks) == 1
  corner = (int(marks[0][0]), int(marks[0][1]))
  world_art[corner] = ord(beneath)
  board_shape = (len(board_art), len(board_art[0]))

  def vpos(ch):
    where = np.argwhere(world_art == ord(ch))
    assert len(where) == 1, ch
    return (int(where[0][0]) - corner[0], int(where[0][1]) - corner[1])

  backdrop, _ = split_art(board_art, 'Pabc#@', ' ')
  things = {}
  for ch, m in zip('#@', margins):
    things[ch] = em.Scrolly(ch, board_shape, world_art == ord(ch), corner, margins=m)
  for ch in 'abc':
    w = em.Walker(ch, board_shape, (0, 0), impassable='#')
    em.walker_teleport(w, *vpos(ch))
    w.aux['moving_east'] = bool(ord(ch) % 2)     # scrolly_maze.py:282
    things[ch] = w
  p = em.Walker('P', board_shape, (0, 0), impassable='#', egocentric=True)
  em.walker_teleport(p, *vpos('P'))
  things['P'] = p
  return em.World(board_shape[0], board_shape[1], backdrop, things,
                  z_order='abc@#P',
                  groups=[['#'], ['a', 'b', 'c', 'P'], ['@']],
                  program=scrolly_maze_program)


# Action -> motion for P, '#', '@' (scrolly_maze.py:262-271, 320-329, 352-363).
_SCROLLY_ACTION_MOTION = {0: em.M_N, 1: em.M_S, 2: em.M_W, 3: em.M_E,
                          4: em.M_STAY}


def scrolly_maze_program(world, ch, actions):
  plot = world.plot
  ent = world.things[ch]
  motion = _SCROLLY_ACTION_MOTION.get(actions, em.NO_MOTION) \
      if actions is not None else em.NO_MOTION
  if ch == '#':                                   # MazeDrape :308-329
    if motion != em.NO_MOTION:
      em.scrolly_move(ent, world, motion)
  elif ch == 'P':                                 # PlayerSprite :245-271
    if motion != em.NO_MOTION:
      em.walker_move(ent, world.board, plot, motion)
  elif ch in 'abc':                               # PatrollerSprite :274-305
    if plot.frame % 2:
      em.walker_move(ent, world.board, plot, em.M_STAY)
      return
    walls = world.things['#']
    prow, pcol = em.scrolly_prescroll(walls, ent.virtual_position, plot)
    step = 1 if ent.aux['moving_east'] else -1
    if walls.pattern[prow, pcol + step]:
      ent.aux['moving_east'] = not ent.aux['moving_east']
    em.walker_move(ent, world.board, plot,
                   em.M_E if ent.aux['moving_east'] else em.M_W)
    if ent.virtual_position == world.things['P'].virtual_position:
      plot.terminate_episode()
  elif ch == '@':                                 # CashDrape :332-364
    where = em.scrolly_prescroll(ent, world.things['P'].position, plot)
    if ent.pattern[where]:
      plot.add_reward(100)
      ent.pattern[where] = False
      if not ent.pattern.any():
        plot.terminate_episode()
    if motion != em.NO_MOTION:
      em.scrolly_move(ent, world, motion)
    elif actions == 5:
      plot.terminate_episode()
  else:
    raise KeyError(ch)


# ==========================================================================
# warehouse_manager
# ==========================================================================

_BOXES = '1234567890'          # update order, warehouse_manager.py:168


def make_warehouse(art, what_lies_beneath=' '):
  """examples/warehouse_manager.py:139-178."""
  flat = ''.join(art)
  boxes = [c for c in _BOXES if c in flat]
  entity_chars = boxes + ['X', 'P']
  backdrop, masks = split_art(art, entity_chars, what_lies_beneath)
  shape = backdrop.shape
  things = {}
  for ch in boxes:                               # BoxSprite :203-206
    things[ch] = em.Walker(ch, shape, mask_position(masks[ch]),
                           impassable=set('#.0123456789PX') - set(ch))
  judge = em.PlainDrape('X', masks['X'])         # JudgeDrape :241-243
  judge.aux['last_on_goals'] = 0
  things['X'] = judge
  things['P'] = em.Walker('P', shape, mask_position(masks['P']),
                          impassable='#.0123456789X')
  world = em.World(shape[0], shape[1], backdrop, things,
                   z_order=entity_chars,
                   groups=[boxes, ['X'], ['P']],
                   program=warehouse_program)
  world.aux_boxes = boxes
  return world


def warehouse_program(world, ch, actions):
  plot = world.plot
  ent = world.things[ch]
  board = world.board
  if ch == 'X':                                   # JudgeDrape.update :245-266
    ent.curtain.fill(False)
    for b in (c for c in '0123456789' if c in world.things):
      ent.curtain[world.things[b].position] = True
    num_boxes = int(ent.curtain.sum())
    ent.curtain &= (world.backdrop == ord('_'))
    on_goals = int(ent.curtain.sum())
    plot.add_reward(on_goals - ent.aux['last_on_goals'])
    ent.aux['last_on_goals'] = on_goals
    if actions == 5 or on_goals == num_boxes:
      plot.terminate_episode()
  elif ch == 'P':                                 # PlayerSprite.update :284-295
    motion = {0: em.M_N, 1: em.M_S, 2: em.M_W, 3: em.M_E}.get(actions) \
        if actions is not None else None
    if motion is not None:
      em.walker_move(ent, board, plot, motion)
  else:                                           # BoxSprite.update :208-226
    r, c = ent.position
    is_p = lambda rr, cc: board[rr, cc] == ord('P')   # layers['P'][rr, cc]
    # NumPy index semantics: -1 wraps, >= size raises.  Boxes are unconfined, so
    # one pushed off the board sits at position (0, 0) (and is marked there by the
    # judge), and every box at (0, 0) moves together when P stands next to it.
    if actions == 0:
      if is_p(r + 1, c): em.walker_move(ent, board, plot, em.M_N)
    elif actions == 1:
      if is_p(r - 1, c): em.walker_move(ent, board, plot, em.M_S)
    elif actions == 2:
      if is_p(r, c + 1): em.walker_move(ent, board, plot, em.M_W)
    elif actions == 3:
      if is_p(r, c - 1): em.walker_move(ent, board, plot, em.M_E)


# ==========================================================================
# extraterrestrial_marauders
# ==========================================================================

_UP_BOLTS = 'abcd'             # extraterrestrial_marauders.py:62
_DOWN_BOLTS = 'yz'             # :66
_ALL_BOLTS = _UP_BOLTS + _DOWN_BOLTS


def make_marauders(art, rng):
  """examples/extraterrestrial_marauders.py:91-101.  `rng` is the
  numpy.random.RandomState standing in for the global NumPy RNG (:253)."""
  order = ['P', 'B', 'X'] + list(_ALL_BOLTS)
  backdrop, masks = split_art(art, order, ' ')
  shape = backdrop.shape
  things = {}
  things['P'] = em.Walker('P', shape, mask_position(masks['P']),
                          impassable='', confined=True)      # :173-176
  things['B'] = em.PlainDrape('B', masks['B'])
  marauders = em.PlainDrape('X', masks['X'])
  marauders.aux['dx'] = -1                                   # :140
  things['X'] = marauders
  for ch in _ALL_BOLTS:                                      # :192-196, :226-230
    w = em.Walker(ch, shape, mask_position(masks[ch]), impassable='')
    em.walker_teleport(w, -1, -1)
    things[ch] = w
  world = em.World(shape[0], shape[1], backdrop, things, z_order=order,
                   groups=[order], program=marauders_program)
  world.rng = rng
  return world


def marauders_program(world, ch, actions):
  plot = world.plot
  ent = world.things[ch]
  board = world.board
  layer = lambda c: board == ord(c)
  if ch == 'P':                                   # PlayerSprite.update :178-186
    if actions == 0:
      em.walker_move(ent, board, plot, em.M_W)
    elif actions == 1:
      em.walker_move(ent, board, plot, em.M_E)
    elif actions == 4:
      plot.terminate_episode()
  elif ch == 'B':                                 # BunkerDrape.update :113-120
    bolts = np.zeros(board.shape, dtype=bool)
    for c in _ALL_BOLTS:
      bolts |= layer(c)
    hits = bolts & ent.curtain
    ent.curtain ^= hits
    plot.add_reward(-int(hits.sum()))
    plot.store['bunker_hitters'] = [chr(c) for c in board[hits]]
  elif ch == 'X':                                 # MarauderDrape.update :142-163
    bolts = np.zeros(board.shape, dtype=bool)
    for c in _UP_BOLTS:
      bolts |= layer(c)
    hits = bolts & ent.curtain
    ent.curtain ^= hits
    plot.add_reward(int(hits.sum()) * 10)
    plot.store['marauder_hitters'] = [chr(c) for c in board[hits]]
    if (not ent.curtain.any()) or ent.curtain[10, :].any():
      plot.terminate_episode()
      return
    # Float cadence: frame % max(1, count // 8.0000001)   (:157)
    if plot.frame % max(1, int(ent.curtain.sum()) // 8.0000001):
      return
    if np.any(ent.curtain[:, 0] | ent.curtain[:, -1]):
      ent.aux['dx'] = -ent.aux['dx']
      ent.curtain[:] = np.roll(ent.curtain, shift=1, axis=0)
    ent.curtain[:] = np.roll(ent.curtain, shift=ent.aux['dx'], axis=1)
  elif ch in _UP_BOLTS:                           # UpwardLaserBoltSprite :198-220
    if ent.visible:
      if (ch in plot.store['bunker_hitters'] or
          ch in plot.store['marauder_hitters']):
        em.walker_teleport(ent, -1, -1)
      else:
        em.walker_move(ent, board, plot, em.M_N)
    elif actions == 2:
      if plot.store.get('last_player_shot') == plot.frame:
        return
      plot.store['last_player_shot'] = plot.frame
      row, col = world.things['P'].position
      em.walker_teleport(ent, row - 1, col)
  elif ch in _DOWN_BOLTS:                         # DownwardLaserBoltSprite :232-256
    if ent.visible:
      if ch in plot.store['bunker_hitters']:
        em.walker_teleport(ent, -1, -1)
        return
      if ent.position == world.things['P'].position:
        plot.terminate_episode()
      em.walker_move(ent, board, plot, em.M_S)
    else:
      if plot.store.get('last_marauder_shot') == plot.frame:
        return
      plot.store['last_marauder_shot'] = plot.frame
      seen = layer('X')
      cols = np.nonzero(seen.sum(axis=0))[0]
      col = int(world.rng.choice(cols))
      row = int(np.nonzero(seen[:, col])[0][-1]) + 1
      em.walker_teleport(ent, row, col)
  else:
    raise KeyError(ch)


# ==========================================================================
# better_scrolly_maze (SURVEY.md §8f-1)
# ==========================================================================

def make_better_scrolly(maze_art):
  """examples/better_scrolly_maze.py:209-221."""
  order = ['a', 'b', 'c', 'P', '@']
  backdrop, masks = split_art(maze_art, order, ' ')
  shape = backdrop.shape
  things = {}
  for ch in 'abc':                               # PatrollerSprite :282-286
    w = em.Walker(ch, shape, mask_position(masks[ch]), impassable='#')
    w.aux['moving_east'] = bool(ord(ch) % 2)
    things[ch] = w
  things['P'] = em.Walker('P', shape, mask_position(masks['P']), impassable='#')
  things['@'] = em.PlainDrape('@', masks['@'])
  return em.World(shape[0], shape[1], backdrop, things, z_order='abc@P',
                  groups=[order], program=better_scrolly_program)


def better_scrolly_program(world, ch, actions):
  plot = world.plot
  ent = world.things[ch]
  board = world.board
  if ch == 'P':                                   # PlayerSprite.update :263-276
    motion = {0: em.M_N, 1: em.M_S, 2: em.M_W, 3: em.M_E, 4: em.M_STAY}.get(actions) \
        if actions is not None else None
    if motion is not None:
      em.walker_move(ent, board, plot, motion)
    if actions == 5:
      plot.terminate_episode()
  elif ch in 'abc':                               # PatrollerSprite.update :288-305
    if plot.frame % 2:
      em.walker_move(ent, board, plot, em.M_STAY)
      return
    row, col = ent.position
    if board[row, col - 1] == ord('#'):           # layers['#'][row, col-1]
      ent.aux['moving_east'] = True
    if board[row, col + 1] == ord('#'):
      ent.aux['moving_east'] = False
    em.walker_move(ent, board, plot, em.M_E if ent.aux['moving_east'] else em.M_W)
    if ent.position == world.things['P'].position:
      plot.terminate_episode()
  elif ch == '@':                                 # CashDrape.update :314-324
    where = world.things['P'].position
    if ent.curtain[where]:
      plot.add_reward(100)
      ent.curtain[where] = False
      if not ent.curtain.any():
        plot.terminate_episode()
  else:
    raise KeyError(ch)


# ==========================================================================
# classics: four_rooms, cliff_walk, chain_walk (SURVEY.md §8f-4).  One
# MazeWalker 'P', no drapes, one update group; rewards are Python floats.
# ==========================================================================

CLASSIC_KINDS = ('four_rooms', 'cliff_walk', 'chain_walk')


def make_classic(kind, art):
  """four_rooms.py:45-49, cliff_walk.py:39-43, chain_walk.py:37-41."""
  assert kind in CLASSIC_KINDS
  beneath = ' ' if kind == 'four_rooms' else '.'
  backdrop, masks = split_art(art, ['P'], beneath)
  shape = backdrop.shape
  walker = em.Walker('P', shape, mask_position(masks['P']),
                     impassable='#' if kind == 'four_rooms' else '',      # four_rooms.py:60-63
                     confined=(kind == 'cliff_walk'))                     # cliff_walk.py:54-57
  world = em.World(shape[0], shape[1], backdrop, {'P': walker}, z_order='P',
                   groups=[['P']], program=classics_program)
  world.classic_kind = kind
  return world


def classics_program(world, ch, actions):
  plot, ent, board = world.plot, world.things[ch], world.board
  kind = world.classic_kind
  if kind == 'chain_walk':                        # chain_walk.py:60-73
    motion = {0: em.M_W, 1: em.M_E}.get(actions) if actions is not None else None
  else:                                           # four_rooms.py:68-76, cliff_walk.py:62-71
    motion = {0: em.M_N, 1: em.M_S, 2: em.M_W, 3: em.M_E}.get(actions) \
        if actions is not None else None
  if motion is not None:
    em.walker_move(ent, board, plot, motion)
  if kind == 'four_rooms':                        # :78-80
    if ent.position == (4, 3):
      plot.add_reward(1.0)
      plot.terminate_episode()
  elif kind == 'cliff_walk':                      # :72-86
    if motion is None:
      return
    row, col = ent.position
    if row == ent.rows - 1 and 0 < col < ent.cols - 2:
      plot.add_reward(-100.0)
    else:
      plot.add_reward(-1.0)
    if row == ent.rows - 1 and 0 < col:
      plot.terminate_episode()
  else:                                           # chain_walk.py:66-73
    if ent.col == 0:
      plot.add_reward(1.0)
      plot.terminate_episode()
    elif ent.col == ent.cols - 1:
      plot.add_reward(100.0)
      plot.terminate_episode()


# ==========================================================================
# fluvial_natation (SURVEY.md §8f-4): a Backdrop with update() logic.
# ==========================================================================

def make_fluvial(art):
  """examples/fluvial_natation.py:53-58."""
  backdrop, masks = split_art(art, ['P'], ' ')
  shape = backdrop.shape
  walker = em.Walker('P', shape, mask_position(masks['P']), impassable='')   # :71-74
  world = em.World(shape[0], shape[1], backdrop, {'P': walker}, z_order='P',
                   groups=[['P']], program=fluvial_program)
  world.backdrop_program = fluvial_backdrop_program
  return world


def fluvial_backdrop_program(world, actions):
  """RiverBackdrop.update :106-110: rows 1..3 flow one cell west on even frames."""
  if world.plot.frame % 2 == 0:
    world.backdrop[1:4, :] = np.roll(world.backdrop[1:4, :], shift=-1, axis=1)


def fluvial_program(world, ch, actions):
  """PlayerSprite.update :76-93."""
  plot, ent, board = world.plot, world.things[ch], world.board
  if plot.frame % 2 == 0:
    em.walker_move(ent, board, plot, em.M_W)
  if actions == 0:
    em.walker_move(ent, board, plot, em.M_W)
  elif actions == 1:
    em.walker_move(ent, board, plot, em.M_E)
  if ent.vcol < 0:
    plot.add_reward(-1)
    plot.terminate_episode()
  elif ent.vcol >= board.shape[1]:
    plot.add_reward(1)
    plot.terminate_episode()


# ==========================================================================
# aperture (SURVEY.md §8f-4): a blaster that opens teleporting apertures.
# ==========================================================================

def make_aperture(art):
  """examples/aperture.py:188-196."""
  backdrop, masks = split_art(art, ['A', 'X'], ' ')
  shape = backdrop.shape
  player = em.Walker('A', shape, mask_position(masks['A']), impassable='#.@')    # :126-128
  drape = em.PlainDrape('X', masks['X'])
  drape.aux['apertures'] = [None, None]                                           # :161
  return em.World(shape[0], shape[1], backdrop, {'A': player, 'X': drape}, z_order='XA',
                  groups=[['A'], ['X']], program=aperture_program)


def aperture_program(world, ch, actions):
  plot, board = world.plot, world.board
  player, drape = world.things['A'], world.things['X']
  if ch == 'A':                                   # PlayerSprite.update :130-149
    motion = {0: em.M_N, 1: em.M_S, 2: em.M_W, 3: em.M_E}.get(actions) \
        if actions is not None else None
    if motion is not None:
      em.walker_move(player, board, plot, motion)
    elif actions == 9:
      plot.terminate_episode()
    if board[player.position] == ord('C'):        # layers['C'][self.position]
      plot.add_reward(1)
      plot.terminate_episode()
    if board[player.position] == ord('X'):        # layers['X'][self.position]
      destinations = [p for p in drape.aux['apertures']
                      if p is not None and p != player.position]
      if destinations:
        em.walker_teleport(player, *destinations[0])
  elif ch == 'X':                                 # ApertureDrape.update :163-190
    ply_y, ply_x = player.position
    if actions not in (5, 6, 7, 8):
      return
    dx, dy = {5: (0, -1), 6: (-1, 0), 7: (0, 1), 8: (1, 0)}[actions]
    height, width = board.shape
    for step in range(1, max(height, width)):
      cur_x, cur_y = ply_x + dx * step, ply_y + dy * step
      if cur_x < 0 or cur_x >= width or cur_y < 0 or cur_y >= height:
        break
      elif board[cur_y, cur_x] == ord('#'):
        break
      elif board[cur_y, cur_x] == ord('X'):
        break
      if board[cur_y, cur_x] == ord('@'):
        drape.aux['apertures'] = drape.aux['apertures'][1:] + [(cur_y, cur_x)]
        drape.curtain.fill(False)
        for aperture in drape.aux['apertures']:
          if aperture is not None:
            drape.curtain[aperture] = True
        break
  else:
    raise KeyError(ch)


# ==========================================================================
# Test-fixture world: generic MazeWalkers / Scrollys / static drapes driven by
# per-entity motion codes (tests/test_things.py:203-295).
# ==========================================================================

def make_fixture_world(art, what_lies_beneath, walkers, scrollys=None,
                       drapes='', update_schedule=None, z_order=None):
  """Build a world of fixture entities from ASCII art.

  walkers:  {char: dict(impassable=..., confined=..., egocentric=..., group=...)}
  scrollys: {char: dict(pattern=bool array, corner=(r, c), margins=..., group=...)}
  drapes:   chars of static drapes (TestDrape: curtain never changes).
  """
  scrollys = scrollys or {}
  chars = list(walkers) + list(scrollys) + list(drapes)
  if update_schedule is None:
    update_schedule = [chars]
  flat = [c for g in update_schedule for c in g]
  assert sorted(flat) == sorted(chars)
  backdrop, masks = split_art(art, flat, what_lies_beneath)
  shape = backdrop.shape
  things = {}
  for ch in flat:
    if ch in walkers:
      things[ch] = em.Walker(ch, shape, mask_position(masks[ch]), **walkers[ch])
    elif ch in scrollys:
      kw = dict(scrollys[ch])
      things[ch] = em.Scrolly(ch, shape, kw.pop('pattern'), kw.pop('corner'),
                              **kw)
    else:
      things[ch] = em.PlainDrape(ch, masks[ch])
  return em.World(shape[0], shape[1], backdrop, things,
                  z_order=z_order if z_order is not None else flat,
                  groups=update_schedule, program=fixture_program)


def fixture_program(world, ch, actions):
  """TestMazeWalker.real_update / TestScrolly.real_update: `actions` is None,
  one motion code for everybody, or {char: motion code}; entities with no code
  call `_stay` (test_things.py:219-250, 268-295)."""
  ent = world.things[ch]
  if isinstance(actions, dict):
    motion = actions.get(ch, em.M_STAY)
  elif actions is None:
    motion = em.M_STAY
  else:
    motion = actions
  if isinstance(ent, em.Walker):
    em.walker_move(ent, world.board, world.plot, motion)
  elif isinstance(ent, em.Scrolly):
    em.scrolly_move(ent, world, motion)
  # Plot directives injected with test_things.post_update upstream
  # (test_things.py:85-104): keys '_reward', '_terminate', '_z' = (this, that).
  if isinstance(actions, dict) and ch == world.groups[-1][-1]:
    if actions.get('_reward') is not None:
      world.plot.add_reward(actions['_reward'])
    if actions.get('_terminate'):
      world.plot.terminate_episode()
    if actions.get('_z') is not None:
      world.plot.change_z_order(*actions['_z'])


# ==========================================================================
# ordeal (SURVEY.md §8f-4): three sub-games chained by storytelling.Story; the
# one real user of Plot.change_z_order (examples/ordeal.py:182-185).
# ==========================================================================

ORDEAL_CHAPTERS = ('castle', 'cavern', 'kansas')


def make_ordeal(chapter, art, story_plot=None):
  """One chapter of examples/ordeal.py:74-97.  `story_plot`: what Story hands the
  new Engine's Plot (storytelling.py:449-457): dict(has_sword, last_position,
  prior_chapter); None for the first chapter."""
  assert chapter in ORDEAL_CHAPTERS
  story_plot = dict(story_plot or {})
  beneath = '~' if chapter == 'kansas' else ' '
  chars = {'castle': 'PD', 'cavern': 'PS', 'kansas': 'P'}[chapter]
  backdrop, masks = split_art(art, list(chars), beneath)
  shape = backdrop.shape
  things = {'P': em.Walker('P', shape, mask_position(masks['P']), impassable='@#w',
                           confined=True)}                       # ordeal.py:199-202
  if chapter == 'castle':                                        # :137-140
    things['D'] = em.Walker('D', shape, mask_position(masks['D']), impassable='#',
                            confined=True)
    z_order, groups = ['D', 'P'], [['P', 'D']]                   # :80-82
  elif chapter == 'cavern':                                      # :85-89; default z = sorted
    things['S'] = em.PlainDrape('S', masks['S'])
    z_order, groups = ['P', 'S'], [['P', 'S']]
  else:                                                          # :91-93
    z_order, groups = ['P'], [['P']]
  world = em.World(shape[0], shape[1], backdrop, things, z_order=z_order, groups=groups,
                   program=ordeal_program)
  world.plot.store.update(
      has_sword=bool(story_plot.get('has_sword')),
      last_position=story_plot.get('last_position'),
      this_chapter=chapter, prior_chapter=story_plot.get('prior_chapter'),
      next_chapter=None)                                         # dict stories: storytelling.py:455
  return world


def ordeal_program(world, ch, actions):
  plot, store, ent, board = world.plot, world.plot.store, world.things[ch], world.board
  if ch == 'P':                                                  # PlayerSprite.update :206-266
    limit_r, limit_c = ent.rows - 1, ent.cols - 1                # self._limits :204
    this, prior = store['this_chapter'], store['prior_chapter']

    def leave(to):
      store['next_chapter'] = to
      plot.terminate_episode()
    if actions == 0:
      if this == 'kansas' and ent.row <= 0:
        leave('castle')
      else:
        em.walker_move(ent, board, plot, em.M_N)
    elif actions == 1:
      if this == 'castle' and ent.row >= limit_r:
        leave('kansas')
      else:
        em.walker_move(ent, board, plot, em.M_S)
    elif actions == 2:
      if this == 'cavern' and ent.col <= 0:
        leave('kansas')
      else:
        em.walker_move(ent, board, plot, em.M_W)
    elif actions == 3:
      if this == 'kansas' and ent.col >= limit_c:
        leave('cavern')
      else:
        em.walker_move(ent, board, plot, em.M_E)
    elif actions == 4:
      leave(None)
    elif plot.frame == 0:                                        # line up with the last game
      last = store['last_position']
      if (prior, this) == ('kansas', 'castle'):
        em.walker_teleport(ent, limit_r, last[1])
      elif (prior, this) == ('castle', 'kansas'):
        em.walker_teleport(ent, 0, last[1])
      elif (prior, this) == ('kansas', 'cavern'):
        em.walker_teleport(ent, last[0], 0)
      elif (prior, this) == ('cavern', 'kansas'):
        em.walker_teleport(ent, last[0], limit_c)
    store['last_position'] = ent.position                        # :266
  elif ch == 'D':                                                # DragonduckSprite.update :142-185
    if plot.frame == 0:
      return
    player = world.things['P']
    rel = (ent.row > player.row, ent.col < player.col, ent.row < player.row,
           ent.col > player.col)
    motion = {(True, False, False, False): em.M_N, (True, True, False, False): em.M_NE,
              (False, True, False, False): em.M_E, (False, True, True, False): em.M_SE,
              (False, False, True, False): em.M_S, (False, False, True, True): em.M_SW,
              (False, False, False, True): em.M_W, (True, False, False, True): em.M_NW}.get(rel)
    if motion is not None:
      em.walker_move(ent, board, plot, motion)
    # layers['P'] of the board as last rendered (occluded layers, rendering.py:177)
    if board[ent.row, ent.col] == ord('P'):
      store['next_chapter'] = None
      plot.terminate_episode()
      if store.get('has_sword'):
        plot.add_reward(1.0)
        plot.change_z_order('D', 'P')
      else:
        plot.add_reward(-1.0)
        plot.change_z_order('P', 'D')
  else:                                                          # SwordDrape.update :120-124
    player = world.things['P']
    if ent.curtain[player.row, player.col]:
      store['has_sword'] = True
      plot.add_reward(1.0)
    if store.get('has_sword'):
      ent.curtain[:] = False


# ==========================================================================
# hello_world (SURVEY.md §8f-4): plain Sprites that wrap around the board and a
# Drape that rolls its curtain — no MazeWalker, no board look-ups at all.
# ==========================================================================

class PlainSprite(object):
  """A `things.Sprite` (things.py:339-391): a position and a visibility flag."""
  is_sprite = True

  def __init__(self, char, shape, position):
    self.char = char
    self.rows, self.cols = shape
    self.row, self.col = position
    self.visible = True

  @property
  def position(self):
    return (self.row, self.col)


HELLO_DX = ([-1, 1, -1, 1], [-1, 1, -1, 1], [1, -1, 1, -1], [1, -1, 1, -1])   # hello_world.py:96
HELLO_DY = ([-1, 1, 1, -1], [1, -1, -1, 1], [1, -1, -1, 1], [-1, 1, 1, -1])   # :97


def make_hello(art):
  """examples/hello_world.py:58-68."""
  backdrop, masks = split_art(art, list('1234@'), ' ')
  shape = backdrop.shape
  things = {ch: PlainSprite(ch, shape, mask_position(masks[ch])) for ch in '1234'}
  things['@'] = em.PlainDrape('@', masks['@'])
  return em.World(shape[0], shape[1], backdrop, things, z_order=list('12@34'),
                  groups=[list('1234@')], program=hello_program)


def hello_program(world, ch, actions):
  ent = world.things[ch]
  if ch == '@':                                   # RollingDrape.update :77-87
    if actions is None:
      return
    if actions == 4:
      world.plot.terminate_episode()
    if actions < 4:
      ent.curtain[:] = np.roll(ent.curtain, [-1, 1, -1, 1][actions], [0, 0, 1, 1][actions])
      world.plot.add_reward(1)
  else:                                           # SlidingSprite.update :113-118
    if actions is None or actions > 3:
      return
    k = int(ch) - 1                               # direction_set :62-65
    ent.col = (ent.col + HELLO_DX[k][actions]) % ent.cols
    ent.row = (ent.row + HELLO_DY[k][actions]) % ent.rows


# ==========================================================================
# apprehend (SURVEY.md §8f-4): a ball falling along a random straight line and a
# catcher; the ball's slope is a float64 drawn from Python's `random` when the
# sprite is BUILT (apprehend.py:95-106), so every episode draws once.
# ==========================================================================

def make_apprehend(art, rng):
  """examples/apprehend.py:56-60; `rng` stands for the `random` module
  (`random.Random(seed)` reproduces `random.seed(seed)` + the module functions)."""
  backdrop, masks = split_art(art, ['P', 'b'], ' ')
  shape = backdrop.shape
  player = em.Walker('P', shape, mask_position(masks['P']), impassable='',
                     confined=True)                                   # :71-74
  ball = em.Walker('b', shape, mask_position(masks['b']), impassable='')   # :98-100
  ball.aux['dx'] = rng.uniform(-2.499, 2.499) / (shape[0] - 1.0)       # :103
  ball.aux['acc'] = 0.0                                                # :107
  return em.World(shape[0], shape[1], backdrop, {'P': player, 'b': ball},
                  z_order=['b', 'P'],              # ascii_art.py:184: the flat update schedule
                  groups=[['b', 'P']], program=apprehend_program)


def apprehend_program(world, ch, actions):
  plot, ent, board = world.plot, world.things[ch], world.board
  if ch == 'P':                                   # PlayerSprite.update :76-87
    if actions == 0:
      em.walker_move(ent, board, plot, em.M_W)
    elif actions == 1:
      em.walker_move(ent, board, plot, em.M_E)
    if ent.virtual_position == world.things['b'].virtual_position:
      plot.add_reward(1)
      plot.terminate_episode()
  else:                                           # BallSprite.update :109-131
    em.walker_move(ent, board, plot, em.M_S)
    ent.aux['acc'] += ent.aux['dx']
    if ent.aux['acc'] < -0.5:
      em.walker_move(ent, board, plot, em.M_W)
      ent.aux['acc'] += 1.0
    elif ent.aux['acc'] > 0.5:
      em.walker_move(ent, board, plot, em.M_E)
      ent.aux['acc'] -= 1.0
    if ent.virtual_position[0] >= board.shape[0]:
      plot.add_reward(-1)
      plot.terminate_episode()


# ==========================================================================
# shockwave (SURVEY.md §8f-4): a walker climbing to the safe top row while rings of
# fire expand from random impact points; `layers[...]` look-ups see the STALE board.
# ==========================================================================

def make_shockwave(art, rng, width=2):
  """examples/shockwave.py:181-197.  `rng` is the np.random.RandomState standing
  for NumPy's global generator (np.random.randint, :133)."""
  backdrop, masks = split_art(art, ['P', '@', ' ', '^'], '+')
  shape = backdrop.shape
  player = em.Walker('P', shape, mask_position(masks['P']), impassable='=',
                     confined=True)                                   # :94-96
  wave = em.PlainDrape('@', masks['@'])
  wave.aux.update(width=width, distance=np.zeros(shape), steps=0)     # :122-124
  things = {'P': player, '@': wave, ' ': em.PlainDrape(' ', masks[' ']),
            '^': em.PlainDrape('^', masks['^'])}
  world = em.World(shape[0], shape[1], backdrop, things, z_order=[' ', '^', '@', 'P'],
                   groups=[[' ', '^', 'P', '@']], program=shockwave_program)
  world.rng = rng
  return world


def shockwave_program(world, ch, actions):
  plot, ent, board = world.plot, world.things[ch], world.board
  if ch == 'P':                                   # PlayerSprite.update :98-109
    motion = {0: em.M_N, 1: em.M_W, 2: em.M_E, 3: em.M_STAY}.get(actions) \
        if actions is not None else None
    if motion is not None:
      em.walker_move(ent, board, plot, motion)
  elif ch == '@':                                 # ShockwaveDrape.update :126-165
    aux = ent.aux
    if not ent.curtain.any():
      k = int(world.rng.randint(0, ent.curtain.size))                 # :133
      ir, ic = divmod(k, world.cols)                                  # np.unravel_index
      rr, cc = np.mgrid[0:world.rows, 0:world.cols]
      # ndimage.distance_transform_edt of "everything but the impact point":
      # the Euclidean distance to that point, float64
      aux['distance'] = np.sqrt(((rr - ir) ** 2 + (cc - ic) ** 2).astype(np.float64))
      aux['steps'] = 0
    stale = world.layers                          # engine.py:725: layers of the last render
    ent.curtain[:] = ((aux['distance'] > aux['steps']) &
                      (aux['distance'] <= aux['steps'] + aux['width']) &
                      np.logical_not(stale['=']))
    pos = world.things['P'].position
    if stale['^'][pos]:
      plot.add_reward(1)
      plot.terminate_episode()
    if ent.curtain[pos] and world.things[' '].curtain[pos]:
      plot.add_reward(-1)
      plot.terminate_episode()
    aux['steps'] += 1
  # MinimalDrape.update (' ' and '^') does nothing :168-172
