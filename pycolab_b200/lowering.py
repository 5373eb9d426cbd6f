"""Lower a set-up `Engine` (Python entity objects) to a device game description.

"Recognise and lower" (SURVEY.md §7 H1): game logic upstream is arbitrary Python
in `update()` methods, which cannot run on a GPU.  The fused step kernels
implement the logic of a fixed set of entity classes — the prefabs plus the
concrete classes of the configured example games — and this module maps a
finished `Engine` onto one of those device programs by class identity:

  * an entity class is recognised by (defining module's last name component,
    class name), looked up along its MRO, and only if `update` is not
    overridden below the recognised class;
  * the example modules may be the reference's own files
    (`pycolab/examples/*.py`, imported through `pycolab_b200.compat`) or this
    package's `pycolab_b200/games/*.py`;
  * everything the constructors decided (positions, visibility, curtains,
    patterns, margins, impassable sets, z-order, update groups) is read from
    the live objects, so `make_game()` code runs unchanged.

Anything else raises `NotLoweredError`; there is no CPU fallback.
"""

import numpy as np

from pycolab_b200 import _lib
from pycolab_b200 import things
from pycolab_b200.errors import NotLoweredError
from pycolab_b200.prefab_parts import drapes as prefab_drapes
from pycolab_b200.prefab_parts import sprites as prefab_sprites

# (module tail, class name) -> device role.
LOWERED_CLASSES = {
    ('scrolly_maze', 'PlayerSprite'): 'scrolly.player',
    ('scrolly_maze', 'PatrollerSprite'): 'scrolly.patroller',
    ('scrolly_maze', 'MazeDrape'): 'scrolly.maze',
    ('scrolly_maze', 'CashDrape'): 'scrolly.cash',
    ('warehouse_manager', 'BoxSprite'): 'warehouse.box',
    ('warehouse_manager', 'JudgeDrape'): 'warehouse.judge',
    ('warehouse_manager', 'PlayerSprite'): 'warehouse.player',
    ('extraterrestrial_marauders', 'PlayerSprite'): 'marauders.player',
    ('extraterrestrial_marauders', 'BunkerDrape'): 'marauders.bunker',
    ('extraterrestrial_marauders', 'MarauderDrape'): 'marauders.marauder',
    ('extraterrestrial_marauders', 'UpwardLaserBoltSprite'): 'marauders.up_bolt',
    ('extraterrestrial_marauders', 'DownwardLaserBoltSprite'): 'marauders.down_bolt',
    ('better_scrolly_maze', 'PlayerSprite'): 'better.player',
    ('better_scrolly_maze', 'PatrollerSprite'): 'better.patroller',
    ('better_scrolly_maze', 'CashDrape'): 'better.cash',
    ('four_rooms', 'PlayerSprite'): 'classics.four_rooms',
    ('cliff_walk', 'PlayerSprite'): 'classics.cliff_walk',
    ('chain_walk', 'PlayerSprite'): 'classics.chain_walk',
    ('fluvial_natation', 'PlayerSprite'): 'classics.fluvial',
    ('aperture', 'PlayerSprite'): 'aperture.player',
    ('aperture', 'ApertureDrape'): 'aperture.drape',
    ('hello_world', 'SlidingSprite'): 'hello.slider',
    ('hello_world', 'RollingDrape'): 'hello.roller',
    ('shockwave', 'PlayerSprite'): 'shockwave.player',
    ('shockwave', 'ShockwaveDrape'): 'shockwave.wave',
    ('shockwave', 'MinimalDrape'): 'shockwave.minimal',
    ('apprehend', 'PlayerSprite'): 'apprehend.player',
    ('apprehend', 'BallSprite'): 'apprehend.ball',
    ('t_maze', 'PlayerSprite'): 't_maze.player',
    ('t_maze', 'CueDrape'): 't_maze.cue',
    ('t_maze', 'MazeDrape'): 't_maze.maze',
    ('t_maze', 'SpeckleDrape'): 't_maze.speckle',
    ('t_maze', 'TeleporterDrape'): 't_maze.teleporter',
    ('t_maze', 'GoalDrape'): 't_maze.goal',
    ('ordeal', 'PlayerSprite'): 'ordeal.player',
    ('ordeal', 'DragonduckSprite'): 'ordeal.dragonduck',
    ('ordeal', 'SwordDrape'): 'ordeal.sword',
    # General entities: the reference's test fixtures and this package's twins.
    ('test_things', 'TestMazeWalker'): 'fixture.walker',
    ('test_things', 'TestScrolly'): 'fixture.scrolly',
    ('test_things', 'TestDrape'): 'fixture.drape',
    ('fixtures', 'FixtureMazeWalker'): 'fixture.walker',
    ('fixtures', 'FixtureScrolly'): 'fixture.scrolly',
    ('fixtures', 'FixtureDrape'): 'fixture.drape',
}

# Backdrop subclasses whose update() has a device counterpart.
LOWERED_BACKDROPS = {
    ('fluvial_natation', 'RiverBackdrop'): 'river',
}

_PROGRAM_OF = {'scrolly': _lib.PROG_SCROLLY_MAZE, 'warehouse': _lib.PROG_WAREHOUSE,
               'marauders': _lib.PROG_MARAUDERS}


def source_fingerprint(text):
  """sha256 over the token stream of `text` (a class definition): comments,
  blank lines and the amount of indentation do not count, everything else does."""
  import hashlib
  import io
  import textwrap
  import tokenize
  skip = (tokenize.COMMENT, tokenize.NL, tokenize.NEWLINE, tokenize.ENCODING,
          tokenize.ENDMARKER)
  h = hashlib.sha256()
  for tok in tokenize.generate_tokens(io.StringIO(textwrap.dedent(text)).readline):
    if tok.type in skip:
      continue
    if tok.type in (tokenize.INDENT, tokenize.DEDENT):
      h.update(b'<%d>' % tok.type)
    else:
      h.update(tok.string.encode('utf-8') + b'\0')
  return h.hexdigest()


def _is_known_implementation(klass, key):
  """Is `klass` one of the implementations the device program was written from?

  Classes of this package (`pycolab_b200.games.*`: set-up twins whose update()
  only says "runs on the device") are trusted by module.  Any other module —
  the reference's own example file loaded through `compat`, or a user's copy of
  it — must match the reference's source for that class token for token: a copy
  with an edited update() (another reward, rule or termination) would otherwise
  be silently replaced by the stock kernel."""
  if klass.__module__.startswith('pycolab_b200.'):
    return True
  from pycolab_b200 import _fingerprints
  want = _fingerprints.KNOWN.get(key)
  if want is None:
    return False
  import inspect
  try:
    text = inspect.getsource(klass)
  except (OSError, TypeError):
    return False
  try:
    return source_fingerprint(text) == want
  except Exception:              # noqa: BLE001 - unparsable source is not a known class
    return False


def role_of(entity):
  """Device role of `entity`, or raise NotLoweredError."""
  cls = type(entity)
  for klass in cls.__mro__:
    key = (klass.__module__.rsplit('.', 1)[-1], klass.__name__)
    if key in LOWERED_CLASSES:
      if cls.update is not klass.update:
        raise NotLoweredError(
            '{} overrides update() of the lowered class {}.{}'.format(
                cls.__name__, *key))
      if not _is_known_implementation(klass, key):
        raise NotLoweredError(
            'class {}.{} is named like the lowered class {}.{} but its source differs '
            'from the implementation the device program restates; edited copies are not '
            'replaced by the stock kernel'.format(klass.__module__, klass.__name__, *key))
      return LOWERED_CLASSES[key]
  raise NotLoweredError(
      'no device program for entity class {}.{} (character {!r}); lowered classes: '
      '{}'.format(cls.__module__, cls.__name__, getattr(entity, 'character', '?'),
                  sorted('%s.%s' % k for k in LOWERED_CLASSES)))


def round_up(x, m):
  return (x + m - 1) // m * m


def pack_rows(mask, words):
  """bool [R, C] -> uint32 [R, words]; cell c is bit c&31 of word c>>5."""
  mask = np.asarray(mask, dtype=bool)
  rows, cols = mask.shape
  assert words * 32 >= cols
  padded = np.zeros((rows, words * 32), dtype=np.uint8)
  padded[:, :cols] = mask
  packed = np.packbits(padded.reshape(rows, words, 32), axis=2, bitorder='little')
  return np.ascontiguousarray(packed).view('<u4').reshape(rows, words)


def unpack_rows(packed, cols):
  packed = np.ascontiguousarray(packed, dtype='<u4')
  rows, words = packed.shape
  bits = np.unpackbits(packed.view(np.uint8).reshape(rows, words * 4), axis=1,
                       bitorder='little')
  return bits[:, :cols].astype(bool)


def char_set_mask(chars):
  out = [0, 0, 0, 0]
  for ch in chars:
    code = ord(ch)
    if code > 127:
      raise NotLoweredError('non-ASCII impassable character {!r}'.format(ch))
    out[code >> 5] |= 1 << (code & 31)
  return out


class LoweredGame(object):
  """One level's device description: spec fields + template arrays."""

  def __init__(self):
    self.program = 0
    self.rows = self.cols = self.pitch = 0
    self.sprite_chars = ''
    self.drape_chars = ''
    self.impassable = []
    self.confined = []
    self.egocentric = []
    self.margins = []
    self.z_order = ''
    self.groups = []
    self.pattern_rows = self.pattern_cols = self.pattern_words = 0
    self.bits_words = 0
    self.backdrop = None        # u8 [H, pitch]
    self.patterns = {}          # drape index -> u32 [PH, PWW]
    self.pattern_mutable = {}   # drape index -> bool
    self.pattern_redraw = {}    # drape index -> u32 [PH, PWW]: reset template of a pattern the
                                # device redraws at every restart (when an RNG is bound)
    self.bits = {}              # drape index -> u32 [H, BW]
    self.sprites = None         # i32 [S, 8]
    self.drapes = None          # i32 [D, 8]
    self.plot = None            # i32 [16]
    self.needs_rng = False
    self.rng_kind = 'numpy'     # whose MT19937 stream the device continues: NumPy's legacy
                                # RandomState ('numpy') or Python's `random` ('python')
    self.backdrop_chars = ''
    self.drape_kind = None      # per drape: 1 = Scrolly (fixture program only)
    self.dynamic_z = False      # per-env z-order array (Plot.change_z_order)
    self.program_arg = [0] * 8  # pcl_spec.program_arg
    self.reward_type = int      # the reference's reward type (classics pay floats)
    self.float_reward = False   # rewards are not integers: pcl_outputs.d_reward_f64
    self.backdrop_role = None   # device counterpart of a Backdrop with update() logic
    self.scroll_groups = ['']   # names of the scrolling groups, index = device group id
    self.sprite_group = []      # per sprite: index into scroll_groups
    self.drape_group = []       # per drape
    self.group_records = None   # i32 [MAX_SCROLL_GROUPS, 4] reset template (groups >= 1)
    self.sync_plot = None       # callable(engine, plot words): mirror device plot state into
                                # the Python Plot after a step (games that keep dict entries)

  def signature(self):
    """Everything that must agree between envs sharing one handle."""
    return (self.program, self.rows, self.cols, self.sprite_chars, self.drape_chars,
            tuple(map(tuple, self.impassable)), tuple(self.confined),
            tuple(self.egocentric), tuple(map(tuple, self.margins)), self.z_order,
            tuple(self.groups), self.pattern_rows, self.pattern_cols,
            tuple(self.program_arg), tuple(self.scroll_groups), tuple(self.sprite_group),
            tuple(self.drape_group))

  def make_spec(self, auto_reset):
    s = _lib.Spec()
    s.abi_version = _lib.ABI_VERSION
    s.program = self.program
    s.rows, s.cols, s.pitch = self.rows, self.cols, self.pitch
    s.n_sprites, s.n_drapes = len(self.sprite_chars), len(self.drape_chars)
    s.auto_reset = 1 if auto_reset else 0
    s.pattern_rows, s.pattern_cols = self.pattern_rows, self.pattern_cols
    s.pattern_words, s.bits_words = self.pattern_words, self.bits_words
    for i, ch in enumerate(self.sprite_chars):
      s.sprite_char[i] = ord(ch)
      for w in range(4):
        s.impassable[i][w] = self.impassable[i][w]
      s.sprite_confined[i] = int(self.confined[i])
      s.sprite_egocentric[i] = int(self.egocentric[i])
    for i, ch in enumerate(self.drape_chars):
      s.drape_char[i] = ord(ch)
      s.margins[i][0], s.margins[i][1] = self.margins[i]
      if self.drape_kind is not None:
        s.drape_kind[i] = self.drape_kind[i]
    for i, ch in enumerate(self.z_order):
      s.z_order[i] = ord(ch)
    for i, v in enumerate(self.program_arg):
      s.program_arg[i] = int(v)
    s.n_scroll_groups = len(self.scroll_groups)
    for i, g in enumerate(self.sprite_group):
      s.sprite_group[i] = g
    for i, g in enumerate(self.drape_group):
      s.drape_group[i] = g
    s.n_groups = len(self.groups)
    k = 0
    for g, group in enumerate(self.groups):
      s.group_len[g] = len(group)
      for ch in group:
        s.group_chars[k] = ord(ch)
        k += 1
    return s


def _sprite_record(sprite, aux0=0, aux1=0, aux2=0):
  if isinstance(sprite, prefab_sprites.MazeWalker):
    vrow, vcol = sprite.virtual_position
    prior = sprite._prior_visible
  else:
    vrow, vcol = sprite.position
    prior = None
  flags = (1 if sprite.visible else 0) | ((0 if prior is None else 2 if prior else 1) << 1)
  return [int(sprite.position[0]), int(sprite.position[1]), int(vrow), int(vcol),
          flags, int(aux0), int(aux1), int(aux2)]


def _walker_meta(sprite, named_groups=False):
  if not isinstance(sprite, prefab_sprites.MazeWalker):
    raise NotLoweredError('sprite {!r} is not a MazeWalker'.format(sprite.character))
  if sprite._scrolling_group != '' and not named_groups:
    raise NotLoweredError('named scrolling groups are lowered by the general program only')
  if (type(sprite)._on_board_exit is not prefab_sprites.MazeWalker._on_board_exit or
      type(sprite)._on_board_enter is not prefab_sprites.MazeWalker._on_board_enter):
    raise NotLoweredError('overridden MazeWalker board exit/enter hooks are not lowered')
  return (char_set_mask(sprite.impassable), bool(sprite._confined_to_board),
          bool(sprite._egocentric_scroller))


def _plot_record(**words):
  rec = [0] * _lib.PLOT_WORDS
  rec[_lib.P_FRAME] = -1
  rec[_lib.P_ORDER_FRAME] = _lib.NEVER
  for name, value in words.items():
    rec[getattr(_lib, 'P_' + name.upper())] = int(value)
  return rec


def _common(engine, game, program):
  game.program = program
  game.rows, game.cols = engine.rows, engine.cols
  game.pitch = round_up(engine.cols, 16)
  game.bits_words = (engine.cols + 31) // 32 + 1
  game.z_order = ''.join(engine.z_order)
  game.groups = [''.join(e.character for e in entities)
                 for _, entities in sorted(engine._update_groups.items())]
  backdrop = engine.backdrop
  game.backdrop_role = None
  if type(backdrop).update is not things.Backdrop.update:
    for klass in type(backdrop).__mro__:
      key = (klass.__module__.rsplit('.', 1)[-1], klass.__name__)
      if (key in LOWERED_BACKDROPS and type(backdrop).update is klass.update and
          _is_known_implementation(klass, key)):
        game.backdrop_role = LOWERED_BACKDROPS[key]
        break
    else:
      raise NotLoweredError('no device program for the update() logic of Backdrop class '
                            '{}.{}'.format(type(backdrop).__module__, type(backdrop).__name__))
  game.backdrop = np.zeros((engine.rows, game.pitch), dtype=np.uint8)
  game.backdrop[:, :engine.cols] = backdrop.curtain
  game.backdrop_chars = ''.join(sorted(backdrop.palette))
  # Unoccluded layers (rendering.py:187-301) change what `layers[...]` look-ups
  # inside update() see; only programs whose logic never reads layers keep
  # their semantics, so only those accept occlusion_in_layers=False.
  if not engine._occlusion_in_layers and program not in (_lib.PROG_SCROLLY_MAZE,
                                                         _lib.PROG_FIXTURE):
    raise NotLoweredError('occlusion_in_layers=False is lowered only for games whose '
                          'entities never consult `layers`')


def _set_sprites(game, sprites, records, named_groups=False):
  game.sprite_chars = ''.join(s.character for s in sprites)
  meta = [_walker_meta(s, named_groups) for s in sprites]
  game.impassable = [m[0] for m in meta]
  game.confined = [m[1] for m in meta]
  game.egocentric = [m[2] for m in meta]
  game.sprites = np.array(records, dtype=np.int32).reshape(len(sprites), _lib.SPRITE_WORDS)


def _scrolly_record(drape, aux0=0, aux1=0):
  r, c = drape._northwest_corner
  return [int(r), int(c), int(r), int(c), _lib.NEVER, int(aux0), int(aux1), 0]


def _lower_scrolly_maze(engine, roles):
  th = engine.things
  want = {'P': 'scrolly.player', 'a': 'scrolly.patroller', 'b': 'scrolly.patroller',
          'c': 'scrolly.patroller', '#': 'scrolly.maze', '@': 'scrolly.cash'}
  if roles != want:
    raise NotLoweredError('scrolly_maze program needs exactly {} (got {})'.format(want, roles))
  game = LoweredGame()
  _common(engine, game, _lib.PROG_SCROLLY_MAZE)
  sprites = [th[c] for c in 'Pabc']
  records = [_sprite_record(th['P'], aux0=0, aux1=_lib.NEVER)]
  records += [_sprite_record(th[c], aux0=int(bool(th[c]._moving_east))) for c in 'abc']
  _set_sprites(game, sprites, records)
  walls, coins = th['#'], th['@']
  for d in (walls, coins):
    if d._scrolling_group != '':
      raise NotLoweredError('only the default scrolling group is lowered')
    if d.whole_pattern.shape != walls.whole_pattern.shape:
      raise NotLoweredError('Scrolly patterns of different shapes')
    if tuple(d._board_shape) != (engine.rows, engine.cols):
      raise NotLoweredError('Scrolly board_shape differs from the Engine board')
  game.drape_chars = '#@'
  game.margins = [(-1, -1) if d._scroll_margins is None else tuple(d._scroll_margins)
                  for d in (walls, coins)]
  game.pattern_rows, game.pattern_cols = walls.whole_pattern.shape
  # zero-padded row: the kernel stages 2 * ceil((63 + W) / 64) words per window row
  # starting at an even word (4 words up to 64 columns).
  slack = 3 if engine.cols <= 64 else 2 * ((63 + engine.cols + 63) // 64) + 1
  game.pattern_words = round_up((game.pattern_cols + 31) // 32 + slack, 2)
  game.patterns = {0: pack_rows(walls.whole_pattern, game.pattern_words),
                   1: pack_rows(coins.whole_pattern, game.pattern_words)}
  game.pattern_mutable = {0: False, 1: True}
  game.drapes = np.array([_scrolly_record(walls), _scrolly_record(coins, -1, -1)],
                         dtype=np.int32)
  game.plot = np.array(_plot_record(aux0=int(coins.whole_pattern.sum())), dtype=np.int32)
  return game


def _lower_warehouse(engine, roles):
  th = engine.things
  groups = [[e.character for e in ents]
            for _, ents in sorted(engine._update_groups.items())]
  if len(groups) != 3 or groups[1] != ['X'] or groups[2] != ['P']:
    raise NotLoweredError('warehouse program needs update groups [boxes, [X], [P]]')
  boxes = groups[0]
  for ch in boxes:
    if roles.get(ch) != 'warehouse.box':
      raise NotLoweredError('unexpected entity {!r} in the box group'.format(ch))
  if roles.get('X') != 'warehouse.judge' or roles.get('P') != 'warehouse.player':
    raise NotLoweredError('warehouse program needs JudgeDrape X and PlayerSprite P')
  game = LoweredGame()
  _common(engine, game, _lib.PROG_WAREHOUSE)
  sprites = [th[c] for c in boxes] + [th['P']]
  _set_sprites(game, sprites, [_sprite_record(s) for s in sprites])
  judge = th['X']
  if judge.curtain.any():
    raise NotLoweredError("a pre-filled 'X' curtain is not lowered")
  game.drape_chars = 'X'
  game.margins = [(-1, -1)]
  rec = [0] * _lib.DRAPE_WORDS
  rec[_lib.D_LAST_FRAME] = _lib.NEVER
  rec[_lib.D_AUX0] = int(judge._last_num_boxes_on_goals)
  game.drapes = np.array([rec], dtype=np.int32)
  game.plot = np.array(_plot_record(), dtype=np.int32)
  if '_' not in engine.backdrop.palette:
    raise NotLoweredError("warehouse backdrop has no goal character '_'")
  return game


def _lower_marauders(engine, roles):
  th = engine.things
  want = {'P': 'marauders.player', 'B': 'marauders.bunker', 'X': 'marauders.marauder',
          'a': 'marauders.up_bolt', 'b': 'marauders.up_bolt', 'c': 'marauders.up_bolt',
          'd': 'marauders.up_bolt', 'y': 'marauders.down_bolt', 'z': 'marauders.down_bolt'}
  if roles != want:
    raise NotLoweredError('marauders program needs exactly {} (got {})'.format(want, roles))
  game = LoweredGame()
  _common(engine, game, _lib.PROG_MARAUDERS)
  sprites = [th[c] for c in 'Pabcdyz']
  _set_sprites(game, sprites, [_sprite_record(s) for s in sprites])
  game.drape_chars = 'BX'
  game.margins = [(-1, -1), (-1, -1)]
  game.bits = {0: pack_rows(th['B'].curtain, game.bits_words),
               1: pack_rows(th['X'].curtain, game.bits_words)}
  recs = []
  for ch in 'BX':
    rec = [0] * _lib.DRAPE_WORDS
    rec[_lib.D_LAST_FRAME] = _lib.NEVER
    recs.append(rec)
  recs[1][_lib.D_AUX0] = int(th['X']._dx)
  game.drapes = np.array(recs, dtype=np.int32)
  game.plot = np.array(_plot_record(aux0=_lib.NEVER, aux1=_lib.NEVER), dtype=np.int32)
  game.needs_rng = True
  return game


def _lower_better_scrolly(engine, roles):
  th = engine.things
  want = {'P': 'better.player', 'a': 'better.patroller', 'b': 'better.patroller',
          'c': 'better.patroller', '@': 'better.cash'}
  if roles != want:
    raise NotLoweredError('better_scrolly_maze program needs exactly {} (got {})'.format(
        want, roles))
  game = LoweredGame()
  _common(engine, game, _lib.PROG_BETTER_SCROLLY)
  sprites = [th[c] for c in 'Pabc']
  records = [_sprite_record(th['P'])]
  records += [_sprite_record(th[c], aux0=int(bool(th[c]._moving_east))) for c in 'abc']
  _set_sprites(game, sprites, records)
  game.drape_chars = '@'
  game.margins = [(-1, -1)]
  game.bits = {0: pack_rows(th['@'].curtain, game.bits_words)}
  rec = [0] * _lib.DRAPE_WORDS
  rec[_lib.D_LAST_FRAME] = _lib.NEVER
  game.drapes = np.array([rec], dtype=np.int32)
  game.plot = np.array(_plot_record(aux0=int(th['@'].curtain.sum())), dtype=np.int32)
  return game


def _lower_classics(engine, roles):
  """examples/classics: one MazeWalker 'P', no drapes; the rule set rides in
  pcl_spec.program_arg (four_rooms.py:78 fixes the goal cell at (4, 3))."""
  if list(roles) != ['P']:
    raise NotLoweredError('classics programs have exactly one entity, P (got {})'.format(roles))
  game = LoweredGame()
  _common(engine, game, _lib.PROG_CLASSICS)
  rule = roles['P'].split('.')[1]
  game.program_arg[0] = {'four_rooms': _lib.CLASSIC_FOUR_ROOMS,
                         'cliff_walk': _lib.CLASSIC_CLIFF_WALK,
                         'chain_walk': _lib.CLASSIC_CHAIN_WALK,
                         'fluvial': _lib.CLASSIC_FLUVIAL}[rule]
  if rule == 'four_rooms':
    game.program_arg[1], game.program_arg[2] = 4, 3
  if (rule == 'fluvial') != (game.backdrop_role == 'river'):
    raise NotLoweredError('the river Backdrop and the swimmer are lowered only together')
  if rule == 'fluvial':
    game.program_arg[1], game.program_arg[2] = 1, 4      # curtain[1:4, :], fluvial_natation.py:110
  if game.rows * game.pitch > 8192:
    raise NotLoweredError('classics boards are staged whole in shared memory (<= 8 KiB)')
  player = engine.things['P']
  _set_sprites(game, [player], [_sprite_record(player)])
  if rule == 'fluvial' and any(game.impassable[0]):
    raise NotLoweredError('the river program needs a swimmer with no impassable characters')
  game.drapes = np.zeros((0, _lib.DRAPE_WORDS), dtype=np.int32)
  game.plot = np.array(_plot_record(), dtype=np.int32)
  game.reward_type = int if rule == 'fluvial' else float
  return game


def _lower_hello(engine, roles):
  """examples/hello_world.py:58-118: up to four SlidingSprites (plain Sprites, each
  with one of four diagonal direction sets) and one RollingDrape, one update group."""
  th = engine.things
  sliders = [c for c in ''.join(_update_order(engine)) if roles[c] == 'hello.slider']
  rollers = [c for c, r in roles.items() if r == 'hello.roller']
  if not 1 <= len(sliders) <= 4 or len(rollers) != 1:
    raise NotLoweredError('hello_world program needs 1-4 SlidingSprites and one RollingDrape')
  game = LoweredGame()
  _common(engine, game, _lib.PROG_HELLO)
  if len(game.groups) != 1:
    raise NotLoweredError('hello_world entities share one update group')
  records = []
  for ch in sliders:
    sp = th[ch]
    sets = list(zip(type(sp)._DX, type(sp)._DY))
    try:
      k = sets.index((sp._dx, sp._dy))
    except ValueError:
      raise NotLoweredError('SlidingSprite {!r} uses an unknown direction set'.format(ch))
    records.append(_sprite_record(sp, aux0=k))
  game.sprite_chars = ''.join(sliders)
  game.impassable = [[0, 0, 0, 0]] * len(sliders)
  game.confined = [False] * len(sliders)
  game.egocentric = [False] * len(sliders)
  game.sprites = np.array(records, dtype=np.int32).reshape(len(sliders), _lib.SPRITE_WORDS)
  game.drape_chars = rollers[0]
  game.margins = [(-1, -1)]
  rec = [0] * _lib.DRAPE_WORDS
  rec[_lib.D_LAST_FRAME] = _lib.NEVER
  game.drapes = np.array([rec], dtype=np.int32)
  game.bits[0] = pack_rows(th[rollers[0]].curtain, game.bits_words)   # the un-rolled curtain
  game.plot = np.array(_plot_record(), dtype=np.int32)
  for k, ch in enumerate(game.z_order):          # the kernel paints in this order
    game.program_arg[k] = ord(ch)
  return game


def _f64_words(x):
  """float64 -> (lo, hi) int32 words, as the kernels' __hiloint2double reads them."""
  lo, hi = np.array([x], dtype='<f8').view('<i4')
  return int(lo), int(hi)


def _lower_apprehend(engine, roles):
  """examples/apprehend.py:56-131: the catcher 'P' and the falling ball, one group
  [ball, catcher].  The ball's float64 slope (drawn when the Python sprite was built)
  and accumulator travel as bit patterns; `needs_rng` lets a BATCHED engine draw a new
  slope per episode on the device from per-env `random.Random` states."""
  th = engine.things
  players = [c for c, r in roles.items() if r == 'apprehend.player']
  balls = [c for c, r in roles.items() if r == 'apprehend.ball']
  if len(players) != 1 or len(balls) != 1 or len(roles) != 2:
    raise NotLoweredError('apprehend program needs one PlayerSprite and one BallSprite')
  game = LoweredGame()
  _common(engine, game, _lib.PROG_APPREHEND)
  pl, ball = th[players[0]], th[balls[0]]
  if _update_order(engine) != [balls[0], players[0]] or len(game.groups) != 1:
    raise NotLoweredError('apprehend program needs update_schedule [ball, player]')
  if game.z_order != balls[0] + players[0]:
    raise NotLoweredError('apprehend program draws the player over the ball')
  lo, hi = _f64_words(ball._dx)
  _set_sprites(game, [pl, ball], [_sprite_record(pl), _sprite_record(ball, aux0=lo, aux1=hi)])
  alo, ahi = _f64_words(ball._x_accumulator)
  game.drape_chars = ''
  game.margins = []
  game.drapes = np.zeros((0, _lib.DRAPE_WORDS), dtype=np.int32)
  game.plot = np.array(_plot_record(aux0=alo, aux1=ahi), dtype=np.int32)
  game.needs_rng = True
  game.rng_kind = 'python'
  return game


def _lower_shockwave(engine, roles):
  """examples/shockwave.py:91-197: the player, the ShockwaveDrape and the two static
  MinimalDrapes the wave's update() names by character (' ' danger zone, '^' safe
  zone; walls are the backdrop's '=')."""
  th = engine.things
  by_role = {}
  for ch, role in roles.items():
    by_role.setdefault(role, []).append(ch)
  if (sorted(by_role) != ['shockwave.minimal', 'shockwave.player', 'shockwave.wave'] or
      len(by_role['shockwave.player']) != 1 or len(by_role['shockwave.wave']) != 1 or
      sorted(by_role['shockwave.minimal']) != [' ', '^']):
    raise NotLoweredError("shockwave program needs one PlayerSprite, one ShockwaveDrape and "
                          "MinimalDrapes ' ' and '^' (got {})".format(roles))
  p_ch, w_ch = by_role['shockwave.player'][0], by_role['shockwave.wave'][0]
  game = LoweredGame()
  _common(engine, game, _lib.PROG_SHOCKWAVE)
  order = _update_order(engine)
  if len(game.groups) != 1 or sorted(order[:2]) != [' ', '^'] or order[2:] != [p_ch, w_ch]:
    raise NotLoweredError("shockwave program needs update_schedule [' ', '^', P, wave]")
  if game.z_order != ' ^' + w_ch + p_ch:
    raise NotLoweredError("shockwave program needs z_order [' ', '^', wave, P]")
  pl, wave = th[p_ch], th[w_ch]
  if set(pl.impassable) != {'='}:
    raise NotLoweredError("the wave's update() stops at '=': the player must do the same")
  if engine.rows > 32 or engine.cols > 64:
    raise NotLoweredError('shockwave program: boards up to 32 x 64')
  _set_sprites(game, [pl], [_sprite_record(pl)])
  game.drape_chars = w_ch + ' ^'
  game.margins = [(-1, -1)] * 3
  recs = []
  for _ in range(3):
    rec = [0] * _lib.DRAPE_WORDS
    rec[_lib.D_LAST_FRAME] = _lib.NEVER
    recs.append(rec)
  recs[0][_lib.D_AUX1] = int(wave._steps_since_impact)
  if wave.curtain.any() or np.any(wave._distance_from_impact):
    raise NotLoweredError('a ShockwaveDrape that is already burning is not lowered')
  game.drapes = np.array(recs, dtype=np.int32)
  for d, ch in enumerate(game.drape_chars):
    game.bits[d] = pack_rows(th[ch].curtain, game.bits_words)
  game.plot = np.array(_plot_record(), dtype=np.int32)
  game.program_arg[0] = int(wave._width)
  game.needs_rng = True                         # np.random.randint, shockwave.py:133
  return game


def _lower_t_maze(engine, roles):
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
  recs = [[0] * _lib.DRAPE_WORDS]
  recs[0][_lib.D_LAST_FRAME] = _lib.NEVER
  recs[0][_lib.D_AUX0] = 0 if cue.which_goal == 'left' else 1
  recs[0][_lib.D_AUX1] = 1 if plot.get('yo_we_have_teleported') else 0
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
  game.needs_rng = True
  game.rng_kind = 't_maze'        # two MT19937 streams per env: Python's random, NumPy's
  game.reward_type = float
  game.float_reward = True

  def sync_plot(eng, words):
    p, b = eng.the_plot, eng.batched
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
    eng.things['Q'].which_goal = 'left' if q[_lib.D_AUX0] == 0 else 'right'
  game.sync_plot = sync_plot
  return game


def _update_order(engine):
  return [e.character for _, ents in sorted(engine._update_groups.items()) for e in ents]


_ORDEAL_CHAPTERS = {'castle': _lib.ORDEAL_CASTLE, 'cavern': _lib.ORDEAL_CAVERN,
                    'kansas': _lib.ORDEAL_KANSAS}


def _lower_ordeal(engine, roles):
  """examples/ordeal.py:74-266: one chapter of the Story.  Which chapter this Engine
  is comes from its entities (castle: P + D, cavern: P + S, kansas: P) and must agree
  with `the_plot.this_chapter`, which Story set before its_showtime()
  (storytelling.py:453-454).  The Plot entries the game code keeps in dict slots —
  `has_sword`, `last_position` — and the chapter bookkeeping enter the device plot
  record here and are mirrored back after every step (`sync_plot`)."""
  th, plot = engine.things, engine.the_plot
  by_role = sorted(roles.values())
  chapter = {('ordeal.dragonduck', 'ordeal.player'): 'castle',
             ('ordeal.player', 'ordeal.sword'): 'cavern',
             ('ordeal.player',): 'kansas'}.get(tuple(by_role))
  if chapter is None:
    raise NotLoweredError('ordeal program: unknown chapter with entities {}'.format(roles))
  if plot.this_chapter is not None and plot.this_chapter != chapter:
    raise NotLoweredError('ordeal chapter {!r} is running under the Story key {!r}'.format(
        chapter, plot.this_chapter))
  if plot.prior_chapter is not None and plot.prior_chapter not in _ORDEAL_CHAPTERS:
    raise NotLoweredError('ordeal chapter entered from an unknown chapter {!r}'.format(
        plot.prior_chapter))
  game = LoweredGame()
  _common(engine, game, _lib.PROG_ORDEAL)
  if len(game.groups) != 1:
    raise NotLoweredError('ordeal chapters have one update group')
  player = [c for c, r in roles.items() if r == 'ordeal.player'][0]
  sprites = [th[player]] + [th[c] for c, r in roles.items() if r == 'ordeal.dragonduck']
  if game.groups[0][0] != player:
    raise NotLoweredError('the ordeal player must update first')
  if game.rows * game.pitch > 8192:
    raise NotLoweredError('ordeal boards are staged whole in shared memory (<= 8 KiB)')
  _set_sprites(game, sprites, [_sprite_record(s) for s in sprites])
  game.program_arg[0] = _ORDEAL_CHAPTERS[chapter]
  drapes = [c for c, r in roles.items() if r == 'ordeal.sword']
  game.drape_chars = ''.join(drapes)
  game.margins = [(-1, -1)] * len(drapes)
  game.drapes = np.zeros((len(drapes), _lib.DRAPE_WORDS), dtype=np.int32)
  for d, ch in enumerate(drapes):
    game.drapes[d, _lib.D_LAST_FRAME] = _lib.NEVER
    game.bits[d] = pack_rows(th[ch].curtain, game.bits_words)
  last = plot.get('last_position')
  game.plot = np.array(_plot_record(
      aux0=1 if plot.get('has_sword') else 0,
      aux1=-1 if last is None else (int(last[0]) << 16) | int(last[1]),
      aux2=_lib.ORDEAL_NEXT_UNSET,
      aux3=_ORDEAL_CHAPTERS.get(plot.prior_chapter, 0)), dtype=np.int32)
  game.dynamic_z = len(sprites) + len(drapes) == 2      # the kernel reads (castle: rewrites) it
  game.reward_type = float                              # ordeal.py pays 1.0 / -1.0
  names = {v: k for k, v in _ORDEAL_CHAPTERS.items()}

  def sync_plot(eng, words):
    p = eng.the_plot
    if words[_lib.P_AUX0]:
      p['has_sword'] = True
    if words[_lib.P_AUX1] >= 0:
      p['last_position'] = things.Sprite.Position(int(words[_lib.P_AUX1]) >> 16,
                                                  int(words[_lib.P_AUX1]) & 0xffff)
    if words[_lib.P_AUX2] != _lib.ORDEAL_NEXT_UNSET:
      p.next_chapter = names.get(int(words[_lib.P_AUX2]))   # 0 -> None: the story ends
  game.sync_plot = sync_plot
  return game


def _lower_aperture(engine, roles):
  """examples/aperture.py:188-196: sprite 'A' + the aperture drape.  The drape's
  state is its `_apertures` list (at most two cells) in the record's AUX words."""
  players = [c for c, r in roles.items() if r == 'aperture.player']
  drapes = [c for c, r in roles.items() if r == 'aperture.drape']
  if len(players) != 1 or len(drapes) != 1 or len(roles) != 2:
    raise NotLoweredError('aperture program needs one player and one aperture drape '
                          '(got {})'.format(roles))
  game = LoweredGame()
  _common(engine, game, _lib.PROG_APERTURE)
  player, drape = engine.things[players[0]], engine.things[drapes[0]]
  if game.z_order != drapes[0] + players[0] or game.groups != [players[0], drapes[0]]:
    raise NotLoweredError('aperture program needs update groups [[player], [drape]] and the '
                          'player drawn over the drape')
  if drape.curtain.any() or list(drape._apertures) != [None, None]:
    raise NotLoweredError('the aperture drape must start with no apertures')
  if game.rows * game.pitch > 8192:
    raise NotLoweredError('aperture boards are staged whole in shared memory (<= 8 KiB)')
  _set_sprites(game, [player], [_sprite_record(player)])
  game.drape_chars = drapes[0]
  game.margins = [(-1, -1)]
  rec = [0] * _lib.DRAPE_WORDS
  rec[_lib.D_LAST_FRAME] = _lib.NEVER
  rec[_lib.D_AUX0] = rec[_lib.D_AUX1] = -1
  game.drapes = np.array([rec], dtype=np.int32)
  game.plot = np.array(_plot_record(), dtype=np.int32)
  return game


def _lower_fixture(engine, roles):
  th = engine.things
  game = LoweredGame()
  _common(engine, game, _lib.PROG_FIXTURE)
  order = ''.join(game.groups)
  sprite_chars = [c for c in order if roles[c] == 'fixture.walker']
  drape_chars = [c for c in order if roles[c] != 'fixture.walker']
  if len(sprite_chars) > _lib.MAX_SPRITES or len(drape_chars) > _lib.MAX_DRAPES:
    raise NotLoweredError('too many entities for the general device program')
  sprites = [th[c] for c in sprite_chars]
  _set_sprites(game, sprites, [_sprite_record(s, aux0=0, aux1=_lib.NEVER) for s in sprites],
               named_groups=True)
  # Scrolling groups (protocols/scrolling.py:198-241): one device record per name.
  names = []
  for ch in order:
    name = getattr(th[ch], '_scrolling_group', None)
    if name is not None and name not in names:
      names.append(name)
  names = names or ['']
  if len(names) > _lib.MAX_SCROLL_GROUPS:
    raise NotLoweredError('more than {} scrolling groups'.format(_lib.MAX_SCROLL_GROUPS))
  game.scroll_groups = names
  game.sprite_group = [names.index(th[c]._scrolling_group) for c in sprite_chars]
  game.drape_group = [names.index(getattr(th[c], '_scrolling_group', names[0]))
                      for c in drape_chars]
  game.group_records = np.zeros((_lib.MAX_SCROLL_GROUPS, _lib.GROUP_WORDS), dtype=np.int32)
  game.group_records[:, _lib.G_ORDER_FRAME] = _lib.NEVER
  game.drape_chars = ''.join(drape_chars)
  game.drape_kind, game.margins, recs = [], [], []
  shape = None
  for d, ch in enumerate(drape_chars):
    ent = th[ch]
    if roles[ch] == 'fixture.scrolly':
      if shape not in (None, ent.whole_pattern.shape):
        raise NotLoweredError('Scrolly patterns of different shapes')
      shape = ent.whole_pattern.shape
      game.drape_kind.append(1)
      game.margins.append((-1, -1) if ent._scroll_margins is None
                          else tuple(ent._scroll_margins))
      recs.append(_scrolly_record(ent))
    else:
      game.drape_kind.append(0)
      game.margins.append((-1, -1))
      rec = [0] * _lib.DRAPE_WORDS
      rec[_lib.D_LAST_FRAME] = _lib.NEVER
      recs.append(rec)
      game.bits[d] = pack_rows(ent.curtain, game.bits_words)
  if shape is not None:
    game.pattern_rows, game.pattern_cols = shape
    game.pattern_words = round_up((shape[1] + 31) // 32 + 3, 2)
    for d, ch in enumerate(drape_chars):
      if game.drape_kind[d]:
        game.patterns[d] = pack_rows(th[ch].whole_pattern, game.pattern_words)
        game.pattern_mutable[d] = False
  game.drapes = np.array(recs, dtype=np.int32).reshape(len(drape_chars), _lib.DRAPE_WORDS)
  game.plot = np.array(_plot_record(), dtype=np.int32)
  game.dynamic_z = True
  return game


def lower(engine):
  """`Engine` (set-up finished, not yet showtime) -> `LoweredGame`."""
  roles = {ch: role_of(ent) for ch, ent in engine.things.items()}
  families = {role.split('.')[0] for role in roles.values()}
  if len(families) != 1:
    raise NotLoweredError('entities from different game programs: {}'.format(roles))
  family = families.pop()
  lowerers = {'scrolly': _lower_scrolly_maze, 'warehouse': _lower_warehouse,
              'marauders': _lower_marauders, 'fixture': _lower_fixture,
              'classics': _lower_classics, 'better': _lower_better_scrolly,
              'aperture': _lower_aperture, 'ordeal': _lower_ordeal,
              'hello': _lower_hello, 'apprehend': _lower_apprehend,
              'shockwave': _lower_shockwave, 't_maze': _lower_t_maze}
  if family not in lowerers:
    raise NotLoweredError(family)
  game = lowerers[family](engine, roles)
  if game.backdrop_role is not None and family != 'classics':
    raise NotLoweredError('a Backdrop with update() logic is lowered only with its own game')
  return game
