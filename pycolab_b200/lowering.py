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

Anything else raises `NotLoweredError`; there is no CPU fallback.  This module
keeps what every program shares; each program's own `lower` and host hooks are
in `pycolab_b200/programs/<program>.py`, named after its `csrc/<program>.cu`.
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
    ('cued_catch', 'PlayerSprite'): 'cued_catch.player',
    ('cued_catch', 'BallSprite'): 'cued_catch.ball',
    ('cued_catch', 'CueDrape'): 'cued_catch.cue',
    ('sequence_recall', 'PlayerSprite'): 'sequence_recall.player',
    ('sequence_recall', 'MaskDrape'): 'sequence_recall.mask',
    ('sequence_recall', 'WaitForSeekDrape'): 'sequence_recall.wait',
    ('box_world', 'PlayerSprite'): 'box_world.player',
    ('box_world', 'BoxThing'): 'box_world.thing',
    ('box_world', 'GemDrape'): 'box_world.gem',
    ('box_world', 'KeyDrape'): 'box_world.key',
    ('box_world', 'LockDrape'): 'box_world.lock',
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

# Module-level functions a device program restates besides the entities' update():
# sequence_recall's restart draw is _make_program's.
LOWERED_FUNCTIONS = {
    ('sequence_recall', '_make_program'),
}

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
  """Device role of `entity`, or raise NotLoweredError.  A class registered with
  `compiler.register` (along the MRO, update() not overridden below it) comes first."""
  cls = type(entity)
  from pycolab_b200 import compiler
  compiled = compiler.registered(cls)
  if compiled is not None:
    return {'sprite': 'compiled.walker', 'plain': 'compiled.sprite',
            'scrolly': 'compiled.scrolly', 'drape': 'compiled.drape'}[compiled.kind]
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
    self.object_chars = ''      # characters of Drapes the program keeps as cells of one object
                                # grid instead of spec drapes (box_world); the curtain and
                                # layers hooks serve them
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
    self.rng_streams = ()       # the MT19937 streams the device continues, one RNG slot each
                                # in this order: NumPy's legacy RandomState ('numpy') or
                                # Python's `random` ('python')
    self.rng_from_globals = False  # the facade hands the global generators of rng_streams to
                                # the device and takes them back after every step (compiled,
                                # cued_catch)
    self.template_draws = None  # (program_arg index, bit) the facade sets when its Python
                                # constructors have drawn already: the device then takes those
                                # draws from the template at a start and draws only in steps
                                # (cued_catch); a batched engine leaves it clear and draws both
    self.actions_per_env = 1    # action words per env and step
    self.backdrop_chars = ''
    self.drape_kind = None      # per drape: 1 = Scrolly (fixture and compiled programs)
    self.dynamic_z = False      # per-env z-order array (Plot.change_z_order)
    self.program_arg = [0] * 8  # pcl_spec.program_arg
    self.reward_type = int      # the reference's reward type (classics pay floats)
    self.float_reward = False   # rewards are not integers: pcl_outputs.d_reward_f64
    self.backdrop_role = None   # device counterpart of a Backdrop with update() logic: 'river'
                                # (classics) or 'compiled.backdrop' (registered code)
    self.scroll_groups = ['']   # names of the scrolling groups, index = device group id
    self.sprite_group = []      # per sprite: index into scroll_groups
    self.drape_group = []       # per drape
    self.group_records = None   # i32 [MAX_SCROLL_GROUPS, 4] reset template (groups >= 1)
    # Host hooks of the program module (pycolab_b200/programs), None where it needs none:
    self.curtain = None         # (BatchedEngine, d) -> u8 [B, rows, pitch] curtain of drape d,
                                # or None where the device exports it (pcl_export_curtain)
    self.occlusion_in_layers = True   # False: layers are un-occluded (rendering.py:187-301)
    self.layers = None          # (BatchedEngine, chars) -> bool [B, len(chars), rows, cols]
    self.sync = None            # (Engine): mirror program-private device state into the
                                # Python objects after a step
    self.python_reward = None   # (Engine, value): the reference's reward of a step that has one,
                                # where its Python type varies by step (cued_catch: int or float)
    self.action_row = None      # (Engine, facade actions) -> the env's action words
    self.code = None            # i32 bytecode words (pcl_bind_code) of the compiled program
    self.registers = {}         # compiled: char -> [(attribute, type)] in register order, type
                                # the value's at lowering: bool, int, things.Sprite.Position
                                # or tuple (the last two: a position attribute, two registers)
    self.plot_keys = []         # compiled: [(the_plot key, is_bool)] in plot register order

  @property
  def needs_rng(self):
    return bool(self.rng_streams)

  def signature(self):
    """Everything that must agree between envs sharing one handle."""
    return (self.program, self.rows, self.cols, self.sprite_chars, self.drape_chars,
            tuple(map(tuple, self.impassable)), tuple(self.confined),
            tuple(self.egocentric), tuple(map(tuple, self.margins)), self.z_order,
            tuple(self.groups), self.pattern_rows, self.pattern_cols,
            tuple(self.program_arg), tuple(self.scroll_groups), tuple(self.sprite_group),
            tuple(self.drape_group), None if self.code is None else self.code.tobytes())

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


def _common(engine, game, program, never_reads_layers=False):
  game.program = program
  game.rows, game.cols = engine.rows, engine.cols
  game.pitch = round_up(engine.cols, 16)
  game.bits_words = (engine.cols + 31) // 32 + 1
  game.z_order = ''.join(engine.z_order)
  game.groups = [''.join(e.character for e in entities)
                 for _, entities in sorted(engine._update_groups.items())]
  backdrop = engine.backdrop
  game.backdrop_role = None
  from pycolab_b200 import compiler
  if compiler.registered(type(backdrop)) is not None:
    game.backdrop_role = 'compiled.backdrop'    # its code runs on the compiled program only
  elif type(backdrop).update is not things.Backdrop.update:
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
  if not engine._occlusion_in_layers and not never_reads_layers:
    raise NotLoweredError('occlusion_in_layers=False is lowered only for games whose '
                          'entities never consult `layers`')
  game.occlusion_in_layers = engine._occlusion_in_layers


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


def _drape_record(**aux):
  rec = [0] * _lib.DRAPE_WORDS
  rec[_lib.D_LAST_FRAME] = _lib.NEVER
  for name, value in aux.items():
    rec[getattr(_lib, 'D_' + name.upper())] = int(value)
  return rec


def _update_order(engine):
  return [e.character for _, ents in sorted(engine._update_groups.items()) for e in ents]


def lower(engine):
  """`Engine` (set-up finished, not yet showtime) -> `LoweredGame`."""
  from pycolab_b200 import programs
  roles = {ch: role_of(ent) for ch, ent in engine.things.items()}
  families = {role.split('.')[0] for role in roles.values()}
  if len(families) != 1:
    raise NotLoweredError('entities from different game programs: {}'.format(roles))
  family = families.pop()
  if family not in programs.BY_FAMILY:
    raise NotLoweredError(family)
  game = programs.BY_FAMILY[family].lower(engine, roles)
  if game.backdrop_role == 'compiled.backdrop' and family != 'compiled':
    raise NotLoweredError('a registered Backdrop is lowered only with registered entities')
  if game.backdrop_role not in (None, 'compiled.backdrop') and family != 'classics':
    raise NotLoweredError('a Backdrop with update() logic is lowered only with its own game')
  return game
