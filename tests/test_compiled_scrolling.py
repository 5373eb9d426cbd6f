"""CPU tests of scrolling games on the compiled step program: Scrollys and egocentric
MazeWalkers in registered update() code (`pycolab_b200.compiler`, csrc/compiled.cu).

  - the forms the compiler accepts for them and the ones it refuses, with the source line;
  - limits refused at lowering: registers, scrolling groups, pattern shapes;
  - the oracle interpreter (oracle/compiled.py) running the compiled maze of
    tests/scrolling_games.py reproduces the reference's scrolly_maze trajectories
    (tests/golden/scrolly_*.npz); the sampler's goldens replay in test_registered_goldens.py;
  - with the reference present, its own scrolly_maze classes compile unchanged;
  - pcl_bind_code / pcl_create checks of the new opcodes, on handles that reach no device.
"""

import ctypes as C
import os

import numpy as np
import pytest

import boundary_sweep
import example_games as eg
import golden_cases as gc
import refdriver
import registered_games as rg
import scrolly_shapes
from oracle import compiled as ocompiled
from pycolab_b200 import _lib, compiler, lowering
from pycolab_b200 import things as b_things
from pycolab_b200.errors import NotLoweredError
from pycolab_b200.prefab_parts import drapes as b_drapes
from pycolab_b200.prefab_parts import sprites as b_sprites

needs_ref = pytest.mark.skipif(not refdriver.available(), reason='/root/reference not present')


@pytest.fixture(scope='module')
def games():
  yield from rg.registered('scrolling_games.py')


def _margins(name):
  """The scroll margins a scrolly_* golden was made with."""
  if name.startswith('scrolly_shape'):
    return scrolly_shapes.SHAPE[name[len('scrolly_shape'):]][2]
  return scrolly_shapes.DEFAULT_MARGINS


def _no_error(world, out):
  assert world.error == 0


# ------------------------------------------------------------- the goldens --

@pytest.mark.parametrize('name', gc.names('scrolly_'))
def test_oracle_runs_compiled_maze_like_the_reference(games, name):
  g = gc.load(name)
  maze, board, beneath = gc.scrolly_art(g)
  lowered = lowering.lower(games.make_maze(maze, board, beneath, margins=_margins(name)))
  assert lowered.program == _lib.PROG_COMPILED
  assert list(lowered.drape_kind) == [1, 1] and lowered.program_arg[2] == 0b10
  eg.assert_replays('oracle', name, make_env=lambda: ocompiled.make_world(lowered),
                    check=_no_error)


def test_oracle_raises_on_postscroll_before_the_move(games):
  world = ocompiled.make_world(lowering.lower(games.make_early()))
  world.its_showtime()
  world.play(0)
  with pytest.raises(RuntimeError, match='postscroll'):
    world.play(1)


# ------------------------------------------------------------ the subset --

def test_maze_compiles_to_the_scrolly_opcodes(games):
  ops = lambda klass: {ins[0] for ins in compiler.registered(klass).ir}
  assert {'PRESCROLL', 'PATTERN', 'MOVE', 'EQ2', 'TERMINATE'} <= ops(games.MazePatroller)
  assert {'PRESCROLL', 'PATTERN', 'SETPAT', 'PATANY', 'SCROLL', 'REWARD'} <= ops(games.MazeCoins)
  assert ops(games.MazeWalls) == {'ACTION', 'PUSH', 'EQ', 'JZ', 'JMP', 'LABEL', 'SCROLL', 'RET'}
  assert compiler.registered(games.MazePatroller).attrs == ['heading_east']
  assert {'POSTSCROLL', 'SETPAT', 'SETP', 'SCROLL'} <= ops(games.Gems)
  assert {'CURTAIN', 'ANY'} <= ops(games.Watcher)


def test_roles_and_lowered_records(games):
  engine = games.make_sampler(0)
  assert lowering.role_of(engine.things['#']) == 'compiled.scrolly'
  assert lowering.role_of(engine.things['P']) == 'compiled.walker'
  lowered = lowering.lower(engine)
  assert lowered.drape_chars == '#*' and lowered.sprite_chars == 'Pe'
  assert lowered.egocentric == [True, False]
  assert lowered.margins == [(-1, -1), (2, 2)]
  assert lowered.program_arg[2] == 0b10 and lowered.pattern_mutable == {0: False, 1: True}
  assert lowered.pattern_words == lowering.round_up((20 + 31) // 32 + 3, 2)
  p = lowered.sprites[0]
  assert (p[_lib.S_AUX0], p[_lib.S_AUX1], p[_lib.S_AUX2]) == (0, _lib.NEVER, 0)
  walls = lowered.drapes[0]
  assert list(walls[:5]) == [2, 3, 2, 3, _lib.NEVER] and walls[_lib.D_AUX0] == 0
  assert 1 in lowered.bits and 0 not in lowered.bits     # the gems' curtain is kept in bits


def _scrolly(update, base=b_drapes.Scrolly):
  return type('Case', (base,), {'update': update, '__module__': __name__})


def _walker(update):
  return type('Case', (b_sprites.MazeWalker,), {'update': update, '__module__': __name__})


# Each refused construct on the marked line.
def _curtain_write(self, actions, board, layers, backdrop, things, the_plot):
  self.curtain[0, 0] = True                           # REFUSED


def _other_pattern_write(self, actions, board, layers, backdrop, things, the_plot):
  things['#'].whole_pattern[0, 0] = True              # REFUSED


def _pattern_slice(self, actions, board, layers, backdrop, things, the_plot):
  self.n = self.whole_pattern[0:2, 1]                 # REFUSED


def _corner_state(self, actions, board, layers, backdrop, things, the_plot):
  self._northwest_corner = (0, 0)                     # REFUSED


def _margin_state(self, actions, board, layers, backdrop, things, the_plot):
  self._margin_north = 1                              # REFUSED


def _walker_helper_form(self, actions, board, layers, backdrop, things, the_plot):
  self._north(board, the_plot)                        # REFUSED


def _log(self, actions, board, layers, backdrop, things, the_plot):
  the_plot.log('coin')                                # REFUSED


def _helper_value(self, actions, board, layers, backdrop, things, the_plot):
  self.n = self._north(the_plot) is None              # REFUSED


SCROLLY_REFUSED = [(_curtain_write, 'curtain write in a scrolly class'),
                   (_other_pattern_write, "another entity's whole_pattern"),
                   (_pattern_slice, 'whole_pattern slice'),
                   (_corner_state, '_northwest_corner'), (_margin_state, '_margin_north'),
                   (_walker_helper_form, 'not called as (the_plot)'),
                   (_log, 'the_plot.log()'), (_helper_value, '_north in a scrolly class')]


def _walker_pattern(self, actions, board, layers, backdrop, things, the_plot):
  self.n = self.whole_pattern[0, 0]                   # REFUSED


def _walker_prescroll(self, actions, board, layers, backdrop, things, the_plot):
  r, c = self.pattern_position_prescroll((0, 0), the_plot)   # REFUSED


def _unpack_three(self, actions, board, layers, backdrop, things, the_plot):
  r, c, d = self.position                             # REFUSED


def _unpack_number(self, actions, board, layers, backdrop, things, the_plot):
  r, c = self.n                                       # REFUSED


WALKER_REFUSED = [(_walker_pattern, 'self.whole_pattern in a sprite class'),
                  (_walker_prescroll, 'pattern_position_prescroll in a sprite class'),
                  (_unpack_three, 'two names'), (_unpack_number, 'not a position')]


@pytest.mark.parametrize('update,what,make', [(u, w, _scrolly) for u, w in SCROLLY_REFUSED] +
                         [(u, w, _walker) for u, w in WALKER_REFUSED],
                         ids=[u.__name__ for u, _ in SCROLLY_REFUSED + WALKER_REFUSED])
def test_refused_construct_names_class_line_and_construct(update, what, make):
  rg.assert_refused(make(update), what)


def test_plain_drapes_keep_refusing_motion_helpers_and_patterns():
  def move(self, actions, board, layers, backdrop, things, the_plot):
    self._north(the_plot)
  with pytest.raises(NotLoweredError, match='_north in a drape class'):
    compiler.compile_class(_scrolly(move, b_things.Drape))

  def pattern(self, actions, board, layers, backdrop, things, the_plot):
    self.n = self.whole_pattern.any()
  with pytest.raises(NotLoweredError, match='self.whole_pattern in a drape class'):
    compiler.compile_class(_scrolly(pattern, b_things.Drape))


def _accepted(self, actions, board, layers, backdrop, things, the_plot):
  pre = self.pattern_position_prescroll((1, -2), the_plot)
  (self._northwest if self.n else self._stay)(the_plot)
  r, c = self.pattern_position_postscroll(pre, the_plot)
  self.n = int(things['#'].whole_pattern[r, c]) + self.whole_pattern[-1, -1]
  self.whole_pattern[r, -c] = self.curtain[0, 0] or things['#'].curtain.any()
  if self.whole_pattern.any() and things['#'].whole_pattern.any():
    self.m = things['#'].pattern_position_prescroll((0, 0), the_plot)[1]


def test_accepted_scrolly_constructs_compile():
  comp = compiler.compile_class(_scrolly(_accepted))
  assert comp.kind == 'scrolly' and comp.attrs == ['n', 'm']
  ops = {ins[0] for ins in comp.ir}
  assert {'PRESCROLL', 'POSTSCROLL', 'SCROLL', 'PATTERN', 'SETPAT', 'PATANY', 'CURTAIN',
          'ANY'} <= ops


# --------------------------------------------------------- lowering limits --

def test_register_limits_are_refused_at_lowering(games):
  engine = games.make_sampler(0)
  engine.things['P'].extra = 1
  player = type(engine.things['P'])
  saved = player.update

  def update(self, actions, board, layers, backdrop, things, the_plot):
    self.steps = self.extra
  player.update = update
  compiler.register(player)
  try:
    with pytest.raises(NotLoweredError, match="'P' needs 2 registers; an egocentric walker has 1"):
      lowering.lower(engine)
  finally:
    player.update = saved
    compiler.register(player)


def test_groups_and_pattern_shapes_are_refused_at_lowering(games):
  engine = games.make_sampler(0)
  engine.things['*']._scrolling_group = 'other'
  with pytest.raises(NotLoweredError, match='more than one scrolling group'):
    lowering.lower(engine)
  engine = games.make_sampler(0)
  gems = engine.things['*']
  gems._w_h_o_l_e_p_a_t_t_e_r_n = np.zeros((13, 20), dtype=bool)
  with pytest.raises(NotLoweredError, match='different shapes'):
    lowering.lower(engine)


# ----------------------------------------------------------- the reference --

@needs_ref
def test_reference_scrolly_maze_classes_compile_and_match_golden(games):
  mod = rg.load(os.path.join(refdriver.REFERENCE_ROOT, 'pycolab', 'examples', 'scrolly_maze.py'))
  with pytest.raises(NotLoweredError, match=r'the_plot\.log\(\)'):
    compiler.compile_class(mod.CashDrape)
  ours = (mod.PlayerSprite, mod.PatrollerSprite, mod.MazeDrape)
  compiler.register(*ours)
  try:
    for name in gc.names('scrolly_stock_'):
      g = gc.load(name)
      maze, board, beneath = gc.scrolly_art(g)
      from pycolab_b200 import ascii_art
      info = b_drapes.Scrolly.PatternInfo(maze, board, board_northwest_corner_mark='+',
                                          what_lies_beneath=beneath)
      sprites = {'P': ascii_art.Partial(mod.PlayerSprite, info.virtual_position('P'))}
      for ch in 'abc':
        sprites[ch] = ascii_art.Partial(mod.PatrollerSprite, info.virtual_position(ch))
      engine = ascii_art.ascii_art_to_game(
          board, what_lies_beneath=' ', sprites=sprites,
          drapes={'#': ascii_art.Partial(mod.MazeDrape, **info.kwargs('#')),
                  '@': ascii_art.Partial(games.MazeCoins, **info.kwargs('@'))},
          update_schedule=[['#'], ['a', 'b', 'c', 'P'], ['@']], z_order='abc@#P')
      lowered = lowering.lower(engine)
      assert lowered.program == _lib.PROG_COMPILED
      eg.assert_replays('oracle', name, make_env=lambda: ocompiled.make_world(lowered))
  finally:
    compiler.unregister(*ours)


# ------------------------------------------------------------ pcl_bind_code --

def test_bind_code_checks_the_scrolly_opcodes(games):
  lib = _lib.load()
  lowered = lowering.lower(games.make_sampler(0))
  spec = lowered.make_spec(True)
  code = lowered.code.copy()
  op = lambda name: _lib.OP[name]
  h = rg.handle(lib, spec)
  try:
    assert rg.bind(lib, h, code) == _lib.OK
    fn = {ch: code[1 + i] for i, ch in enumerate(lowered.sprite_chars + lowered.drape_chars)}
    starts = sorted(set(fn.values())) + [len(code)]
    span = lambda ch: ocompiled.instructions(code, fn[ch], starts[starts.index(fn[ch]) + 1])
    find = lambda ch, name: [i for i in span(ch) if code[i] == op(name)][0]

    def mutated(at, value):
      c = code.copy()
      c[at] = value
      return c
    walls_scroll = find('#', 'SCROLL')
    gems_post = find('*', 'POSTSCROLL')
    player_move = find('P', 'MOVE')
    watcher_curtain = find('e', 'CURTAIN')
    cases = {
        'SCROLL in a walker': mutated(player_move, op('SCROLL')),
        'SCROLL motion out of range': mutated(walls_scroll + 1, 9),
        'SETPAT on a read-only pattern': mutated(find('#', 'SCROLL'), op('SETPAT')),
        'POSTSCROLL of a walker': mutated(gems_post + 1, 0),
        'POSTSCROLL past the entities': mutated(gems_post + 1, 9),
        'PATTERN of self in a walker': mutated(watcher_curtain, op('PATTERN')),
        'egocentric register 1': mutated(find('P', 'GETR') + 1, 1),
        'Scrolly register 3': mutated(find('*', 'GETR') + 1, 3),
    }
    cases['PATTERN of self in a walker'][watcher_curtain + 1] = -1
    for label, words in cases.items():
      assert rg.bind(lib, h, words) == _lib.ERR_INVALID, label
  finally:
    lib.pcl_destroy(h)


def test_create_checks_written_patterns(games):
  lib = _lib.load()
  lowered = lowering.lower(games.make_sampler(0))
  for bits, want in ((0b10, _lib.OK), (0b01 | 0b10, _lib.OK), (0b100, _lib.ERR_INVALID),
                     (-2 ** 31, _lib.ERR_INVALID)):
    spec = lowered.make_spec(True)
    spec.program_arg[2] = bits
    h = C.c_void_p()
    assert lib.pcl_create(C.byref(spec), 4, -1, C.byref(h)) == want, bits
    if want == _lib.OK:
      lib.pcl_destroy(h)
  # a plain drape may not be marked
  spec = lowered.make_spec(True)
  spec.drape_kind[1] = 0
  spec.program_arg[2] = 0b10
  h = C.c_void_p()
  assert lib.pcl_create(C.byref(spec), 4, -1, C.byref(h)) == _lib.ERR_INVALID


def test_bind_state_needs_the_written_pattern_template(games):
  lib = _lib.load()
  spec = lowering.lower(games.make_sampler(0)).make_spec(True)
  h = rg.handle(lib, spec)
  try:
    st = boundary_sweep._full_state()
    for d in range(2):
      st.d_pattern[d] = boundary_sweep.FAKE
      st.pattern_bstride[d] = 64
    st.d_pattern_init[1] = boundary_sweep.FAKE
    assert lib.pcl_bind_state(h, C.byref(st)) == _lib.OK
    st.d_pattern_init[1] = None
    assert lib.pcl_bind_state(h, C.byref(st)) == _lib.ERR_INVALID
    st.d_pattern_init[1] = boundary_sweep.FAKE
    st.d_pattern[0] = None
    assert lib.pcl_bind_state(h, C.byref(st)) == _lib.ERR_INVALID
  finally:
    lib.pcl_destroy(h)
