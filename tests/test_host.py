"""CPU tests of the host side: C-ABI library surface, facade set-up API,
lowering, compat loading of the reference's example modules."""

import os
import sys
import re

import numpy as np
import pytest

import golden_cases as gc
import refdriver
import trajectory as tj
from oracle import games as ogames
from pycolab_b200 import _lib
from pycolab_b200 import ascii_art
from pycolab_b200 import engine as engine_mod
from pycolab_b200 import levels
from pycolab_b200 import lowering
from pycolab_b200 import things
from pycolab_b200.errors import DeviceOnlyError, NotLoweredError
from pycolab_b200.games import extraterrestrial_marauders as g_marauders
from pycolab_b200.games import scrolly_maze as g_scrolly
from pycolab_b200.games import shockwave as g_shockwave
from pycolab_b200.games import warehouse_manager as g_warehouse
from pycolab_b200.prefab_parts import sprites as prefab_sprites

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ------------------------------------------------------------ C-ABI library

def _header_functions():
  text = open(os.path.join(ROOT, 'include', 'pcl.h')).read()
  text = re.sub(r'/\*.*?\*/', '', text, flags=re.S)
  return sorted(set(re.findall(r'\b(pcl_[a-z_]+)\s*\(', text)))


def test_library_exports_every_declared_symbol():
  import ctypes
  assert os.path.exists(_lib.LIB_PATH), 'build libpcl.so first (__graft_entry__.build)'
  lib = ctypes.CDLL(_lib.LIB_PATH)
  declared = _header_functions()
  assert len(declared) >= 14
  for name in declared:
    assert hasattr(lib, name), name
  assert sorted(_lib.SYMBOLS) == declared


def test_binding_loads_and_reports_abi():
  lib = _lib.load()
  assert lib.pcl_abi_version() == _lib.ABI_VERSION
  assert _lib.status_string(_lib.ERR_UNSUPPORTED) == 'game not lowered to a device program'


def test_binding_structs_match_the_header():
  """The library reports sizeof() of every struct that crosses the boundary;
  `_lib.load()` refuses a binding whose ctypes layouts disagree."""
  import ctypes as C
  lib = _lib.load()
  sizes = (C.c_int32 * 4)()
  assert lib.pcl_struct_sizes(sizes) == _lib.OK
  assert list(sizes) == [C.sizeof(_lib.Spec), C.sizeof(_lib.State), C.sizeof(_lib.Outputs),
                         C.sizeof(_lib.CropSpec)]


def test_create_rejects_bad_specs_without_gpu():
  import ctypes as C
  lib = _lib.load()
  h = C.c_void_p()
  spec = _lib.Spec()
  assert lib.pcl_create(C.byref(spec), 4, -1, C.byref(h)) == _lib.ERR_INVALID  # abi 0
  spec.abi_version = _lib.ABI_VERSION
  spec.rows, spec.cols, spec.pitch = 10, 30, 30                              # pitch % 16
  assert lib.pcl_create(C.byref(spec), 4, -1, C.byref(h)) == _lib.ERR_INVALID
  spec.pitch = 32
  spec.program = 99
  assert lib.pcl_create(C.byref(spec), 4, -1, C.byref(h)) == _lib.ERR_UNSUPPORTED
  spec.program = _lib.PROG_NONE
  assert lib.pcl_create(C.byref(spec), 4, -1, C.byref(h)) == _lib.OK
  out = _lib.Outputs()
  assert lib.pcl_step(h, None, C.byref(out), None) == _lib.ERR_UNBOUND
  assert lib.pcl_destroy(h) == _lib.OK


def _create(spec, batch=4):
  import ctypes as C
  lib = _lib.load()
  h = C.c_void_p()
  status = lib.pcl_create(C.byref(spec), batch, -1, C.byref(h))   # device -1: no CUDA call
  if status == _lib.OK:
    lib.pcl_destroy(h)
  return status


def test_every_lowered_game_passes_create_validation_without_gpu():
  """lowering -> pcl_spec -> pcl_create's validation, for one level of every
  device program (no GPU needed: device = -1 skips cudaSetDevice)."""
  import importlib
  import golden_cases as gc
  import trajectory as tj
  from pycolab_b200.games import aperture, better_scrolly_maze, fluvial_natation
  games = [g_scrolly.make_game(*levels.scrolly_maze_level(0, world_shape=(33, 33),
                                                          board_shape=(16, 16))),
           g_warehouse.make_game(levels.warehouse_level(1), ' '),
           g_marauders.make_game(levels.marauders_level()),
           better_scrolly_maze.make_game(tj.u8_to_art(gc.load('better_stock_L0')['art'])),
           fluvial_natation.make_game(), aperture.make_game(levels.aperture_level())]
  for kind in ('four_rooms', 'cliff_walk', 'chain_walk'):
    mod = importlib.import_module('pycolab_b200.games.classics.' + kind)
    games += [mod.make_game(), mod.make_game(levels.classic_level(kind))]
  programs = set()
  for game in games:
    lowered = lowering.lower(game)
    programs.add(lowered.program)
    assert _create(lowered.make_spec(auto_reset=True)) == _lib.OK, lowered.program
  assert programs == {_lib.PROG_SCROLLY_MAZE, _lib.PROG_WAREHOUSE, _lib.PROG_MARAUDERS,
                      _lib.PROG_BETTER_SCROLLY, _lib.PROG_CLASSICS, _lib.PROG_APERTURE}


def test_create_rejects_malformed_specs_of_the_newer_programs():
  from pycolab_b200.games import aperture, fluvial_natation
  from pycolab_b200.games.classics import four_rooms
  spec = lowering.lower(four_rooms.make_game()).make_spec(True)
  spec.program_arg[0] = 9                                   # unknown rule set
  assert _create(spec) == _lib.ERR_INVALID
  spec = lowering.lower(fluvial_natation.make_game()).make_spec(True)
  spec.impassable[0][1] = 1 << 3                            # a swimmer that reads the board ('#')
  assert _create(spec) == _lib.ERR_UNSUPPORTED
  spec = lowering.lower(aperture.make_game(levels.aperture_level())).make_spec(True)
  spec.z_order[0], spec.z_order[1] = spec.z_order[1], spec.z_order[0]   # player under the drape
  assert _create(spec) == _lib.ERR_UNSUPPORTED
  spec = lowering.lower(aperture.make_game(levels.aperture_level())).make_spec(True)
  spec.n_groups, spec.group_len[0], spec.group_len[1] = 1, 2, 0         # one update group
  assert _create(spec) == _lib.ERR_UNSUPPORTED
  spec = lowering.lower(four_rooms.make_game()).make_spec(True)
  assert _create(spec, batch=0) == _lib.ERR_INVALID


def test_missing_library_fails_loudly(monkeypatch):
  monkeypatch.setattr(_lib, '_lib', None)
  monkeypatch.setattr(_lib, 'LIB_PATH', '/nonexistent/libpcl.so')
  with pytest.raises(_lib.PclLibraryError):
    _lib.load()


def test_no_cpu_path():
  import torch
  if torch.cuda.is_available():
    pytest.skip('GPU present')
  from pycolab_b200 import batched
  art = levels.scrolly_maze_level(0, world_shape=(33, 33), board_shape=(16, 16))
  with pytest.raises(_lib.PclLibraryError):
    batched.BatchedEngine([g_scrolly.make_game(*art)], batch=2)
  with pytest.raises(_lib.PclLibraryError):
    g_scrolly.make_game(*art).its_showtime()


# ----------------------------------------------------------------- lowering

def test_pack_rows_round_trip():
  rs = np.random.RandomState(0)
  for cols in (1, 31, 32, 33, 64, 89, 129):
    mask = rs.random_sample((7, cols)) < 0.4
    words = (cols + 31) // 32 + 1
    packed = lowering.pack_rows(mask, words)
    assert packed.shape == (7, words) and packed.dtype == np.uint32
    np.testing.assert_array_equal(lowering.unpack_rows(packed, cols), mask)
    assert not packed[:, -1].any()
    c = cols - 1
    assert bool((packed[3, c >> 5] >> (c & 31)) & 1) == bool(mask[3, c])


def _check_sprites(game, world, chars):
  for i, ch in enumerate(chars):
    w, rec = world.things[ch], game.sprites[i]
    assert tuple(rec[:4]) == (w.row, w.col, w.vrow, w.vcol), ch
    assert bool(rec[_lib.S_FLAGS] & 1) == bool(w.visible), ch
    prior = (rec[_lib.S_FLAGS] >> 1) & 3
    assert {0: None, 1: False, 2: True}[prior] == w.prior_visible, ch


@pytest.mark.parametrize('name', ['scrolly_stock_L0', 'scrolly_stock_L2', 'scrolly_gen64_s0'])
def test_lower_scrolly_matches_oracle_initial_state(name):
  g = gc.load(name)
  maze, board, beneath = gc.scrolly_art(g)
  game = lowering.lower(g_scrolly.make_game(maze, board, beneath))
  world = ogames.make_scrolly_maze(maze, board, '+', beneath)
  assert game.program == _lib.PROG_SCROLLY_MAZE
  assert (game.rows, game.cols) == (world.rows, world.cols)
  assert game.pitch % 16 == 0 and game.pitch >= game.cols
  assert game.sprite_chars == 'Pabc' and game.drape_chars == '#@'
  assert game.z_order == 'abc@#P' and game.groups == ['#', 'abcP', '@']
  _check_sprites(game, world, 'Pabc')
  for d, ch in enumerate('#@'):
    np.testing.assert_array_equal(
        lowering.unpack_rows(game.patterns[d], game.pattern_cols), world.things[ch].pattern)
    assert tuple(game.drapes[d][:2]) == world.things[ch].corner
    assert game.margins[d] == (2, 3)
  assert game.plot[_lib.P_AUX0] == world.things['@'].pattern.sum()
  assert game.plot[_lib.P_FRAME] == -1
  np.testing.assert_array_equal(game.backdrop[:, :game.cols], world.backdrop)
  assert [int(game.sprites[i][_lib.S_AUX0]) for i in (1, 2, 3)] == [
      int(world.things[c].aux['moving_east']) for c in 'abc']
  assert game.egocentric == [True, False, False, False]


@pytest.mark.parametrize('name', ['warehouse_stock_L0', 'warehouse_stock_L1',
                                  'warehouse_gen80_s3'])
def test_lower_warehouse_matches_oracle_initial_state(name):
  g = gc.load(name)
  art, wlb = gc.warehouse_art(g)
  game = lowering.lower(g_warehouse.make_game(art, wlb))
  world = ogames.make_warehouse(art, wlb)
  chars = bytes(g['sprite_chars']).decode()
  assert game.program == _lib.PROG_WAREHOUSE and game.sprite_chars == chars
  _check_sprites(game, world, chars)
  np.testing.assert_array_equal(game.backdrop[:, :game.cols], world.backdrop)
  for i, ch in enumerate(chars):
    want = lowering.char_set_mask(chr(c) for c in world.things[ch].impassable)
    assert game.impassable[i] == want


def test_lower_marauders_matches_oracle_initial_state():
  art = levels.marauders_level()
  game = lowering.lower(g_marauders.make_game(art))
  world = ogames.make_marauders(art, np.random.RandomState(0))
  assert game.program == _lib.PROG_MARAUDERS and game.needs_rng
  _check_sprites(game, world, 'Pabcdyz')
  for d, ch in enumerate('BX'):
    np.testing.assert_array_equal(lowering.unpack_rows(game.bits[d], game.cols),
                                  world.things[ch].curtain)
  assert game.drapes[1][_lib.D_AUX0] == -1
  assert game.confined == [True] + [False] * 6
  # bolts start hidden off-board with their visibility stashed (sprites.py:223-249)
  assert all(game.sprites[i][_lib.S_FLAGS] == 4 for i in range(1, 7))


def test_unknown_entity_class_is_refused():
  class Wanderer(prefab_sprites.MazeWalker):
    def __init__(self, corner, position, character):
      super(Wanderer, self).__init__(corner, position, character, impassable='#')

    def update(self, actions, board, layers, backdrop, things, the_plot):
      self._north(board, the_plot)

  game = ascii_art.ascii_art_to_game(['#####', '# w #', '#####'], ' ', {'w': Wanderer})
  with pytest.raises(NotLoweredError):
    lowering.lower(game)
  with pytest.raises(NotLoweredError):
    game.its_showtime()
  with pytest.raises(DeviceOnlyError):
    game.things['w']._north(None, None)


def test_overriding_update_of_a_lowered_class_is_refused():
  class Cheater(g_scrolly.PlayerSprite):
    def update(self, actions, board, layers, backdrop, things, the_plot):
      pass
  assert lowering.role_of.__name__ == 'role_of'
  corner = things.Sprite.Position(5, 5)
  with pytest.raises(NotLoweredError):
    lowering.role_of(Cheater(corner, things.Sprite.Position(1, 1), 'P', (1, 1)))


# ----------------------------------------------- facade set-up API behaviour

def test_engine_setup_errors_match_reference_contract():
  eng = engine_mod.Engine(3, 4)
  with pytest.raises(TypeError):
    eng.add_sprite('a', (0, 0), object)
  with pytest.raises(ValueError):
    eng.add_sprite('a', (5, 0), g_warehouse.PlayerSprite)
  eng.add_sprite('a', (1, 1), g_warehouse.PlayerSprite)
  with pytest.raises(RuntimeError):
    eng.add_sprite('a', (1, 2), g_warehouse.PlayerSprite)
  with pytest.raises(ValueError):
    eng.add_sprite('ab', (1, 2), g_warehouse.PlayerSprite)
  with pytest.raises(ValueError):
    eng.set_z_order('ab')
  with pytest.raises(RuntimeError):
    eng.play(0)
  eng.set_prefilled_backdrop(' #', np.full((3, 4), 32, np.uint8), things.Backdrop)
  with pytest.raises(RuntimeError):
    eng.set_backdrop(' ', things.Backdrop)
  assert eng.backdrop.palette.hash == ord('#')
  assert eng.backdrop.palette[' '] == 32
  with pytest.raises(AttributeError):
    eng.backdrop.palette.at


def test_ascii_art_errors():
  with pytest.raises(TypeError):
    ascii_art.ascii_art_to_uint8_nparray([['a', 'b'], ['c', 'd']])
  with pytest.raises(ValueError):
    ascii_art.ascii_art_to_uint8_nparray(['ab', 'c'])
  with pytest.raises(ValueError):
    ascii_art.ascii_art_to_game(['P '], ' ', {'P': g_warehouse.PlayerSprite},
                                update_schedule=[['Q']])
  with pytest.raises(ValueError):
    ascii_art.ascii_art_to_game(['PP'], ' ', {'P': g_warehouse.PlayerSprite})
  with pytest.raises(TypeError):
    ascii_art.Partial(int)


def test_maze_walker_constructor_contract():
  corner = things.Sprite.Position(4, 4)
  class Plain(prefab_sprites.MazeWalker):
    def update(self, *args):
      pass
  with pytest.raises(ValueError):
    Plain(corner, things.Sprite.Position(0, 0), 'x', 'x#')
  with pytest.raises(TypeError):
    Plain(corner, things.Sprite.Position(0, 0), 'x', [1, 2])
  bolt = g_marauders.UpwardLaserBoltSprite(corner, things.Sprite.Position(2, 2), 'a')
  assert bolt.position == (0, 0) and not bolt.visible and not bolt.on_the_board
  assert bolt.virtual_position == (-1, -1) and bolt._prior_visible is True
  bolt._teleport((3, 1))
  assert bolt.position == (3, 1) and bolt.visible


# --------------------------------- the reference's own example files, unchanged

needs_ref = pytest.mark.skipif(not refdriver.available(),
                               reason='/root/reference not present')


@pytest.fixture
def compat_examples():
  import sys
  from pycolab_b200 import compat
  saved = {k: v for k, v in sys.modules.items()
           if k == 'pycolab' or k.startswith('pycolab.')}
  compat.uninstall()
  compat.install()
  base = os.path.join(refdriver.REFERENCE_ROOT, 'pycolab', 'examples')
  yield lambda name: compat.load_example(os.path.join(base, name + '.py'))
  compat.uninstall()
  sys.modules.update(saved)


def _same_lowering(a, b):
  assert a.signature() == b.signature()
  for name in ('backdrop', 'sprites', 'drapes', 'plot'):
    np.testing.assert_array_equal(getattr(a, name), getattr(b, name), err_msg=name)
  for d in a.patterns:
    np.testing.assert_array_equal(a.patterns[d], b.patterns[d])
  for d in a.bits:
    np.testing.assert_array_equal(a.bits[d], b.bits[d])


@needs_ref
def test_reference_scrolly_maze_example_loads_and_lowers(compat_examples):
  mod = compat_examples('scrolly_maze')
  assert mod.PlayerSprite.__mro__[1] is prefab_sprites.MazeWalker
  for level in (0, 1, 2):
    theirs = lowering.lower(mod.make_game(level))
    ours = lowering.lower(g_scrolly.make_game(
        mod.MAZES_ART[level], mod.STAR_ART, mod.MAZES_WHAT_LIES_BENEATH[level]))
    _same_lowering(theirs, ours)


@needs_ref
def test_edited_copy_of_an_example_is_refused_not_replaced(compat_examples, tmp_path):
  """A user's copy of scrolly_maze.py lowers while it is token-for-token the
  reference's; with an edited update() (reward 7 instead of 100) the class is
  named like a lowered class but is NOT that class: NotLoweredError, never the
  stock kernel (lowering._is_known_implementation)."""
  from pycolab_b200 import compat
  from pycolab_b200.errors import NotLoweredError
  src = open(os.path.join(refdriver.REFERENCE_ROOT, 'pycolab', 'examples',
                          'scrolly_maze.py')).read()
  same = tmp_path / 'same' / 'scrolly_maze.py'
  same.parent.mkdir()
  same.write_text('# my copy\n' + src.replace('\n\n', '\n\n\n', 1))   # comments/blank lines only
  lowering.lower(compat.load_example(str(same)).make_game(0))
  assert 'the_plot.add_reward(100)' in src
  edited = tmp_path / 'edited' / 'scrolly_maze.py'
  edited.parent.mkdir()
  edited.write_text(src.replace('the_plot.add_reward(100)', 'the_plot.add_reward(7)'))
  with pytest.raises(NotLoweredError, match='source differs'):
    lowering.lower(compat.load_example(str(edited)).make_game(0))


@needs_ref
def test_reference_warehouse_example_loads_and_lowers(compat_examples):
  mod = compat_examples('warehouse_manager')
  for level in (0, 1, 2):
    theirs = lowering.lower(mod.make_game(level))
    ours = lowering.lower(g_warehouse.make_game(
        mod.WAREHOUSES_ART[level], mod.WAREHOUSES_WHAT_LIES_BENEATH[level]))
    _same_lowering(theirs, ours)


@needs_ref
def test_reference_marauders_example_loads_and_lowers(compat_examples):
  mod = compat_examples('extraterrestrial_marauders')
  _same_lowering(lowering.lower(mod.make_game()),
                 lowering.lower(g_marauders.make_game(levels.marauders_level())))


@needs_ref
def test_reference_example_outside_the_lowered_set_is_refused(compat_examples):
  # every other example now has a device program; tennis stays out of scope (SURVEY §2)
  mod = compat_examples('tennnnnnnnnnnnnnnnnnnnnnnnis')
  with pytest.raises(NotLoweredError):
    lowering.lower(mod.make_game())


@needs_ref
def test_reference_better_scrolly_example_loads_and_lowers(compat_examples):
  from pycolab_b200.games import better_scrolly_maze as g_better
  mod = compat_examples('better_scrolly_maze')
  for level in (0, 1, 2):
    theirs = lowering.lower(mod.make_game(level))
    ours = lowering.lower(g_better.make_game(mod.MAZES_ART[level]))
    assert theirs.program == _lib.PROG_BETTER_SCROLLY
    _same_lowering(theirs, ours)
  # the example's own croppers are this package's classes
  views = mod.make_croppers(0)
  assert [type(v).__name__ for v in views] == ['ScrollingCropper', 'ScrollingCropper',
                                               'FixedCropper']


@needs_ref
@pytest.mark.parametrize('kind', ['four_rooms', 'cliff_walk', 'chain_walk'])
def test_reference_classics_examples_load_and_lower(compat_examples, kind):
  import importlib
  from oracle import games as ogames
  mod = compat_examples(os.path.join('classics', kind))
  ours_mod = importlib.import_module('pycolab_b200.games.classics.' + kind)
  assert list(mod.GAME_ART) == list(ours_mod.GAME_ART)
  theirs, ours = lowering.lower(mod.make_game()), lowering.lower(ours_mod.make_game())
  assert theirs.program == _lib.PROG_CLASSICS and theirs.reward_type is float
  _same_lowering(theirs, ours)
  # ... and the lowered initial state is the oracle's
  world = ogames.make_classic(kind, list(mod.GAME_ART))
  w = world.things['P']
  assert tuple(theirs.sprites[0, :5]) == (w.row, w.col, w.vrow, w.vcol, 1)
  np.testing.assert_array_equal(theirs.backdrop[:, :theirs.cols], world.backdrop)
  assert bool(theirs.confined[0]) == w.confined


@needs_ref
def test_reference_aperture_example_loads_and_lowers(compat_examples):
  from pycolab_b200.games import aperture as ours_mod
  mod = compat_examples('aperture')
  for level in (0, 1, 2):
    theirs = lowering.lower(mod.make_game(level))
    ours = lowering.lower(ours_mod.make_game(mod.LEVELS[level]))
    assert theirs.program == _lib.PROG_APERTURE
    assert list(theirs.drapes[0, [_lib.D_AUX0, _lib.D_AUX1]]) == [-1, -1]
    _same_lowering(theirs, ours)


@needs_ref
def test_reference_fluvial_natation_loads_and_lowers(compat_examples):
  """A Backdrop subclass with update() logic is lowered with its own game only."""
  from pycolab_b200.games import fluvial_natation as ours_mod
  mod = compat_examples('fluvial_natation')
  theirs, ours = lowering.lower(mod.make_game()), lowering.lower(ours_mod.make_game())
  assert theirs.program == _lib.PROG_CLASSICS and theirs.backdrop_role == 'river'
  assert list(theirs.program_arg[:3]) == [_lib.CLASSIC_FLUVIAL, 1, 4] and theirs.reward_type is int
  _same_lowering(theirs, ours)
  # the river under another game's entities is refused, and so is an unknown Backdrop
  aa = sys.modules['pycolab.ascii_art']
  four_rooms = compat_examples(os.path.join('classics', 'four_rooms'))
  with pytest.raises(NotLoweredError):
    lowering.lower(aa.ascii_art_to_game(four_rooms.GAME_ART, ' ',
                                        sprites={'P': four_rooms.PlayerSprite},
                                        backdrop=mod.RiverBackdrop))

  class Odd(mod.RiverBackdrop):
    def update(self, *args, **kwargs):
      pass
  with pytest.raises(NotLoweredError):
    lowering.lower(aa.ascii_art_to_game(mod.GAME_ART, ' ', sprites={'P': mod.PlayerSprite},
                                        backdrop=Odd))


@needs_ref
def test_reference_host_only_unit_tests_pass_against_this_package(compat_examples):
  """The reference's own unit tests that need no step — ascii_art_test.py and
  scrolling_test.py::testProtocol (the scrolling-protocol helpers incl. their
  error messages) — run UNMODIFIED with `pycolab` aliased to this package."""
  import importlib.util
  import types
  import unittest
  base = os.path.join(refdriver.REFERENCE_ROOT, 'pycolab', 'tests')
  package = sys.modules.setdefault('pycolab.tests', types.ModuleType('pycolab.tests'))

  def load(name):
    spec = importlib.util.spec_from_file_location('pycolab.tests.' + name,
                                                  os.path.join(base, name + '.py'))
    module = importlib.util.module_from_spec(spec)
    sys.modules[spec.name] = module
    setattr(package, name, module)
    spec.loader.exec_module(module)
    return module
  load('test_things')
  suite = unittest.TestSuite()
  suite.addTests(unittest.defaultTestLoader.loadTestsFromModule(load('ascii_art_test')))
  suite.addTest(load('scrolling_test').ScrollingTest('testProtocol'))
  result = unittest.TextTestRunner(verbosity=0).run(suite)
  assert result.testsRun == 2 and result.wasSuccessful(), result.failures + result.errors


@needs_ref
def test_reference_test_fixtures_load_and_lower(compat_examples):
  """The reference's own tests/test_things.py fixtures lower to the general
  device program, identically to this package's games/fixtures.py."""
  import sys
  from pycolab_b200 import compat
  from pycolab_b200.games import fixtures
  tt = compat.load_example(os.path.join(refdriver.REFERENCE_ROOT, 'pycolab', 'tests',
                                        'test_things.py'))
  g = gc.load('fixture_scrolly_0')
  kw, cfg = gc.fixture_kwargs(g)
  aa = sys.modules['pycolab.ascii_art']
  shape = (len(kw['art']), len(kw['art'][0]))
  sprites = {ch: aa.Partial(tt.TestMazeWalker, impassable=w.get('impassable', ''),
                            confined_to_board=w.get('confined', False),
                            egocentric_scroller=w.get('egocentric', False))
             for ch, w in kw['walkers'].items()}
  drapes = {ch: aa.Partial(tt.TestScrolly, board_shape=shape, whole_pattern=s['pattern'],
                           board_northwest_corner=s['corner'], scroll_margins=s['margins'])
            for ch, s in kw['scrollys'].items()}
  theirs = aa.ascii_art_to_game(kw['art'], ' ', sprites, drapes,
                                update_schedule=kw['update_schedule'],
                                z_order=kw['z_order'])
  ours = fixtures.make_game(kw['art'], ' ', kw['walkers'], kw['scrollys'], '',
                            kw['update_schedule'], kw['z_order'])
  a, b = lowering.lower(theirs), lowering.lower(ours)
  assert a.program == _lib.PROG_FIXTURE and a.dynamic_z
  assert a.drape_kind == [1, 1] and a.egocentric == b.egocentric
  _same_lowering(a, b)


@pytest.mark.parametrize('call', [lambda p: p.add_reward(1), lambda p: p.terminate_episode(),
                                  lambda p: p.change_default_discount(0.5),
                                  lambda p: p.change_z_order('P', None)])
def test_plot_directives_before_showtime_are_refused(call):
  """engine.py:761-847 folds whatever the Plot holds into frame 0; the device's frame 0
  starts from clean directives, so the facade refuses instead of dropping them."""
  art = levels.scrolly_maze_level(3, world_shape=(33, 33), board_shape=(16, 16))
  game = g_scrolly.make_game(*art)
  call(game.the_plot)
  with pytest.raises(NotLoweredError, match='before its_showtime'):
    game.its_showtime()


def _bound_handle(game, batch=4):
  """A handle created and BOUND on the CPU: pcl_bind_state only records pointers, so
  made-up non-null addresses are enough to reach the argument checks of the entry
  points behind it (nothing is launched)."""
  import ctypes as C
  lib = _lib.load()
  handle = C.c_void_p()
  spec = game.make_spec(True)
  assert lib.pcl_create(C.byref(spec), batch, -1, C.byref(handle)) == _lib.OK
  st = _lib.State()
  fake = 0x10000
  for name in ('d_backdrop', 'd_sprites', 'd_sprites_init', 'd_drapes', 'd_drapes_init',
               'd_plot', 'd_plot_init'):
    setattr(st, name, fake)
  for d in range(2):
    st.d_pattern[d], st.d_pattern_init[d] = fake, fake
    st.pattern_bstride[d], st.pattern_init_bstride[d] = 64, 64
  # What shockwave requires: drape 0's live bits and every drape's reset bits.
  st.d_bits[0], st.bits_bstride[0], st.d_rng = fake, 64, fake
  for d in range(3):
    st.d_bits_init[d] = fake
  assert lib.pcl_bind_state(handle, C.byref(st)) == _lib.OK
  return lib, handle


def test_attach_cropper_argument_checks_on_cpu():
  """pcl_attach_cropper: unbound handle, bad window, drape tracking, programs without
  the epilogue, detach — all decided before anything touches the device."""
  import ctypes as C
  from pycolab_b200 import batched
  art = levels.scrolly_maze_level(3, world_shape=(33, 33), board_shape=(16, 16))
  game = lowering.lower(g_scrolly.make_game(*art))
  lib = _lib.load()
  raw = C.c_void_p()
  spec0 = game.make_spec(True)
  assert lib.pcl_create(C.byref(spec0), 4, -1, C.byref(raw)) == _lib.OK
  crop = batched.scrolling_crop_spec(5, 5, 0, pad_char=' ', scroll_margins=(None, None))
  assert lib.pcl_attach_cropper(raw, C.byref(crop), 0x20000, 0x30000) == _lib.ERR_UNBOUND
  lib.pcl_destroy(raw)

  lib, h = _bound_handle(game)
  assert lib.pcl_attach_cropper(h, C.byref(crop), 0x20000, 0x30000) == _lib.OK
  assert lib.pcl_attach_cropper(h, C.byref(crop), None, 0x30000) == _lib.ERR_INVALID
  assert lib.pcl_attach_cropper(h, None, None, None) == _lib.OK              # detach
  too_big = batched.scrolling_crop_spec(31, 31, 0, pad_char=None, scroll_margins=(2, 3))
  assert lib.pcl_attach_cropper(h, C.byref(too_big), 0x20000, 0x30000) == _lib.ERR_INVALID
  drape = batched.scrolling_crop_spec(5, 5, 0, pad_char=' ', scroll_margins=(None, None),
                                      track=[-1, 1])
  assert lib.pcl_attach_cropper(h, C.byref(drape), 0x20000, 0x30000) == _lib.ERR_UNSUPPORTED
  no_such = batched.scrolling_crop_spec(5, 5, 0, pad_char=' ', scroll_margins=(None, None),
                                        track=[9])
  assert lib.pcl_attach_cropper(h, C.byref(no_such), 0x20000, 0x30000) == _lib.ERR_INVALID
  lib.pcl_destroy(h)

  other = lowering.lower(g_warehouse.make_game(levels.warehouse_level(1, shape=(20, 24))))
  lib, h = _bound_handle(other)
  crop = batched.scrolling_crop_spec(5, 5, 0, pad_char=' ', scroll_margins=(None, None))
  assert lib.pcl_attach_cropper(h, C.byref(crop), 0x20000, 0x30000) == _lib.ERR_UNSUPPORTED
  lib.pcl_destroy(h)


@pytest.mark.parametrize('game, call, arg, want', [
    ('scrolly', 'attach', [-1, 1], _lib.ERR_UNSUPPORTED),       # drape medians need scratch
    ('scrolly', 'attach', [9], _lib.ERR_INVALID),
    ('scrolly', 'attach', [1, 9], _lib.ERR_INVALID),
    ('scrolly', 'tracking', [9], _lib.ERR_INVALID),
    ('scrolly', 'tracking', [1, 9], _lib.ERR_INVALID),
    ('scrolly', 'handoff', [9], _lib.ERR_INVALID),
    ('scrolly', 'handoff', [1, 9], _lib.ERR_INVALID),           # sprite 8 of a 4-sprite env
    ('scrolly', 'handoff', [-1, 1], _lib.ERR_UNSUPPORTED),
    ('scrolly', 'export', 2, _lib.ERR_INVALID),                 # only drapes 0 and 1
    ('shockwave', 'export', 1, _lib.ERR_INVALID),               # its bits were never bound
    ('warehouse', 'export', 0, _lib.ERR_UNSUPPORTED),           # 'X' is implicit in the boxes
    ('warehouse', 'layers', b'X', _lib.ERR_UNSUPPORTED),
])
def test_cropper_and_curtain_argument_checks_on_cpu(game, call, arg, want):
  """Every cropper entry point refuses a tracking list naming no sprite, and those without
  drape tracking refuse drapes; pcl_export_curtain and pcl_layers refuse a drape that is
  out of range, implicit, or not in the bound state — all before anything is launched."""
  import ctypes as C
  from pycolab_b200 import batched
  if game == 'scrolly':
    art = levels.scrolly_maze_level(3, world_shape=(33, 33), board_shape=(16, 16))
    lib, h = _bound_handle(lowering.lower(g_scrolly.make_game(*art)))
  elif game == 'shockwave':
    lib, h = _bound_handle(lowering.lower(g_shockwave.make_game(0)))
  else:
    lib, h = _bound_handle(lowering.lower(
        g_warehouse.make_game(levels.warehouse_level(1, shape=(20, 24)))))
  if call in ('attach', 'tracking', 'handoff'):
    crop = batched.scrolling_crop_spec(9, 9, 0, pad_char=' ', scroll_margins=(None, None),
                                       track=arg)
  if call == 'attach':
    got = lib.pcl_attach_cropper(h, C.byref(crop), 0x20000, 0x30000)
  elif call == 'tracking':
    got = lib.pcl_crop_tracking(h, C.byref(crop), 0x9000, 0x20000, 0x30000, None, None)
  elif call == 'handoff':
    out = _lib.Outputs(0x1000, 0x2000, 0x3000, 0x4000, 0x5000)
    x = _lib.HandoffState()
    x.n_peers, x.rank, x.record_bytes, x.rows, x.first_row = 1, 0, 96, 4, 0
    x.d_peer_base[0], x.d_peer_flags[0], x.d_local = 0x6000, 0x7000, 0x8000
    got = lib.pcl_crop_handoff(h, C.byref(crop), 0x9000, 0xa000, C.byref(out), C.byref(x), None)
  elif call == 'export':
    got = lib.pcl_export_curtain(h, arg, 0x20000, None)
  else:
    got = lib.pcl_layers(h, arg, len(arg), 0x20000, None)
  lib.pcl_destroy(h)
  assert got == want


def test_crop_handoff_mode_checks_on_cpu():
  """pcl_crop_handoff refuses inconsistent hand-off descriptions before it launches:
  unknown mode bits, split phase with fewer than three buffer parts, record sizes."""
  import ctypes as C
  from pycolab_b200 import batched
  art = levels.scrolly_maze_level(3, world_shape=(33, 33), board_shape=(16, 16))
  lib, h = _bound_handle(lowering.lower(g_scrolly.make_game(*art)))
  crop = batched.scrolling_crop_spec(9, 9, 0, pad_char=' ', scroll_margins=(None, None))
  out = _lib.Outputs(0x1000, 0x2000, 0x3000, 0x4000, 0x5000)

  def call(**kw):
    x = _lib.HandoffState()
    x.n_peers, x.rank, x.record_bytes, x.rows, x.first_row = 1, 0, 96, 4, 0
    x.d_peer_base[0], x.d_peer_flags[0], x.d_local = 0x6000, 0x7000, 0x8000
    for k, v in kw.items():
      setattr(x, k, v)
    return lib.pcl_crop_handoff(h, C.byref(crop), 0x9000, 0xa000, C.byref(out), C.byref(x), None)

  assert call(mode=8) == _lib.ERR_INVALID                              # unknown bit
  assert call(mode=_lib.HANDOFF_LAG, n_bufs=2) == _lib.ERR_INVALID     # split phase needs 3 parts
  assert call(mode=_lib.HANDOFF_LAG) == _lib.ERR_INVALID               # n_bufs 0 means 2
  assert call(n_bufs=9) == _lib.ERR_INVALID
  assert call(record_bytes=90) == _lib.ERR_INVALID                     # not a multiple of 16
  assert call(record_bytes=80) == _lib.ERR_INVALID                     # too small for 81 + 9 bytes
  assert call(rows=3) == _lib.ERR_INVALID                              # this rank's rows do not fit
  assert call(rank=1) == _lib.ERR_INVALID
  lib.pcl_destroy(h)


# ------------------------------------- scrolly_maze: shapes pcl_create accepts

import scrolly_shapes as ss   # noqa: E402


def _scrolly_spec(H, W, pitch=None, PW=None, pattern_words=None):
  """A scrolly_maze pcl_spec at any board shape (margins None on both drapes)."""
  game = lowering.lower(g_scrolly.make_game(*levels.scrolly_maze_level(
      0, world_shape=(33, 33), board_shape=(16, 16))))
  spec = game.make_spec(auto_reset=True)
  PW = PW if PW is not None else W + 64
  spec.rows, spec.cols = H, W
  spec.pitch = pitch if pitch is not None else ss.ceil16(W)
  spec.pattern_rows, spec.pattern_cols = H + 16, PW
  spec.pattern_words = pattern_words if pattern_words is not None else ss.min_pattern_words(W, PW)
  for d in range(2):
    spec.margins[d][0] = spec.margins[d][1] = -1
  return spec


def test_create_rejects_a_one_column_scrolly_pattern_too_short_for_four_staged_words():
  """The narrow path stages and reads 4 words per window row even at W = 1: a corner at
  column 64 of a 65-column pattern reads words 2..5, so 4 words per row are too few."""
  assert _create(_scrolly_spec(9, 1, PW=65, pattern_words=4)) == _lib.ERR_INVALID
  assert _create(_scrolly_spec(9, 1, PW=65, pattern_words=6)) == _lib.OK
  assert ss.min_pattern_words(1, 65) == 6


@pytest.mark.parametrize('W', [1, 2, 16, 31, 32, 33, 48, 63, 64, 65, 96, 127, 128, 129, 130])
def test_create_enforces_the_window_word_rule(W):
  """pcl_create accepts pattern_words exactly from the minimum the mirror computes."""
  for PW in (W, W + 1, W + 31, W + 64, W + 95, 3 * W + 70):
    want = ss.min_pattern_words(W, PW)
    assert _create(_scrolly_spec(7, W, PW=PW, pattern_words=want)) == _lib.OK, (W, PW)
    assert _create(_scrolly_spec(7, W, PW=PW, pattern_words=want - 2)) == _lib.ERR_INVALID, (W, PW)


def test_every_staged_word_stays_inside_its_warp_region_and_pattern_row():
  """The mirror of the kernel's layout: for every board width 1..130 (and pitches one
  segment wider), every shared-memory access of one warp lies inside the region
  warp_smem_bytes gives it, the two windows do not overlap, and every pattern word a
  staged row reads lies inside a row of the minimum pattern_words."""
  for W in range(1, 131):
    for pitch in (ss.ceil16(W), ss.ceil16(W) + 16):
      for H in (1, 5, 32, 33, 65):
        size = ss.warp_smem_bytes(H, W, pitch)
        nw = ss.window_words(W)
        wall = ss.REC_WORDS * 4 + H * pitch
        coin = wall + 4 * ((H * nw + 3) & ~3)
        assert coin >= wall + 4 * H * nw and coin + 4 * H * nw <= size, (W, pitch, H)
        for PW in (W, W + 40, W + 64, 2 * W + 100):
          for corner_c in {0, 31, 32, 63, 64, 95, 96, PW - W}:
            if corner_c > PW - W:
              continue
            acc, words = ss.warp_accesses(H, W, pitch, corner_c, PW)
            for off, n in acc:
              assert 0 <= off and off + n <= size, (W, pitch, H, corner_c, off, n, size)
            assert max(words) < ss.min_pattern_words(W, PW), (W, PW, corner_c)


@pytest.mark.parametrize('W', [16, 48, 64, 65, 128])
@pytest.mark.parametrize('extra', [0, 16])
def test_largest_accepted_scrolly_board_is_launchable(W, extra):
  """pcl_create's shared-memory test and the launcher's agree: at the largest H it
  accepts, the block (4 warps + the static selector tables) fits the 227 KB a block can
  opt in to; one row more is refused."""
  pitch = ss.ceil16(W) + extra
  lo, hi = 1, 4096
  assert _create(_scrolly_spec(lo, W, pitch)) == _lib.OK
  assert _create(_scrolly_spec(hi, W, pitch)) == _lib.ERR_UNSUPPORTED
  while hi - lo > 1:
    mid = (lo + hi) // 2
    if _create(_scrolly_spec(mid, W, pitch)) == _lib.OK:
      lo = mid
    else:
      hi = mid
  assert ss.accepted_smem(lo, W, pitch) and not ss.accepted_smem(lo + 1, W, pitch), (W, pitch, lo)
  block = ss.WARPS_PER_BLOCK * (ss.warp_smem_bytes(lo, W, pitch) + ss.SEL_TABLE_BYTES)
  assert block <= ss.MAX_BLOCK_SMEM
