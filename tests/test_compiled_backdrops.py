"""CPU tests of Backdrops with registered update() code on the compiled step program
(`pycolab_b200.compiler` kind 'backdrop', PCL_OP_SETBACK / FILLBACK / ROLLBACK, program_arg[4]):

  - the oracle interpreter (oracle/compiled.py) running the fluvial pair of
    tests/backdrop_games.py reproduces the reference's fluvial goldens (tests/golden/fluvial_*);
  - with the reference present, its own fluvial_natation classes, registered, lower to the
    compiled program and replay its goldens (tests/golden/fluvial_*), and the fluvial pair of
    tests/backdrop_games.py compiles to the same words;
  - the forms the compiler accepts and the ones it refuses, with the source line;
  - what lowering sets and refuses;
  - pcl_bind_code, pcl_bind_backdrop and pcl_create checks, on handles that reach no device;
  - no step kernel instantiation has a stack.
"""

import ctypes as C
import os

import numpy as np
import pytest

import example_games as eg
import golden_cases as gc
import refdriver
import registered_games as rg
import test_kernel_resources as resources
import trajectory as tj
from oracle import compiled as ocompiled
from pycolab_b200 import _lib, ascii_art, compiler, lowering
from pycolab_b200 import things as b_things
from pycolab_b200.errors import NotLoweredError
from pycolab_b200.prefab_parts import sprites as b_sprites

needs_ref = pytest.mark.skipif(not refdriver.available(), reason='reference not present')


@pytest.fixture(scope='module')
def games():
  yield from rg.registered('backdrop_games.py')


def _assert_oracle_replays(name, engine):
  """The oracle runs lowered `engine` like golden `name`, latching no error."""
  lowered = lowering.lower(engine)

  def no_error(world, out):
    assert world.error == 0
  eg.assert_replays('oracle', name, make_env=lambda: ocompiled.make_world(lowered),
                    check=no_error)


@pytest.mark.parametrize('name', gc.names('fluvial_'))
def test_oracle_runs_the_fluvial_pair_like_the_reference(games, name):
  _assert_oracle_replays(name, games.make_fluvial(tj.u8_to_art(gc.load(name)['art'])))


@pytest.fixture(scope='module')
def ref_fluvial():
  mod = rg.load(os.path.join(refdriver.REFERENCE_ROOT, 'pycolab', 'examples',
                             'fluvial_natation.py'))
  compiler.register(mod.PlayerSprite, mod.RiverBackdrop)
  yield mod
  compiler.unregister(mod.PlayerSprite, mod.RiverBackdrop)


@needs_ref
@pytest.mark.parametrize('name', gc.names('fluvial_'))
def test_reference_fluvial_classes_compile_and_replay(ref_fluvial, name):
  g = gc.load(name)
  art = tj.u8_to_art(g['art'])
  make = lambda: ascii_art.ascii_art_to_game(art, what_lies_beneath=' ',
                                             sprites={'P': ref_fluvial.PlayerSprite},
                                             backdrop=ref_fluvial.RiverBackdrop)
  lowered = lowering.lower(make())
  assert lowered.program == _lib.PROG_COMPILED and lowered.program_arg[4] == 1
  _assert_oracle_replays(name, make())


@needs_ref
def test_the_fluvial_pair_compiles_like_the_reference_classes(games, ref_fluvial):
  art = tj.u8_to_art(gc.load('fluvial_stock')['art'])
  ours = lowering.lower(games.make_fluvial(art))
  theirs = lowering.lower(ascii_art.ascii_art_to_game(
      art, what_lies_beneath=' ', sprites={'P': ref_fluvial.PlayerSprite},
      backdrop=ref_fluvial.RiverBackdrop))
  assert ours.code.tolist() == theirs.code.tolist()


def test_unregistered_river_stays_on_the_classics_program(games):
  from pycolab_b200.games import fluvial_natation
  lowered = lowering.lower(fluvial_natation.make_game())
  assert lowered.program == _lib.PROG_CLASSICS and lowered.backdrop_role == 'river'


# ------------------------------------------------------------ the subset --

def _backdrop(update, **attrs):
  attrs.update(update=update, __module__=__name__)
  return type('Case', (b_things.Backdrop,), attrs)


def _accepted(self, actions, board, layers, things, the_plot):
  n = board.shape[1] + self.curtain.shape[0] + board.shape[0]
  self.curtain[0, 1] = self.palette.hash
  self.curtain[things['P'].position] = self.palette['#'] if n > 3 else ord('x')
  self.curtain[1, 1] = self.curtain[0, 0] if layers['#'][1, 2] else True
  self.curtain[2, 2] = board[1, 1]
  self.curtain[:] = 255
  self.curtain[1:-1] = np.roll(self.curtain[1:-1], -n, 0)
  self.curtain[:, :] = np.roll(self.curtain[:], shift=np.random.randint(3), axis=1)
  self.curtain[-9:2, :] = np.roll(self.curtain[-9:2, :], the_plot['k'], axis=1)
  the_plot['k'] = self.curtain[0, 0] + things['P'].visible


def test_accepted_forms_compile_to_the_backdrop_opcodes():
  comp = compiler.compile_class(_backdrop(_accepted))
  assert comp.kind == 'backdrop' and comp.attrs == [] and comp.keys == ['k']
  ops = [ins[0] for ins in comp.ir]
  assert ops.count('SETBACK') == 4 and ops.count('FILLBACK') == 1 and ops.count('ROLLBACK') == 3
  assert ('PUSH', ('palette', '#')) in comp.ir and ('PUSH', ('cols',)) in comp.ir
  assert ('PUSH', ('rows',)) in comp.ir and 'BACKDROP' in ops and 'RANDINT' in ops
  rolls = [ins for ins in comp.ir if ins[0] == 'ROLLBACK']
  assert rolls == [('ROLLBACK', 0, ('lo', 1, -1), ('hi', 1, -1)),
                   ('ROLLBACK', 1, ('lo', None, None), ('hi', None, None)),
                   ('ROLLBACK', 1, ('lo', -9, 2), ('hi', -9, 2))]
  # clipped as a Python slice at link time: rows 1..3 of 5, none of [-9:2] past row 2
  words = compiler._encode(comp, 0, ['P'], 1, 5, 7, ['k'], ('numpy',))
  at = [i for i, w in enumerate(words) if w == _lib.OP['ROLLBACK']]
  assert [words[i + 1:i + 4] for i in at[-3:]] == [[0, 1, 4], [1, 0, 5], [1, 0, 2]]


def _shape_in_a_walker(self, actions, board, layers, backdrop, things, the_plot):
  if self.virtual_position[1] >= board.shape[1] or board.shape == (3, 4):
    the_plot.add_reward(board.shape[0])


def test_board_shape_compiles_in_every_kind():
  klass = type('Case', (b_sprites.MazeWalker,), dict(update=_shape_in_a_walker,
                                                     __module__=__name__))
  ir = compiler.compile_class(klass).ir
  assert ('PUSH', ('cols',)) in ir and ('PUSH', ('rows',)) in ir and ('EQ2',) in ir


# Each refused construct on the marked line.
def _attribute(self, actions, board, layers, things, the_plot):
  self._t += 1                                                    # REFUSED


def _column_slice(self, actions, board, layers, things, the_plot):
  self.curtain[:, 1] = 0                                          # REFUSED


def _stepped(self, actions, board, layers, things, the_plot):
  self.curtain[::2] = np.roll(self.curtain[::2], 1, 1)           # REFUSED


def _other_band(self, actions, board, layers, things, the_plot):
  self.curtain[1:3] = np.roll(self.curtain[1:4], 1, axis=1)      # REFUSED


def _no_axis(self, actions, board, layers, things, the_plot):
  self.curtain[1:3] = np.roll(self.curtain[1:3], 1)              # REFUSED


def _axis_variable(self, actions, board, layers, things, the_plot):
  a = 1
  self.curtain[:] = np.roll(self.curtain, 1, axis=a)             # REFUSED


def _big_int(self, actions, board, layers, things, the_plot):
  self.curtain[0, 0] = 256                                        # REFUSED


def _local_value(self, actions, board, layers, things, the_plot):
  v = 3
  self.curtain[0, 0] = v                                          # REFUSED


def _sum_value(self, actions, board, layers, things, the_plot):
  self.curtain[0, 0] = self.palette.a + 1                         # REFUSED


def _band_fill(self, actions, board, layers, things, the_plot):
  self.curtain[1:3] = 0                                           # REFUSED


def _draw_value(self, actions, board, layers, things, the_plot):
  self.curtain[:] = np.random.randint(3)                          # REFUSED


def _motion(self, actions, board, layers, things, the_plot):
  self._north(board, the_plot)                                    # REFUSED


REFUSED = [(_attribute, 'a Backdrop has no registers'), (_column_slice, 'a band of rows'),
           (_stepped, 'a stepped slice'), (_other_band, 'another band'),
           (_no_axis, 'axis that is not the literal 0 or 1'),
           (_axis_variable, 'axis that is not the literal 0 or 1'),
           (_big_int, 'outside 0..255'), (_local_value, 'outside 0..255'),
           (_sum_value, 'outside 0..255'), (_band_fill, 'other than np.roll'),
           (_draw_value, 'outside 0..255'), (_motion, '_north in a backdrop class')]


@pytest.mark.parametrize('update,what', REFUSED, ids=[u.__name__ for u, _ in REFUSED])
def test_refused_construct_names_class_line_and_construct(update, what):
  rg.assert_refused(_backdrop(update), what)


def _sprite_writes_backdrop(self, actions, board, layers, backdrop, things, the_plot):
  backdrop.curtain[0, 0] = 1                                      # REFUSED


def test_sprites_and_drapes_may_not_write_the_backdrop():
  for base in (b_sprites.MazeWalker, b_things.Drape):
    klass = type('Case', (base,), dict(update=_sprite_writes_backdrop, __module__=__name__))
    with pytest.raises(NotLoweredError, match='a write to backdrop.curtain'):
      compiler.compile_class(klass)


def test_a_backdrop_without_update_is_refused():
  with pytest.raises(NotLoweredError, match='no update'):
    compiler.register(type('Plain', (b_things.Backdrop,), {}))


# ------------------------------------------------------------ lowering --

def _palette_x(self, actions, board, layers, things, the_plot):
  self.curtain[0, 0] = self.palette.x


def test_lowering_sets_the_backdrop_entry_and_checks_the_palette(games):
  lowered = lowering.lower(games.make_trail(0))
  n = len(lowered.sprite_chars + lowered.drape_chars)
  assert lowered.program_arg[4] == 1 and lowered.backdrop_role == 'compiled.backdrop'
  code = lowered.code
  entry = code[1 + n]
  assert code[0] == n and entry > max(code[1:1 + n])
  assert _lib.OP['SETBACK'] in code[entry:].tolist()
  klass = _backdrop(_palette_x)
  compiler.register(klass)
  try:
    engine = ascii_art.ascii_art_to_game(['#P#'], ' ', sprites={'P': games.Walker},
                                         backdrop=klass)
    with pytest.raises(NotLoweredError, match="self.palette names 'x'"):
      lowering.lower(engine)
  finally:
    compiler.unregister(klass)


def test_a_registered_backdrop_needs_registered_entities(games):
  from pycolab_b200.games import fluvial_natation
  engine = ascii_art.ascii_art_to_game(fluvial_natation.GAME_ART, ' ',
                                       sprites={'P': fluvial_natation.PlayerSprite},
                                       backdrop=games.River)
  with pytest.raises(NotLoweredError):
    lowering.lower(engine)
  # an unregistered Backdrop with logic under registered entities is refused as before
  engine = ascii_art.ascii_art_to_game(fluvial_natation.GAME_ART, ' ',
                                       sprites={'P': games.Swimmer},
                                       backdrop=fluvial_natation.RiverBackdrop)
  with pytest.raises(NotLoweredError):
    lowering.lower(engine)


# ------------------------------------------------------------ the C boundary --

def test_bind_code_checks_the_backdrop_function(games):
  lib = _lib.load()
  lowered = lowering.lower(games.make_flow(0))
  spec = lowered.make_spec(True)
  code = lowered.code.copy()
  n = len(lowered.sprite_chars + lowered.drape_chars)
  op = lambda name: _lib.OP[name]
  entry = int(code[1 + n])
  h = rg.handle(lib, spec)
  try:
    assert rg.bind(lib, h, code) == _lib.OK
    roll = entry + [i for i, w in enumerate(code[entry:].tolist()) if w == op('ROLLBACK')][0]
    fill = entry + [i for i, w in enumerate(code[entry:].tolist()) if w == op('FILLBACK')][0]
    walker = int(code[1])
    move = walker + [i for i, w in enumerate(code[walker:entry].tolist()) if w == op('MOVE')][0]

    def mutated(*changes):
      c = code.copy()
      for at, value in changes:
        c[at] = value
      return c
    cases = {
        'no entry word': np.concatenate([code[:1 + n], code[2 + n:]]),
        'entry out of range': mutated((1 + n, len(code))),
        'entry shared with the walker': mutated((1 + n, walker)),
        'axis 2': mutated((roll + 1, 2)),
        'lo > hi': mutated((roll + 2, 3), (roll + 3, 2)),
        'hi past the rows': mutated((roll + 3, lowered.rows + 1)),
        'lo < 0': mutated((roll + 2, -1)),
        'FILLBACK in the walker': mutated((move, op('FILLBACK')), (move + 1, op('POP'))),
        'SETR in the Backdrop': mutated((fill, op('SETR'))),
        'FILL in the Backdrop': mutated((fill, op('FILL'))),
    }
    for label, words in cases.items():
      assert rg.bind(lib, h, words) == _lib.ERR_INVALID, label
    assert rg.bind(lib, h, mutated((roll + 2, 0), (roll + 3, lowered.rows))) == _lib.OK
  finally:
    lib.pcl_destroy(h)


def test_bind_backdrop_and_create_checks(games):
  lib = _lib.load()
  lowered = lowering.lower(games.make_flow(0))
  spec = lowered.make_spec(True)
  h = rg.handle(lib, spec)
  try:
    assert lib.pcl_bind_backdrop(h, None) == _lib.ERR_INVALID
    assert lib.pcl_bind_backdrop(h, 0x1000) == _lib.OK
    assert lib.pcl_bind_backdrop(None, 0x1000) == _lib.ERR_INVALID
  finally:
    lib.pcl_destroy(h)
  # handles without a compiled Backdrop refuse it
  spec0 = lowered.make_spec(True)
  spec0.program_arg[4] = 0
  h = rg.handle(lib, spec0)
  try:
    assert lib.pcl_bind_backdrop(h, 0x1000) == _lib.ERR_INVALID
  finally:
    lib.pcl_destroy(h)
  from pycolab_b200.games import fluvial_natation
  h = rg.handle(lib, lowering.lower(fluvial_natation.make_game()).make_spec(True))
  try:
    assert lib.pcl_bind_backdrop(h, 0x1000) == _lib.ERR_INVALID
  finally:
    lib.pcl_destroy(h)
  for bad in (2, -1):
    spec = lowered.make_spec(True)
    spec.program_arg[4] = bad
    h = C.c_void_p()
    assert lib.pcl_create(C.byref(spec), 4, -1, C.byref(h)) == _lib.ERR_INVALID, bad


def test_steps_wait_for_the_live_backdrop(games):
  """A handle with a compiled Backdrop and bound state and code but no live curtain refuses
  every step and reset entry point before it launches anything."""
  lib = _lib.load()
  lowered = lowering.lower(games.make_flow(0))
  h = rg.handle(lib, lowered.make_spec(True))
  try:
    st = _lib.State()
    fake = 0x1000
    st.d_backdrop = st.d_plot = st.d_plot_init = st.d_sprites = st.d_sprites_init = fake
    st.d_z_order = st.d_z_order_init = st.d_rng = fake
    assert lib.pcl_bind_state(h, C.byref(st)) == _lib.OK
    assert rg.bind(lib, h, lowered.code) == _lib.OK
    out = _lib.Outputs(fake, fake, fake, fake, fake)
    assert lib.pcl_reset(h, None, C.byref(out), None) == _lib.ERR_UNBOUND
    assert lib.pcl_step(h, fake, C.byref(out), None) == _lib.ERR_UNBOUND
    assert lib.pcl_run(h, fake, 3, C.byref(out), None) == _lib.ERR_UNBOUND
    chars = b'P'
    assert lib.pcl_layers(h, chars, 1, fake, None) == _lib.ERR_UNBOUND
  finally:
    lib.pcl_destroy(h)


@pytest.mark.skipif(resources._cuobjdump() is None, reason='cuobjdump not found')
def test_step_kernels_run_without_a_stack():
  assert os.path.exists(_lib.LIB_PATH), 'build libpcl.so first'
  kernels = {n: u for n, u in resources._resource_usage(_lib.LIB_PATH).items()
             if 'compiled_step' in n or 'backdrop_step' in n}
  assert len(kernels) == 8, sorted(kernels)
  for name, u in kernels.items():
    assert u['STACK'] == 0, (name, u)
