"""CPU tests of plain Sprites on the compiled step program: things.Sprite subclasses whose
registered update() code sets their own position and visibility (`pycolab_b200.compiler`,
PCL_OP_SETFIELD in csrc/compiled.cu).

  - the oracle interpreter (oracle/compiled.py) raises IndexError where the reference fell
    (tests/golden/sprite_fallen.npz), after every frame before it;
  - the forms the compiler accepts and the ones it refuses, with the source line;
  - what lowering refuses: registers, position values, a plain Sprite's virtual_position;
  - pcl_bind_code / pcl_create checks of SETFIELD and program_arg[3], on handles that reach
    no device;
  - every compiled_step instantiation in the built library runs without a stack.
"""

import ctypes as C
import os

import pytest

import registered_games as rg
import test_kernel_resources as resources
from oracle import compiled as ocompiled
from pycolab_b200 import _lib, compiler, lowering
from pycolab_b200 import things as b_things
from pycolab_b200.errors import NotLoweredError
from pycolab_b200.prefab_parts import sprites as b_sprites


@pytest.fixture(scope='module')
def games():
  yield from rg.registered('sprite_games.py')


def test_oracle_raises_where_the_reference_fell(games):
  """sprite_fallen on the oracle: every frame before the reference's IndexError, then the
  IndexError (a case of test_registered_goldens too)."""
  rg.assert_oracle_replays(games, 'sprite_fallen')


# ------------------------------------------------------------ the subset --

def test_plain_sprites_compile_to_setfield(games):
  comp = lambda klass: compiler.registered(klass)
  ops = lambda klass: {ins[0] for ins in comp(klass).ir}
  for klass in (games.Ball, games.Blinker, games.Edge, games.Ghost, games.Faller):
    assert comp(klass).kind == 'plain'
    assert 'SETFIELD' in ops(klass), klass
  assert ('SETFIELD', _lib.FIELD_VISIBLE) in comp(games.Blinker).ir
  assert comp(games.Ball).attrs == ['_serve', 'dx', 'dy']
  assert comp(games.Ball).attr_types == {'dy': 'int', 'dx': 'int', '_serve': 'pos'}
  assert comp(games.Ball).n_registers == 4 and comp(games.Ball).slot('dx') == 2
  assert comp(games.Wanderer).attr_types == {'_home': 'pos', 'seen': 'int'}
  assert comp(games.Marker).attr_types == {'_mark': 'pos'}
  assert 'SETFIELD' not in ops(games.Paddle) and 'SETFIELD' not in ops(games.Bricks)


def test_roles_and_lowered_records(games):
  engine = games.make_bounce(0)
  assert lowering.role_of(engine.things['o']) == 'compiled.sprite'
  assert lowering.role_of(engine.things['P']) == 'compiled.walker'
  lowered = lowering.lower(engine)
  assert lowered.sprite_chars == 'Po' and lowered.program_arg[3] == 0b10
  ball = lowered.sprites[1]
  # row, col, _serve in VROW / VCOL, hidden, dx / dy in AUX0 / AUX1
  assert list(ball) == [4, 4, 4, 4, 0, 1, 1, 0]
  assert lowered.registers['o'] == [('_serve', b_things.Sprite.Position), ('dx', int), ('dy', int)]
  sampler = lowering.lower(games.make_sampler(0))
  assert sampler.registers['x'] == [('_mark', tuple)]
  assert sampler.program_arg[3] == sum(1 << sampler.sprite_chars.index(c) for c in 'bceg')


def _sprite(update, base=b_things.Sprite, **attrs):
  attrs.update(update=update, __module__=__name__)
  return type('Case', (base,), attrs)


def _accepted(self, actions, board, layers, backdrop, things, the_plot):
  self._position = self.Position(row=1, col=2)
  self._position = b_things.Sprite.Position(3, col=4)
  self._position = things['P'].position
  self._visible = self._position.row > 2 and not self._visible


def test_accepted_forms(games):
  ir = compiler.compile_class(_sprite(_accepted)).ir
  assert ir.count(('SETFIELD', _lib.FIELD_ROW)) == 3
  assert ir.count(('SETFIELD', _lib.FIELD_COL)) == 3
  assert ir.count(('SETFIELD', _lib.FIELD_VISIBLE)) == 1
  assert ('FIELD', ('ent', 'P'), _lib.FIELD_ROW) in ir


# Each refused construct on the marked line.
def _bare_tuple(self, actions, board, layers, backdrop, things, the_plot):
  self._position = (1, 2)                             # REFUSED


def _north(self, actions, board, layers, backdrop, things, the_plot):
  self._north(board, the_plot)                        # REFUSED


def _teleport(self, actions, board, layers, backdrop, things, the_plot):
  self._teleport((1, 2))                              # REFUSED


def _virtual(self, actions, board, layers, backdrop, things, the_plot):
  self.n = self.virtual_position.row                  # REFUSED


def _conflict(self, actions, board, layers, backdrop, things, the_plot):
  self._p = self.position
  self.n = self._p + 1                                # REFUSED


def _position_kwargs(self, actions, board, layers, backdrop, things, the_plot):
  self._position = self.Position(1, row=2)            # REFUSED


SPRITE_REFUSED = [(_bare_tuple, 'bare tuple'), (_north, '_north in a plain class'),
                  (_teleport, '_teleport in a plain class'),
                  (_virtual, '.virtual_position in a plain class'),
                  (_conflict, 'a position where a number is needed'),
                  (_position_kwargs, 'arguments of Position()')]


@pytest.mark.parametrize('update,what', SPRITE_REFUSED,
                         ids=[u.__name__ for u, _ in SPRITE_REFUSED])
def test_refused_construct_names_class_line_and_construct(update, what):
  rg.assert_refused(_sprite(update), what)


def _walker_writes_position(self, actions, board, layers, backdrop, things, the_plot):
  self._position = self.Position(1, 2)                # REFUSED


def test_walkers_still_refuse_position_writes():
  with pytest.raises(NotLoweredError, match='attribute self._position'):
    compiler.compile_class(_sprite(_walker_writes_position, base=b_sprites.MazeWalker))


def test_unregistered_plain_sprite_is_refused(games):
  engine = games.make_fallen()
  compiler.unregister(games.Faller)
  try:
    with pytest.raises(NotLoweredError, match='no device program'):
      lowering.lower(engine)
  finally:
    compiler.register(games.Faller)


# ------------------------------------------------------------ lowering limits --

def _many(self, actions, board, layers, backdrop, things, the_plot):
  self._a = self.position
  self._b = self.position
  self._c = self.position


def _reads_virtual(self, actions, board, layers, backdrop, things, the_plot):
  self.n = things['f'].virtual_position.row


def _fallen_with(games, klass, **attrs):
  """The fallen game with a second sprite 'P' of `klass`."""
  from pycolab_b200 import ascii_art
  compiler.register(klass)
  return ascii_art.ascii_art_to_game(
      [' f ', ' P ', '   '], what_lies_beneath=' ', sprites={'f': games.Faller, 'P': klass},
      update_schedule=[['f', 'P']], z_order='fP')


def test_lowering_refuses_register_overflow_and_bad_positions(games):
  klass = _sprite(_many)
  try:
    engine = _fallen_with(games, klass)
    ent = engine.things['P']
    ent._a, ent._b, ent._c = ent.position, (0, 0), (1, 1)
    with pytest.raises(NotLoweredError, match='needs 6 registers; a plain Sprite has 5'):
      lowering.lower(engine)
  finally:
    compiler.unregister(klass)

  def _two(self, actions, board, layers, backdrop, things, the_plot):
    self._a = self.position
    self.n = 1
  src_klass = _sprite(_two)
  try:
    engine = _fallen_with(games, src_klass)
    engine.things['P']._a, engine.things['P'].n = (1, 2.5), 0
    with pytest.raises(NotLoweredError, match='a position attribute holds'):
      lowering.lower(engine)
    engine = _fallen_with(games, src_klass)
    engine.things['P']._a, engine.things['P'].n = 7, 0
    with pytest.raises(NotLoweredError, match='a position attribute holds'):
      lowering.lower(engine)
    engine = _fallen_with(games, src_klass)
    engine.things['P']._a, engine.things['P'].n = (1, 2), 0
    assert lowering.lower(engine).registers['P'] == [('_a', tuple), ('n', int)]
  finally:
    compiler.unregister(src_klass)


def test_lowering_refuses_virtual_position_of_a_plain_sprite(games):
  klass = _sprite(_reads_virtual)
  try:
    engine = _fallen_with(games, klass)
    engine.things['P'].n = 0
    with pytest.raises(NotLoweredError, match="things\\['f'\\].virtual_position"):
      lowering.lower(engine)
  finally:
    compiler.unregister(klass)


# ------------------------------------------------------------ pcl_bind_code --

def test_bind_code_checks_setfield(games):
  lib = _lib.load()
  lowered = lowering.lower(games.make_bounce(0))
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

    def mutated(*changes):
      c = code.copy()
      for at, value in changes:
        c[at] = value
      return c
    ball_set = find('o', 'SETFIELD')
    ball_field = find('o', 'FIELD')
    paddle_move = find('P', 'MOVE')
    ball_getr = find('o', 'GETR')
    cases = {
        'SETFIELD in a walker': mutated((paddle_move, op('SETFIELD')), (paddle_move + 1, 0)),
        'SETFIELD of a virtual row': mutated((ball_set + 1, _lib.FIELD_VROW)),
        'SETFIELD of word 5': mutated((ball_set + 1, 5)),
        'MOVE in a plain sprite': mutated((ball_set, op('MOVE')), (ball_set + 1, 0)),
        'TELEPORT in a plain sprite': mutated((ball_set, op('TELEPORT'))),
        'FIELD 2 of a plain sprite': mutated((ball_field + 2, _lib.FIELD_VROW)),
        'FIELD 3 of a plain sprite by index': mutated((ball_field + 1, 1),
                                                      (ball_field + 2, _lib.FIELD_VCOL)),
        'plain register 5': mutated((ball_getr + 1, 5)),
    }
    # a TELEPORT pops two: keep the stack balanced so only the opcode is wrong
    for label, words in cases.items():
      assert rg.bind(lib, h, words) == _lib.ERR_INVALID, label
    assert rg.bind(lib, h, mutated((ball_getr + 1, 4))) == _lib.OK     # AUX2, the fifth
    # the paddle and the ball may not share a function
    shared = code.copy()
    shared[1 + lowered.sprite_chars.index('o')] = fn['P']
    assert rg.bind(lib, h, shared) == _lib.ERR_INVALID
  finally:
    lib.pcl_destroy(h)


def test_create_checks_plain_sprite_bits(games):
  lib = _lib.load()
  lowered = lowering.lower(games.make_sampler(0))
  ego = lowered.sprite_chars.index('P')
  for bits, want in ((lowered.program_arg[3], _lib.OK), (0, _lib.OK),
                     (lowered.program_arg[3] | 1 << ego, _lib.ERR_INVALID),
                     (1 << len(lowered.sprite_chars), _lib.ERR_INVALID),
                     (-2 ** 31, _lib.ERR_INVALID)):
    spec = lowered.make_spec(True)
    spec.program_arg[3] = bits
    h = C.c_void_p()
    assert lib.pcl_create(C.byref(spec), 4, -1, C.byref(h)) == want, bits
    if want == _lib.OK:
      lib.pcl_destroy(h)


@pytest.mark.skipif(resources._cuobjdump() is None, reason='cuobjdump not found')
def test_compiled_step_runs_without_a_stack():
  assert os.path.exists(_lib.LIB_PATH), 'build libpcl.so first'
  kernels = {n: u for n, u in resources._resource_usage(_lib.LIB_PATH).items()
             if 'compiled_step' in n}
  assert len(kernels) == 4, sorted(kernels)
  for name, u in kernels.items():
    assert u['STACK'] == 0, (name, u)
